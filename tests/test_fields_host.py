"""CPU tests of execute(values=...) (several value fields through one factorisation) on the host side.

`_cabi.Handle` is replaced by tests/fields_emulator.py, which implements kb200_set_values with the oracle per column, so
what is checked here is the product code above the C ABI: validation of `values`, the problem cache key, chunking above
the field limit, the scatter of masked grids and the output shapes. The device kernels are tests/test_fields_gpu.py."""
import numpy as np
import pytest
from numpy.testing import assert_array_equal

import cases
from fields_emulator import FieldsEmulatedHandle

EXP = [1.0, 300.0, 0.05]


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", FieldsEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def _fields(seed, n, V):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(n, V)) * np.linspace(1.0, 5.0, V) + np.arange(V)


def _make(pk, kind, xyz, z, **kw):
    kw = dict(variogram_model="exponential", variogram_parameters=EXP, **kw)
    if kind == "ok":
        return pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], z, **kw)
    if kind == "uk":
        return pk.UniversalKriging(xyz[:, 0], xyz[:, 1], z, drift_terms=["regional_linear"], **kw)
    if kind == "ok3d":
        return pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, **kw)
    return pk.UniversalKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, drift_terms=["regional_linear"], **kw)


def _data(kind, n=30, seed=5):
    dim = 3 if kind.endswith("3d") else 2
    return cases.synth_data(seed, n, dim)


def _grid_args(kind):
    ax = [np.linspace(50.0, 950.0, 7), np.linspace(80.0, 900.0, 5)]
    if kind.endswith("3d"):
        ax.append(np.linspace(10.0, 240.0, 3))
    return ax


def _execute(model, kind, style, coords, **kw):
    mask = None
    if style == "masked":
        shape = tuple(c.size for c in coords)[::-1]
        mask = np.zeros(shape, dtype=bool)
        mask.flat[::3] = True
    return model.execute(style, *coords, mask=mask, **kw) if mask is not None else model.execute(style, *coords, **kw)


KINDS = ["ok", "uk", "ok3d", "uk3d"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("style", ["grid", "masked", "points"])
def test_shapes_and_fields_match_single_field_calls(pk, kind, style):
    """zvalues gains a leading field axis, sigmasq keeps its shape, and field v equals execute() on an object built
    with z = values[:, v] and the same fixed variogram; a 1-D values gives today's shapes."""
    xyz, val = _data(kind)
    F = _fields(1, xyz.shape[0], 3)
    model = _make(pk, kind, xyz, val)
    if style == "points":
        pts = cases.synth_points(2, 9, xyz.shape[1], xyz)
        coords = [pts[:, c] for c in range(xyz.shape[1])]
    else:
        coords = _grid_args(kind)
    z0, s0 = _execute(model, kind, style, coords)
    z, s = _execute(model, kind, style, coords, values=F)
    assert z.shape == (3,) + z0.shape and s.shape == s0.shape
    assert_array_equal(np.ma.getdata(s), np.ma.getdata(s0))
    if style == "masked":
        assert np.ma.is_masked(z)
        assert_array_equal(np.ma.getmaskarray(z), np.broadcast_to(np.ma.getmaskarray(z0), z.shape))
    for v in range(3):
        zv, sv = _execute(_make(pk, kind, xyz, F[:, v]), kind, style, coords)
        assert_array_equal(np.ma.getdata(z[v]), np.ma.getdata(zv))
        assert_array_equal(np.ma.getdata(s), np.ma.getdata(sv))
    z1, s1 = _execute(model, kind, style, coords, values=F[:, 1])
    assert z1.shape == z0.shape and s1.shape == s0.shape
    assert_array_equal(np.ma.getdata(z1), np.ma.getdata(z[1]))


@pytest.mark.parametrize("kind", ["ok", "ok3d"])
def test_moving_window_with_fields(pk, kind):
    xyz, val = _data(kind, n=40)
    F = _fields(3, xyz.shape[0], 4)
    model = _make(pk, kind, xyz, val)
    coords = _grid_args(kind)
    z, s = _execute(model, kind, "grid", coords, values=F, n_closest_points=6)
    for v in (0, 3):
        zv, sv = _execute(_make(pk, kind, xyz, F[:, v]), kind, "grid", coords, n_closest_points=6)
        assert_array_equal(z[v], zv)
        assert_array_equal(s, sv)


def test_refusals(pk):
    xyz, val = _data("ok")
    n = xyz.shape[0]
    ok = _make(pk, "ok", xyz, val)
    p = [np.array([100.0, 500.0]), np.array([200.0, 300.0])]
    for bad in (np.zeros((n + 1, 2)), np.zeros((2, n)), np.zeros((n, 2, 1)), np.zeros(()), np.zeros((n, 0))):
        with pytest.raises(ValueError):
            ok.execute("points", *p, values=bad)
    F = _fields(0, n, 2)
    F[3, 1] = np.nan
    with pytest.raises(ValueError):
        ok.execute("points", *p, values=F)
    F[3, 1] = np.inf
    with pytest.raises(ValueError):
        ok.execute("points", *p, values=F)
    good = _fields(0, n, 2)
    for dtype in ("float32", "float64x"):
        with pytest.raises(NotImplementedError):
            ok.execute("points", *p, values=good, dtype=dtype)
    with pytest.raises(NotImplementedError):
        ok.execute("points", *p, values=good, n_gpus=2)
    pinv = _make(pk, "ok", xyz, val, pseudo_inv=True)
    with pytest.raises(NotImplementedError):
        pinv.execute("points", *p, values=good)
    z, _ = pinv.execute("points", *p, values=good, n_closest_points=5)   # the moving window ignores pseudo_inv
    assert z.shape == (2, 2)
    # the reference's own argument checks come first and are unchanged
    with pytest.raises(ValueError, match="style argument"):
        ok.execute("nope", *p, values=good)
    with pytest.raises(ValueError, match="at least two"):
        ok.execute("points", *p, values=good, n_closest_points=1)


def test_every_float64_spelling_is_accepted(pk):
    """Every dtype spelling that execute() runs as float64 also runs with values=, with the same result."""
    xyz, val = _data("ok")
    coords = _grid_args("ok")
    F = _fields(4, xyz.shape[0], 2)
    z0, s0 = _make(pk, "ok", xyz, val).execute("grid", *coords, values=F)
    for dtype in ("f8", np.float64, np.dtype("float64")):
        z, s = _make(pk, "ok", xyz, val).execute("grid", *coords, values=F, dtype=dtype)
        assert_array_equal(z, z0)
        assert_array_equal(s, s0)


def test_chunking_is_invisible(pk, monkeypatch):
    """Above the field limit the call runs as several problems; field v's result does not change."""
    from pykrige_b200 import _cabi
    xyz, val = _data("uk")
    F = _fields(7, xyz.shape[0], 7)
    coords = _grid_args("uk")
    whole = _make(pk, "uk", xyz, val).execute("grid", *coords, values=F)
    monkeypatch.setattr(_cabi, "MAX_FIELDS", 3)
    model = _make(pk, "uk", xyz, val)
    z, s = model.execute("grid", *coords, values=F)
    assert model._kb_handle.calls.count("set_problem") == 3          # chunks of 3, 3, 1
    assert_array_equal(z, whole[0])
    assert_array_equal(s, whole[1])


def test_cache_and_statistics_are_unchanged(pk):
    """A fields call does not leave its values behind: a later execute() without values gives exactly what it gave
    before, and the statistics still belong to the constructor's z."""
    xyz, val = _data("ok")
    coords = _grid_args("ok")
    ok = _make(pk, "ok", xyz, val, enable_statistics=True)
    q = (ok.Q1, ok.Q2, ok.cR)
    z0, s0 = ok.execute("grid", *coords)
    F = _fields(9, xyz.shape[0], 2)
    ok.execute("grid", *coords, values=F)
    assert ok._kb_key.n_fields == 2
    z1, s1 = ok.execute("grid", *coords)
    assert_array_equal(z1, z0)
    assert_array_equal(s1, s0)
    assert ok._kb_key.n_fields == 0 and ok._kb_key == ok._problem_key(ok._kb_key.dtype, False)
    assert (ok.Q1, ok.Q2, ok.cR) == q
    np.testing.assert_array_equal(ok.Z, val)
    F2 = F.copy()
    F2[0, 0] += 1.0                            # other values: a new problem, not the cached one
    za, _ = ok.execute("grid", *coords, values=F)
    zb, _ = ok.execute("grid", *coords, values=F2)
    assert not np.array_equal(za[0], zb[0])
    assert_array_equal(za[1], zb[1])
