"""CPU tests of add_data() on the host side.

`_cabi.Handle` is replaced by tests/append_emulator.py (kb200_append_data with the header's semantics on the oracle), so
what is checked here is the product code above the C ABI: the public attributes after add_data against an object built
on the concatenated data with the current variogram as fixed parameters, the argument checks, which cases extend the
held problem and which fall back, and the problem cache afterwards. The device kernels are tests/test_append_gpu.py."""
import inspect

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import cases
from append_emulator import AppendEmulatedHandle

EXP = [1.0, 300.0, 0.05]
NAMES = {"linear": ("slope", "nugget"), "power": ("scale", "exponent", "nugget")}


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated device: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", AppendEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def fixed(model):
    """The object's current variogram as the dict of fixed parameters a new object is given."""
    p = list(model.variogram_model_parameters)
    return dict(zip(NAMES.get(model.variogram_model, ("psill", "range", "nugget")), p))


def _make(pk, kind, xyz, z, spec=None, **kw):
    kw.setdefault("variogram_model", "exponential")
    kw.setdefault("variogram_parameters", EXP)
    if kind == "ok":
        return pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], z, **kw)
    if kind == "uk":
        kw.setdefault("drift_terms", ["regional_linear"])
        return pk.UniversalKriging(xyz[:, 0], xyz[:, 1], z, specified_drift=spec, **kw)
    if kind == "ok3d":
        return pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, **kw)
    kw.setdefault("drift_terms", ["regional_linear"])
    return pk.UniversalKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, specified_drift=spec, **kw)


def _add(model, xyz, z, spec=None):
    if xyz.shape[1] == 2:
        model.add_data(xyz[:, 0], xyz[:, 1], z, specified_drift=spec)
    else:
        model.add_data(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, specified_drift=spec)


def _split(kind, n=30, m=7, seed=3):
    xyz, val = cases.synth_data(seed, n + m, 3 if kind.endswith("3d") else 2)
    return xyz, val, n


def _points(kind):
    g = np.linspace(-50.0, 1050.0, 6)
    return (g, g) if not kind.endswith("3d") else (g, g, np.linspace(0.0, 250.0, 3))


KINDS = ["ok", "uk", "ok3d", "uk3d"]
ANISO = {"ok": dict(anisotropy_scaling=2.0, anisotropy_angle=30.0), "uk": dict(anisotropy_scaling=1.5, anisotropy_angle=-20.0),
         "ok3d": dict(anisotropy_scaling_y=1.5, anisotropy_angle_z=25.0),
         "uk3d": dict(anisotropy_scaling_z=2.0, anisotropy_angle_x=10.0)}


def test_emulator_method_has_the_handle_signature():
    from pykrige_b200 import _cabi
    assert inspect.signature(AppendEmulatedHandle.append_data) == inspect.signature(_cabi.Handle.append_data)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("held", [False, True])
def test_attributes_and_results_equal_a_new_object(pk, kind, held):
    """X_ORIG... and the values bit for bit, the centre and adjusted coordinates, lags / semivariance, execute() and
    leave_one_out() equal those of an object built on old + new stations with the current variogram fixed; with a
    held problem the device problem is extended (no new set_problem), without one the next execute() sets it up."""
    xyz, val, n = _split(kind)
    model = _make(pk, kind, xyz[:n], val[:n], **ANISO[kind])
    if held:
        model.execute("grid", *_points(kind))
    h = getattr(model, "_kb_handle", None)
    _add(model, xyz[n:], val[n:])
    ref = _make(pk, kind, xyz, val, variogram_parameters=fixed(model), **ANISO[kind])
    for c in ref._AXES:
        assert_array_equal(getattr(model, c + "_ORIG"), getattr(ref, c + "_ORIG"))
        assert getattr(model, c + "CENTER") == getattr(ref, c + "CENTER")
        assert_array_equal(getattr(model, c + "_ADJUSTED"), getattr(ref, c + "_ADJUSTED"))
    assert_array_equal(getattr(model, model._VALUES), getattr(ref, ref._VALUES))
    assert_array_equal(model.lags, ref.lags)
    assert_array_equal(model.semivariance, ref.semivariance)
    z, s = model.execute("grid", *_points(kind))
    zr, sr = ref.execute("grid", *_points(kind))
    assert_allclose(z, zr, rtol=1e-9, atol=1e-9 * np.abs(zr).max())
    assert_allclose(s, sr, rtol=1e-9, atol=1e-9 * np.abs(sr).max())
    if held:
        assert h is model._kb_handle and h.calls.count("set_problem") == 1 and "append_data" in h.calls
    else:
        assert model._kb_handle.calls.count("set_problem") == 1 and "append_data" not in model._kb_handle.calls
    lz, ls = model.leave_one_out()
    rz, rs = ref.leave_one_out()
    assert_allclose(lz, rz, rtol=1e-9, atol=1e-9 * np.abs(rz).max())
    assert_allclose(ls, rs, rtol=1e-9, atol=1e-9 * np.abs(rs).max())


def test_refitted_variogram_is_kept_and_statistics_follow_the_data(pk):
    """An automatically fitted variogram is not refitted; the statistics are those of the new object."""
    xyz, val, n = _split("ok3d", n=26, m=6)
    model = pk.OrdinaryKriging3D(xyz[:n, 0], xyz[:n, 1], xyz[:n, 2], val[:n], variogram_model="spherical")
    params = list(model.variogram_model_parameters)
    assert model.Q1 is not None
    _add(model, xyz[n:], val[n:])
    assert list(model.variogram_model_parameters) == params
    ref = pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], val, variogram_model="spherical",
                               variogram_parameters=fixed(model))
    for name in ("delta", "sigma", "epsilon"):
        assert_allclose(getattr(model, name), getattr(ref, name), rtol=1e-12, atol=1e-12)
    assert model.Q1 == pytest.approx(ref.Q1, rel=1e-12) and model.cR == pytest.approx(ref.cR, rel=1e-12)


def test_universal_drift_terms(pk):
    """regional_linear + point_log + external_Z + specified + functional: the drift data of the new stations as the
    constructor computes them, and the results of the new object."""
    xyz, val, n = _split("uk", n=30, m=9)
    rng = np.random.default_rng(4)
    ex, ey = np.linspace(-100.0, 1100.0, 13), np.linspace(-100.0, 1100.0, 11)
    ez = rng.normal(size=(ey.size, ex.size))
    spec = rng.normal(size=n + 9)
    kw = dict(drift_terms=["regional_linear", "point_log", "external_Z", "specified", "functional"],
              point_drift=[[480.0, 520.0, 0.7]], external_drift=ez, external_drift_x=ex, external_drift_y=ey,
              functional_drift=[lambda x, y: np.sin(x / 300.0) * y / 1000.0])
    model = _make(pk, "uk", xyz[:n], val[:n], spec=[spec[:n]], **kw)
    pts = (np.linspace(0.0, 1000.0, 5), np.linspace(0.0, 1000.0, 4))
    sdrift = [rng.normal(size=(4, 5))]
    model.execute("grid", *pts, specified_drift_arrays=sdrift)
    _add(model, xyz[n:], val[n:], spec=[spec[n:]])
    assert "append_data" in model._kb_handle.calls
    ref = _make(pk, "uk", xyz, val, spec=[spec], variogram_parameters=fixed(model), **kw)
    assert_array_equal(model.z_scalars, ref.z_scalars)
    assert_array_equal(model.specified_drift_data_arrays[0], ref.specified_drift_data_arrays[0])
    assert_allclose(model.point_log_array, ref.point_log_array, rtol=0, atol=1e-9)
    z, s = model.execute("grid", *pts, specified_drift_arrays=sdrift)
    zr, sr = ref.execute("grid", *pts, specified_drift_arrays=sdrift)
    assert model._kb_handle.calls.count("set_problem") == 1
    assert_allclose(z, zr, rtol=1e-9, atol=1e-9 * np.abs(zr).max())
    assert_allclose(s, sr, rtol=1e-9, atol=1e-9 * np.abs(sr).max())


def test_argument_errors_change_nothing(pk):
    xyz, val, n = _split("uk", n=20, m=4)
    ex, ey = np.linspace(0.0, 1000.0, 9), np.linspace(0.0, 1000.0, 9)
    model = _make(pk, "uk", xyz[:n], val[:n], spec=[np.ones(n)], drift_terms=["specified", "external_Z"],
                  external_drift=np.ones((9, 9)), external_drift_x=ex, external_drift_y=ey)
    new, v = xyz[n:], val[n:]
    with pytest.raises(ValueError, match="same non-zero length"):
        model.add_data(new[:, 0], new[:3, 1], v, specified_drift=[np.ones(4)])
    with pytest.raises(ValueError, match="finite"):
        model.add_data(new[:, 0], new[:, 1], np.where(np.arange(4) == 2, np.nan, v), specified_drift=[np.ones(4)])
    with pytest.raises(ValueError, match="at least one drift-value array"):
        model.add_data(new[:, 0], new[:, 1], v)
    with pytest.raises(TypeError, match="encapsulated in a list"):
        model.add_data(new[:, 0], new[:, 1], v, specified_drift=np.ones(4))
    with pytest.raises(ValueError, match="for each data point"):
        model.add_data(new[:, 0], new[:, 1], v, specified_drift=[np.ones(3)])
    with pytest.raises(ValueError, match="Inconsistent number"):
        model.add_data(new[:, 0], new[:, 1], v, specified_drift=[np.ones(4), np.ones(4)])
    with pytest.raises(ValueError, match="does not cover"):
        model.add_data(new[:, 0] + 2000.0, new[:, 1], v, specified_drift=[np.ones(4)])
    assert model.X_ORIG.size == n and model.z_scalars.size == n and model.specified_drift_data_arrays[0].size == n
    ok = _make(pk, "ok", xyz[:n], val[:n])
    with pytest.warns(RuntimeWarning, match="'specified' drift was not initialized"):
        ok.add_data(new[:, 0], new[:, 1], v, specified_drift=[np.ones(4)])


def _appended(model):
    h = getattr(model, "_kb_handle", None)
    return h is not None and "append_data" in h.calls


@pytest.mark.parametrize("case", ["knn", "pinv", "fields", "functional_aniso", "nothing_held"])
def test_fallbacks_equal_a_new_object(pk, case):
    """No device extension in these cases: the next execute() sets the problem up from scratch."""
    xyz, val, n = _split("uk", n=24, m=5)
    xyz[n:, 0] += 200.0                                  # the centre moves
    pts = (np.linspace(0.0, 1000.0, 5), np.linspace(0.0, 1000.0, 4))
    kw, ex = {}, {}
    kind = "ok"
    if case == "pinv":
        kw = dict(pseudo_inv=True)
    if case == "functional_aniso":
        kind = "uk"
        kw = dict(drift_terms=["functional"], functional_drift=[lambda x, y: (x / 500.0) ** 2],
                  anisotropy_scaling=2.0, anisotropy_angle=40.0)
    if case == "knn":
        ex = dict(n_closest_points=6)
    model = _make(pk, kind, xyz[:n], val[:n], **kw)
    if case == "fields":
        model.execute("grid", *pts, values=np.ones((n, 2)))
    elif case != "nothing_held":
        model.execute("grid", *pts, **ex)
    _add(model, xyz[n:], val[n:])
    assert not _appended(model)
    ref = _make(pk, kind, xyz, val, variogram_parameters=fixed(model), **kw)
    z, s = model.execute("grid", *pts, **ex)
    zr, sr = ref.execute("grid", *pts, **ex)
    assert_allclose(z, zr, rtol=1e-9, atol=1e-9 * np.abs(zr).max())
    assert_allclose(s, sr, rtol=1e-9, atol=1e-9 * np.abs(sr).max())


def test_functional_drift_without_anisotropy_is_extended(pk):
    xyz, val, n = _split("uk", n=24, m=5)
    kw = dict(drift_terms=["functional"], functional_drift=[lambda x, y: (x / 500.0) ** 2])
    model = _make(pk, "uk", xyz[:n], val[:n], **kw)
    pts = (np.linspace(0.0, 1000.0, 5), np.linspace(0.0, 1000.0, 4))
    model.execute("grid", *pts)
    _add(model, xyz[n:], val[n:])
    assert _appended(model)
    ref = _make(pk, "uk", xyz, val, variogram_parameters=fixed(model), **kw)
    assert_allclose(model.execute("grid", *pts)[0], ref.execute("grid", *pts)[0], rtol=1e-9)


def test_cache_key_hits_next_execute_and_misses_every_other_change(pk):
    xyz, val, n = _split("ok", n=24, m=10)
    model = _make(pk, "ok", xyz[:n], val[:n])
    pts = (np.linspace(0.0, 1000.0, 5), np.linspace(0.0, 1000.0, 4))
    model.execute("grid", *pts)
    h = model._kb_handle
    _add(model, xyz[n:n + 5], val[n:n + 5])
    _add(model, xyz[n + 5:], val[n + 5:])                # a chain: the extended problem grows again
    assert h.calls.count("append_data") == 2
    model.execute("grid", *pts)
    model.leave_one_out()
    assert h.calls.count("set_problem") == 1 and h.problem["X"].shape[0] == n + 10
    model.execute("grid", *pts, dtype="float32")         # another dtype misses, as it does today
    assert h.calls.count("set_problem") == 2
    model.execute("grid", *pts)
    assert h.calls.count("set_problem") == 3
    model.execute("grid", *pts, values=np.ones(n + 10))  # value fields miss
    assert h.calls.count("set_problem") == 4
    model.execute("grid", *pts)
    _add(model, xyz[:2] + 1.0, val[:2])
    model.update_variogram_model("exponential", [2.0, 300.0, 0.05])
    model.execute("grid", *pts)                          # a new variogram refactors
    assert h.calls.count("set_problem") == 6


def test_singular_append_falls_back_to_the_new_objects_error(pk):
    """A duplicate station with nugget 0: the extension is singular, the handle holds nothing, and the next execute()
    raises LinAlgError exactly as the new object does."""
    xyz, val, n = _split("ok", n=20, m=1)
    model = _make(pk, "ok", xyz[:n], val[:n], variogram_parameters=[1.0, 300.0, 0.0])
    pts = (np.linspace(0.0, 1000.0, 5), np.linspace(0.0, 1000.0, 4))
    model.execute("grid", *pts)
    _add(model, xyz[:1], val[:1] + 1.0)
    assert _appended(model) and model._kb_key is None
    ref = _make(pk, "ok", np.vstack([xyz[:n], xyz[:1]]), np.concatenate([val[:n], val[:1] + 1.0]),
                variogram_parameters=[1.0, 300.0, 0.0])
    with pytest.raises(np.linalg.LinAlgError):
        ref.execute("grid", *pts)
    with pytest.raises(np.linalg.LinAlgError):
        model.execute("grid", *pts)
