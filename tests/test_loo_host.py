"""CPU tests of leave_one_out() on the host side.

`_cabi.Handle` is replaced by tests/loo_emulator.py, which implements kb200_loo / kb200_knn_loo by brute force with the
oracle, so what is checked here is the product code above the C ABI: argument checks and their exception types, the
shapes with 1-D and 2-D `values`, chunks of 64 fields, and that the problem cache is shared with execute(). The device
kernels are tests/test_loo_gpu.py."""
import inspect

import numpy as np
import pytest
from numpy.testing import assert_array_equal

import cases
from cv_emulator import CvEmulatedHandle as LooEmulatedHandle

EXP = [1.0, 300.0, 0.05]


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", LooEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def _make(pk, kind, xyz, z, **kw):
    kw = dict(variogram_model="exponential", variogram_parameters=EXP, **kw)
    if kind == "ok":
        return pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], z, **kw)
    if kind == "uk":
        return pk.UniversalKriging(xyz[:, 0], xyz[:, 1], z, drift_terms=["regional_linear"], **kw)
    if kind == "ok3d":
        return pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, **kw)
    return pk.UniversalKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], z, drift_terms=["regional_linear"], **kw)


def _data(kind, n=24, seed=5):
    return cases.synth_data(seed, n, 3 if kind.endswith("3d") else 2)


KINDS = ["ok", "uk", "ok3d", "uk3d"]


def test_emulator_methods_have_the_handle_signatures():
    from pykrige_b200 import _cabi
    for name in ("loo", "knn_loo"):
        assert inspect.signature(getattr(LooEmulatedHandle, name)) == inspect.signature(getattr(_cabi.Handle, name))


@pytest.mark.parametrize("kind", KINDS)
def test_shapes_and_fields(pk, kind):
    """zvalues (N,) or (V, N), sigmasq (N,); field v equals leave_one_out() of an object built with z = values[:, v];
    a 1-D values gives the (N,) shape; the constructor's values are untouched."""
    xyz, val = _data(kind)
    n = xyz.shape[0]
    model = _make(pk, kind, xyz, val)
    z0, s0 = model.leave_one_out()
    assert z0.shape == (n,) and s0.shape == (n,)
    F = np.random.default_rng(1).normal(size=(n, 3))
    z, s = model.leave_one_out(values=F)
    assert z.shape == (3, n) and s.shape == (n,)
    assert_array_equal(s, s0)
    for v in range(3):
        zv, sv = _make(pk, kind, xyz, F[:, v]).leave_one_out()
        assert_array_equal(z[v], zv)
        assert_array_equal(s, sv)
    z1, s1 = model.leave_one_out(values=F[:, 2])
    assert z1.shape == (n,)
    assert_array_equal(z1, z[2])
    np.testing.assert_array_equal(model._data_arrays()[3], val)
    if kind in ("ok", "ok3d"):
        zk, sk = model.leave_one_out(n_closest_points=5, values=F)
        assert zk.shape == (3, n) and sk.shape == (n,)


def test_65_fields_run_in_two_chunks(pk):
    xyz, val = _data("ok", n=12)
    model = _make(pk, "ok", xyz, val)
    F = np.random.default_rng(2).normal(size=(12, 65))
    z, s = model.leave_one_out(values=F)
    assert z.shape == (65, 12)
    assert model._kb_handle.calls.count("set_problem") == 2
    assert_array_equal(z[64], _make(pk, "ok", xyz, F[:, 64]).leave_one_out()[0])
    assert_array_equal(z[3], _make(pk, "ok", xyz, F[:, 3]).leave_one_out()[0])


def test_cache_is_shared_with_execute(pk):
    """execute -> leave_one_out -> execute factorises once; the moving window likewise shares its set-up."""
    xyz, val = _data("uk")
    model = _make(pk, "uk", xyz, val)
    g = [np.linspace(50.0, 950.0, 4), np.linspace(80.0, 900.0, 3)]
    a = model.execute("grid", *g)
    model.leave_one_out()
    b = model.execute("grid", *g)
    assert model._kb_handle.calls.count("set_problem") == 1
    assert_array_equal(a[0], b[0])
    ok = _make(pk, "ok", *_data("ok"))
    ok.leave_one_out(n_closest_points=4)
    ok.execute("grid", *g, n_closest_points=4)
    ok.leave_one_out(n_closest_points=6)
    assert ok._kb_handle.calls.count("set_problem_knn") == 1


def test_refusals(pk):
    xyz, val = _data("ok")
    n = xyz.shape[0]
    ok = _make(pk, "ok", xyz, val)
    for k in (1, 0, n, n + 3):
        with pytest.raises(ValueError, match="n_closest_points"):
            ok.leave_one_out(n_closest_points=k)
    with pytest.raises(ValueError, match="backend"):
        ok.leave_one_out(backend="vectorized")
    with pytest.raises(ValueError, match="backend"):
        _make(pk, "uk", *_data("uk")).leave_one_out(backend="C")
    for bad in (np.zeros((n + 1, 2)), np.zeros((n, 0)), np.full(n, np.nan)):
        with pytest.raises(ValueError):
            ok.leave_one_out(values=bad)
    one = pk.OrdinaryKriging([1.0], [2.0], [3.0], variogram_model="linear", variogram_parameters=[1.0, 0.0])
    with pytest.raises(ValueError, match="at least two"):
        one.leave_one_out()
    pinv = _make(pk, "ok", xyz, val, pseudo_inv=True)
    with pytest.raises(NotImplementedError):
        pinv.leave_one_out()
    with pytest.warns(UserWarning, match="pseudo_inv is ignored"):
        z, s = pinv.leave_one_out(n_closest_points=5)
    assert z.shape == (n,)
    X = np.array([[0.0, 0.0], [10.0, 1.0], [3.0, 9.0]])
    uk3 = pk.UniversalKriging(X[:, 0], X[:, 1], [1.0, 2.0, 0.5], variogram_model="exponential",
                              variogram_parameters=[1.0, 20.0, 0.1], drift_terms=["regional_linear"])
    with pytest.raises(np.linalg.LinAlgError, match="station"):
        uk3.leave_one_out()


def test_blob_problem_is_refused():
    """A problem received through kb200_blob_commit has no factor on the handle."""
    from pykrige_b200 import _cabi
    xyz, val = _data("ok", n=10)
    args = (2, 0, xyz[:, 0], xyz[:, 1], None, val, [500.0, 500.0], np.eye(2), 3, [0.95, 300.0, 0.05], True, 1e-10)
    src, dst = LooEmulatedHandle(), LooEmulatedHandle()
    src.set_problem(*args)
    dst.describe_problem(*args)
    dst.blob_t.copy_(src.blob_t)
    dst.blob_commit()
    with pytest.raises(_cabi.KrigeB200Error, match="blob_commit"):
        dst.loo(10)
    assert src.loo(10)[0].shape == (10,)
