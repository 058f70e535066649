"""CPU tests of leave_group_out() on the host side.

`_cabi.Handle` is replaced by tests/lgo_emulator.py, which implements kb200_lgo / kb200_knn_lgo by brute force with the
oracle, so what is checked here is the product code above the C ABI: the mapping of the user's labels to dense group
indices and back into error messages, argument checks and their exception types, the shapes with 1-D and 2-D `values`,
chunks of 64 fields, that the problem is shared with execute(), and that singleton groups take the leave-one-out route.
The device kernels are tests/test_lgo_gpu.py."""
import inspect

import numpy as np
import pytest
from numpy.testing import assert_array_equal

import cases
from cv_emulator import CvEmulatedHandle as LgoEmulatedHandle

EXP = [1.0, 300.0, 0.05]
KINDS = ["ok", "uk", "ok3d", "uk3d"]


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", LgoEmulatedHandle)
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


def test_emulator_methods_have_the_handle_signatures():
    from pykrige_b200 import _cabi
    for name in ("lgo", "knn_lgo"):
        assert inspect.signature(getattr(LgoEmulatedHandle, name)) == inspect.signature(getattr(_cabi.Handle, name))


def test_public_signatures(pk):
    for cls in (pk.OrdinaryKriging, pk.OrdinaryKriging3D):
        assert list(inspect.signature(cls.leave_group_out).parameters) == ["self", "groups", "n_closest_points",
                                                                          "values", "backend"]
    for cls in (pk.UniversalKriging, pk.UniversalKriging3D):
        assert list(inspect.signature(cls.leave_group_out).parameters) == ["self", "groups", "values", "backend"]


@pytest.mark.parametrize("kind", KINDS)
def test_shapes_and_fields(pk, kind):
    """zvalues (N,) or (V, N), sigmasq (N,); field v equals leave_group_out() of an object built with z = values[:, v]."""
    xyz, val = _data(kind)
    n = xyz.shape[0]
    groups = np.arange(n) % 4
    model = _make(pk, kind, xyz, val)
    z0, s0 = model.leave_group_out(groups)
    assert z0.shape == (n,) and s0.shape == (n,)
    F = np.random.default_rng(1).normal(size=(n, 3))
    z, s = model.leave_group_out(groups, values=F)
    assert z.shape == (3, n) and s.shape == (n,)
    assert_array_equal(s, s0)
    for v in range(3):
        zv, sv = _make(pk, kind, xyz, F[:, v]).leave_group_out(groups)
        assert_array_equal(z[v], zv)
        assert_array_equal(s, sv)
    z1, _ = model.leave_group_out(groups, values=F[:, 2])
    assert z1.shape == (n,)
    assert_array_equal(z1, z[2])
    if kind in ("ok", "ok3d"):
        zk, sk = model.leave_group_out(groups, n_closest_points=5, values=F)
        assert zk.shape == (3, n) and sk.shape == (n,)


def test_label_mapping(pk):
    """Any labels np.unique sorts: strings, negative and sparse integers give the same result as dense indices."""
    xyz, val = _data("ok")
    n = xyz.shape[0]
    dense = np.arange(n) % 3
    model = _make(pk, "ok", xyz, val)
    ref = model.leave_group_out(dense)
    for labels in (np.array(["c", "a", "b"])[dense], np.array([-7, 1000, 3])[dense], (dense * 10 ** 9).tolist()):
        got = model.leave_group_out(labels)
        assert_array_equal(got[0], ref[0])
        assert_array_equal(got[1], ref[1])
    handle = model._kb_handle
    model.leave_group_out(np.array(["c", "a", "b"])[dense])
    assert handle.calls[-1] == "lgo"


def test_65_fields_run_in_two_chunks(pk):
    xyz, val = _data("ok", n=12)
    groups = np.arange(12) % 3
    model = _make(pk, "ok", xyz, val)
    F = np.random.default_rng(2).normal(size=(12, 65))
    z, _ = model.leave_group_out(groups, values=F)
    assert z.shape == (65, 12)
    assert model._kb_handle.calls.count("set_problem") == 2
    assert_array_equal(z[64], _make(pk, "ok", xyz, F[:, 64]).leave_group_out(groups)[0])


def test_problem_is_shared_with_execute(pk):
    """execute -> leave_group_out -> leave_one_out -> execute factorises once; the moving window shares its set-up."""
    xyz, val = _data("uk")
    model = _make(pk, "uk", xyz, val)
    g = [np.linspace(50.0, 950.0, 4), np.linspace(80.0, 900.0, 3)]
    a = model.execute("grid", *g)
    model.leave_group_out(np.arange(24) % 4)
    model.leave_one_out()
    b = model.execute("grid", *g)
    assert model._kb_handle.calls.count("set_problem") == 1
    assert_array_equal(a[0], b[0])
    ok = _make(pk, "ok", *_data("ok"))
    ok.leave_group_out(np.arange(24) % 4, n_closest_points=4)
    ok.execute("grid", *g, n_closest_points=4)
    ok.leave_one_out(n_closest_points=6)
    assert ok._kb_handle.calls.count("set_problem_knn") == 1


def test_singleton_groups_take_the_leave_one_out_route(pk):
    xyz, val = _data("uk")
    model = _make(pk, "uk", xyz, val)
    z, s = model.leave_group_out(["s%d" % i for i in range(24)])
    assert model._kb_handle.calls[-2:] == ["lgo", "loo"]
    zl, sl = model.leave_one_out()
    assert_array_equal(z, zl)
    assert_array_equal(s, sl)


def test_refusals(pk):
    xyz, val = _data("ok")
    n = xyz.shape[0]
    groups = np.arange(n) % 4
    ok = _make(pk, "ok", xyz, val)
    for bad in (np.zeros(n + 1), np.zeros((n, 2)), np.arange(n - 1)):
        with pytest.raises(ValueError, match="groups must have shape"):
            ok.leave_group_out(bad)
    with pytest.raises(ValueError, match="at least two distinct groups"):
        ok.leave_group_out(np.full(n, "one"))
    big = np.where(np.arange(n) < 14, "big", "small")
    for k in (1, n - 13):
        with pytest.raises(ValueError, match="group 'big'"):
            ok.leave_group_out(big, n_closest_points=k)
    assert ok.leave_group_out(big, n_closest_points=n - 14)[0].shape == (n,)
    with pytest.raises(ValueError, match="backend"):
        ok.leave_group_out(groups, backend="vectorized")
    for bad in (np.zeros((n + 1, 2)), np.full(n, np.nan)):
        with pytest.raises(ValueError):
            ok.leave_group_out(groups, values=bad)
    pinv = _make(pk, "ok", xyz, val, pseudo_inv=True)
    with pytest.raises(NotImplementedError):
        pinv.leave_group_out(groups)
    with pytest.warns(UserWarning, match="pseudo_inv is ignored"):
        pinv.leave_group_out(groups, n_closest_points=5)
    # a drift left undetermined: every station outside group 'edge' on one line
    rng = np.random.default_rng(9)
    t = rng.uniform(0, 100, 20)
    X = np.vstack([rng.uniform(0, 100, (6, 2)), np.column_stack([t, 0.5 * t + 3.0])])
    gl = np.r_[np.full(6, "edge"), np.array(["a", "b", "c"])[np.arange(20) % 3]]
    uk = pk.UniversalKriging(X[:, 0], X[:, 1], rng.normal(size=26), variogram_model="exponential",
                             variogram_parameters=[1.0, 40.0, 0.1], drift_terms=["regional_linear"])
    with pytest.raises(np.linalg.LinAlgError, match="group 'edge'"):
        uk.leave_group_out(gl)
    # more than 32 stations of other groups within eps of one station
    Xd = xyz.copy()
    Xd = np.vstack([Xd, np.repeat(Xd[:1], 40, axis=0)])
    gd = np.r_[np.arange(n) % 4, np.arange(40) % 3 + 1]
    okd = _make(pk, "ok", Xd, np.r_[val, np.zeros(40)])
    with pytest.raises(NotImplementedError, match="within eps"):
        okd.leave_group_out(gd)


def test_blob_problem_is_refused():
    from pykrige_b200 import _cabi
    xyz, val = _data("ok", n=10)
    args = (2, 0, xyz[:, 0], xyz[:, 1], None, val, [500.0, 500.0], np.eye(2), 3, [0.95, 300.0, 0.05], True, 1e-10)
    src, dst = LgoEmulatedHandle(), LgoEmulatedHandle()
    src.set_problem(*args)
    dst.describe_problem(*args)
    dst.blob_t.copy_(src.blob_t)
    dst.blob_commit()
    groups = np.arange(10) % 2
    with pytest.raises(_cabi.KrigeB200Error, match="blob_commit"):
        dst.lgo(groups, 2, 10)
    assert src.lgo(groups, 2, 10)[0].shape == (10,)
    for g, ng in ((np.zeros(10, int), 1), (groups, 3), (groups - 1, 2)):
        with pytest.raises(ValueError):
            src.lgo(g, ng, 10)
