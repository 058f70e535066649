"""GPU tests of execute(values=...): V value fields through one factorisation and one solve pass.

Every field is compared with the extended-precision reference (oracle.krige_oracle.exec_vector_refined) at the fp64
tolerance of tests/test_solve_boundaries_gpu.py, with the dual rows n + K + 1 + V on both sides of the 16-row m-tiles and
256-row blocks (including field rows that spill into one more row block), and the two invariants are pinned bit for
bit: field v does not depend on V or on its position in the call (which makes chunking invisible), and a fields call
equals the single-field execute() of an object built with z = values[:, v]."""
import numpy as np
import pytest

import cases
from oracle import krige_oracle as ko
from test_solve_boundaries_gpu import TOL, TOL_GJ, Problem, _judge, _set_tile

pytestmark = pytest.mark.gpu

CAP = 64                                   # KB200_MAX_FIELDS
F64 = TOL["float64"]


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


def _fields(n, V, seed=0):
    rng = np.random.default_rng(seed)
    return 40.0 + 10.0 * rng.standard_normal((n, V))


def _refs(prob, F, idx=None, bd_ok=True):
    """refined reference of every field (z per field, sigma^2 of the first)."""
    out = []
    Q = prob.Q if idx is None else prob.Q[idx]
    for v in range(F.shape[1]):
        bd = prob._bd(Q, prob.P) if prob._bd else None
        out.append(ko.exec_vector_refined(prob.a, prob.P, Q, F[:, v], prob.mname, prob.m, prob.exact,
                                          prob._dcols(Q) if prob._dcols else (), bd=bd))
    return out


def _run(prob, F, idx=None):
    p = prob.pts if idx is None else prob.pts[idx]
    z, ss = prob.model.execute("points", *[p[:, c] for c in range(p.shape[1])], backend="cuda", values=F)
    return np.asarray(z), np.asarray(ss)


def _check(prob, F, tol, label, monkeypatch, tiles=(16, 32, 64), idx=None):
    refs = _refs(prob, F, idx)
    failures = []
    for tile in tiles:
        _set_tile(monkeypatch, tile)
        z, ss = _run(prob, F, idx)
        assert z.shape == (F.shape[1], ss.shape[0])
        for v, ref in enumerate(refs):
            _judge("%s/t%s" % (label, tile), tol, prob.what + " V=%d v=%d" % (F.shape[1], v), ref[2], (z[v], ss),
                   ref[:2], failures)
    _set_tile(monkeypatch, None)
    assert not failures, "\n".join(failures)


# (n, na) with na = K + 2 of the single-field problem: n + K + 1 + V crosses 16-row m-tiles and the 256-row block for
# the V below (e.g. n = 240, K = 0: the dual rows end at 241 + V, past 256 from V = 16 on; n = 254: from V = 2 on)
SIZES = [(240, 2), (254, 2), (239, 4), (224, 17), (250, 17), (767, 2)]
VS = [1, 2, 6, 7, 17, CAP]


@pytest.mark.parametrize("n,na", SIZES, ids=["n%d_na%d" % s for s in SIZES])
def test_fields_against_refined_reference(pk, monkeypatch, n, na):
    prob = Problem(pk, n, na, "2d", "exponential", m_scatter=60)
    for V in VS:
        _check(prob, _fields(n, V, seed=V), F64, "fields", monkeypatch, tiles=(16, 32, 64) if V in (7, CAP) else (64,))


KINDS = [(255, 2, "3d", "spherical"), (255, 2, "geo", "exponential"), (257, 4, "2d", "linear"),
         (129, 2, "2d", "exponential")]


@pytest.mark.parametrize("n,na,kind,model", KINDS, ids=["n%d_na%d_%s" % k[:3] for k in KINDS])
def test_fields_3d_geographic_anisotropic(pk, monkeypatch, n, na, kind, model):
    """3-D, geographic, anisotropic (n = 129, 257) and exact_values=False problems; the scattered points include up to
    16 exact hits of data points."""
    for exact in (True, False):
        prob = Problem(pk, n, na, kind, model, m_scatter=60, exact=exact)
        _check(prob, _fields(n, 6, seed=n), F64, "fields-" + kind, monkeypatch, tiles=(32, 64))


def test_exact_hits_return_the_field_values(pk):
    prob = Problem(pk, 200, 2, "2d", "exponential", m_scatter=20, params=[1.0, 300.0, 0.0])
    F = _fields(200, 5, seed=3)
    hits = prob.data[:16]
    z, ss = prob.model.execute("points", hits[:, 0], hits[:, 1], values=F)
    np.testing.assert_allclose(z, F[:16].T, rtol=1e-8, atol=1e-8 * np.abs(F).max())
    assert np.all(np.abs(ss) < 1e-8)


def test_device_and_specified_drifts(pk):
    """UK with point_log and external_Z (evaluated in the solve kernel) and a specified drift: every field equals the
    single-field execute() of an object with z = that field, bit for bit."""
    xyz, val = cases.synth_data(41, 300, 2)
    pts = cases.synth_points(41, 70, 2, xyz)
    ex, ey = np.linspace(-10.0, 1010.0, 40), np.linspace(-10.0, 1010.0, 30)
    ez = np.sin(ex[None, :] / 200.0) + np.cos(ey[:, None] / 300.0)
    spec = np.cos(xyz[:, 0] / 300.0)
    spec_p = np.cos(pts[:, 0] / 300.0)
    F = _fields(300, 9, seed=41)

    def make(z):
        return pk.UniversalKriging(
            xyz[:, 0], xyz[:, 1], z, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05],
            drift_terms=["regional_linear", "point_log", "external_Z", "specified"],
            point_drift=[[500.0, 500.0, 0.4], [200.0, 700.0, 0.3]], external_drift=ez, external_drift_x=ex,
            external_drift_y=ey, specified_drift=[spec])
    z, ss = make(val).execute("points", pts[:, 0], pts[:, 1], specified_drift_arrays=[spec_p], values=F)
    for v in (0, 4, 8):
        zv, sv = make(F[:, v]).execute("points", pts[:, 0], pts[:, 1], specified_drift_arrays=[spec_p])
        np.testing.assert_array_equal(z[v], zv)
        np.testing.assert_array_equal(ss, sv)


def test_several_tiles_per_cta(pk, monkeypatch):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 2 * sms * 64 + 37
    prob = Problem(pk, 250, 4, "2d", "spherical", m_scatter=M - 16, seed=777)
    rng = np.random.default_rng(1)
    idx = np.union1d(rng.choice(M - 64, 200, replace=False), np.arange(M - 64, M))
    F = _fields(250, 7, seed=5)
    refs = _refs(prob, F, idx)
    failures = []
    for tile in (16, 32, 64):
        _set_tile(monkeypatch, tile)
        z, ss = _run(prob, F)
        for v, ref in enumerate(refs):
            _judge("multi/t%d" % tile, F64, prob.what + " v=%d" % v, ref[2], (z[v][idx], ss[idx]), ref[:2], failures)
    _set_tile(monkeypatch, None)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("n,na", [(255, 2), (256, 4)])
def test_general_inverse_path(pk, monkeypatch, n, na):
    """gform 1 (hole-effect: Gauss-Jordan inverse + quadratic form) with fields."""
    prob = Problem(pk, n, na, "2d", "hole-effect", params=[1.0, 300.0, 0.02], m_scatter=60)
    _check(prob, _fields(n, 7, seed=n), TOL_GJ, "gform1-fields", monkeypatch)


@pytest.mark.parametrize("k", [2, 8, 64, 128, 130])
def test_moving_window(pk, k):
    """Every field against the oracle's moving window (scipy solve per point), and bit for bit against the
    single-field moving window; V = 9 needs two augmented tile rows."""
    xyz, val = cases.synth_data(60 + k, 700, 2)
    pts = cases.synth_points(60 + k, 90, 2, xyz)
    F = _fields(700, 9, seed=k)
    kw = dict(variogram_model="spherical", variogram_parameters=[1.0, 250.0, 0.05])
    ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, **kw)
    z, ss = ok.execute("points", pts[:, 0], pts[:, 1], n_closest_points=k, values=F)
    m = ko.stored_parameters("spherical", kw["variogram_parameters"])
    for v in range(9):
        zr, sr = ko.exec_moving_window(xyz, pts, F[:, v], "spherical", m, k, True)
        np.testing.assert_allclose(z[v], zr, rtol=1e-9, atol=1e-9 * np.abs(zr).max())
        np.testing.assert_allclose(ss, sr, rtol=1e-9, atol=1e-9 * np.abs(sr).max())
    for v in (0, 8):
        zv, sv = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], F[:, v], **kw).execute(
            "points", pts[:, 0], pts[:, 1], n_closest_points=k)
        np.testing.assert_array_equal(z[v], zv)
        np.testing.assert_array_equal(ss, sv)


def test_moving_window_lu_fallback(pk):
    """hole-effect: a local covariance block that is not positive definite sends the launch to the pivoted LU."""
    xyz, val = cases.synth_data(71, 500, 2)
    pts = cases.synth_points(71, 60, 2, xyz)
    F = _fields(500, 8, seed=71)
    kw = dict(variogram_model="hole-effect", variogram_parameters=[1.0, 60.0, 0.0])
    z, ss = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, **kw).execute("points", pts[:, 0], pts[:, 1],
                                                                         n_closest_points=40, values=F)
    m = ko.stored_parameters("hole-effect", kw["variogram_parameters"])
    for v in range(8):
        zr, sr = ko.exec_moving_window(xyz, pts, F[:, v], "hole-effect", m, 40, True)
        np.testing.assert_allclose(z[v], zr, rtol=1e-8, atol=1e-8 * np.abs(zr).max())
    zv, sv = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], F[:, 3], **kw).execute("points", pts[:, 0], pts[:, 1],
                                                                              n_closest_points=40)
    np.testing.assert_array_equal(z[3], zv)
    np.testing.assert_array_equal(ss, sv)


def test_invariants_and_chunking(pk):
    """Field v is bit-identical whatever V and its position, sigma^2 is bit-identical for every V, a fields call equals
    the single-field execute() bit for bit, and V = 2 * cap + 3 runs as three chunks with the same bits."""
    n = 250
    prob = Problem(pk, n, 4, "2d", "exponential", m_scatter=150)
    Fbig = _fields(n, 2 * CAP + 3, seed=11)
    p = prob.pts
    zb, sb = prob.model.execute("grid", np.linspace(0, 1000, 37), np.linspace(0, 1000, 23), values=Fbig)
    z0, s0 = prob.model.execute("grid", np.linspace(0, 1000, 37), np.linspace(0, 1000, 23))
    np.testing.assert_array_equal(sb, s0)
    for V, first in ((1, 5), (2, 0), (7, 3), (17, 100), (CAP, 60)):
        z, s = prob.model.execute("grid", np.linspace(0, 1000, 37), np.linspace(0, 1000, 23),
                                  values=Fbig[:, first:first + V])
        np.testing.assert_array_equal(z, zb[first:first + V])
        np.testing.assert_array_equal(s, s0)
    zp, sp = prob.model.execute("points", p[:, 0], p[:, 1], values=Fbig[:, [4, 70]])
    for j, v in enumerate((4, 70)):
        kw = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05],
                  drift_terms=["regional_linear"])
        single = pk.UniversalKriging(prob.data[:, 0], prob.data[:, 1], Fbig[:, v], **kw)
        zs, ss = single.execute("points", p[:, 0], p[:, 1])
        np.testing.assert_array_equal(zp[j], zs)
        np.testing.assert_array_equal(sp, ss)


def test_refusals_through_the_classes(pk):
    xyz, val = cases.synth_data(3, 100, 2)
    ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential",
                            variogram_parameters=[1.0, 300.0, 0.05])
    F = _fields(100, 3)
    p = (np.array([10.0, 20.0]), np.array([30.0, 40.0]))
    for dtype in ("float32", "float64x"):
        with pytest.raises(NotImplementedError):
            ok.execute("points", *p, dtype=dtype, values=F)
    with pytest.raises(ValueError):
        ok.execute("points", *p, values=F.T)
    pinv = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential",
                              variogram_parameters=[1.0, 300.0, 0.05], pseudo_inv=True)
    with pytest.raises(NotImplementedError):
        pinv.execute("points", *p, values=F)
    from pykrige_b200 import _cabi
    h = _cabi.Handle()
    with pytest.raises(ValueError):
        h.set_values(np.zeros((CAP + 1, 10)))
    h.set_values(np.ones((2, 10)))
    with pytest.raises(NotImplementedError):
        h.describe_problem(2, 0, np.arange(10.0), np.arange(10.0) ** 2, None, np.ones(10), [0, 0], np.eye(2), 3,
                           [1.0, 300.0, 0.05], True, 1e-10)
    z, ss = ok.execute("points", *p)        # the object's own problem is untouched
    assert z.shape == (2,)
