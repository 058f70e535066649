"""GPU tests of leave_group_out(): every station kriged from the stations outside its group (kb200_lgo, kb200_knn_lgo).

The global path is compared, station by station, with brute-force reduced solves in extended precision
(tests/lgo_emulator.py: brute_force_lgo) on problems of 255, 256, 257 and 513 stations, which cross the 64-row tiles of
the Gram kernel, for the four classes, every drift kind, anisotropy, geographic coordinates, a custom callable, both
exact_values and coincident stations; with random folds, spatial blocks, groups on both sides of the shared-memory
threshold (one of N/2 stations through the Cholesky route) and the Gauss-Jordan fallback; and at full size (config 2,
N = 5000) on eight stations. G itself is checked against scipy's inverse. The moving window is compared with the
oracle's moving window on each reduced data set. The bit invariants and the device refusals are pinned.
Bounds: max|out - ref| / max|ref| <= 1e-8."""
import numpy as np
import pytest
import scipy.linalg
from scipy.spatial.distance import cdist

import cases
from cv_emulator import brute_force_lgo, _refined_solve_many
from oracle import krige_oracle as ko
from test_loo_gpu import EXP, GLOBAL, _build, _obj, _reference_inputs, _stations

pytestmark = pytest.mark.gpu

LGO_TOL = 1e-8
T = 128                 # LGO_SMALL
WORST = {}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


def _judge(label, out, ref, tol=LGO_TOL):
    err = max(np.abs(out[0] - ref[0]).max() / np.abs(ref[0]).max(), np.abs(out[1] - ref[1]).max() / np.abs(ref[1]).max())
    WORST[label] = err
    print("lgo %s: max rel err %.3e" % (label, err))
    assert err <= tol, (label, err)


def kfold(n, k, seed):
    return np.random.default_rng(seed).permutation(np.arange(n) % k)


def blocks(X, nb):
    lo, hi = X[:, :2].min(0), X[:, :2].max(0)
    c = np.minimum((nb * (X[:, :2] - lo) / np.maximum(hi - lo, 1e-300)).astype(int), nb - 1)
    return c[:, 0] * nb + c[:, 1]


def mixed(n, seed):
    """Groups of 1, 2, T - 1, T and T + 1 stations, the rest in groups of 7 (labels shuffled over the stations)."""
    sizes = [1, 2, T - 1, T, T + 1]
    lab = np.concatenate([np.full(s, g) for g, s in enumerate(sizes)])
    rest = n - lab.size
    lab = np.concatenate([lab, len(sizes) + np.arange(rest) // 7])
    return np.random.default_rng(seed).permutation(lab)


def half(n, seed):
    """One group of N/2 stations (the Cholesky route) and five folds over the rest."""
    lab = np.concatenate([np.zeros(n // 2, int), 1 + np.arange(n - n // 2) % 5])
    return np.random.default_rng(seed).permutation(lab)


def _global_ref(obj, val, groups):
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    return brute_force_lgo(P, val, fn, m, exact, groups, cols, geo=geo, refined=not geo)


CASES = [("ok2d_n256", "kfold5"), ("ok2d_n512_sph_aniso_nonexact", "blocks"), ("ok2d_n257_linear", "kfold5"),
         ("uk2d_n300_rl_spec_func", "blocks"), ("uk2d_n257_pointlog_extz", "kfold5"), ("ok3d_n256_gauss_aniso", "blocks"),
         ("uk3d_n300_rl", "kfold5"), ("geo_ok_n256", "kfold5"), ("custom_ok_n256", "blocks"), ("dups_ok_n256", "kfold5"),
         ("dups_uk_n512", "mixed"), ("dups_ok_n256_nonexact", "kfold5"), ("ok2d_n512_sph_aniso_nonexact", "mixed"),
         ("ok2d_n256", "half")]


def _groups(kind, X, n):
    if kind == "kfold5":
        return kfold(n, 5, n)
    if kind == "blocks":
        return blocks(X, 4)
    if kind == "mixed":
        return mixed(n, n)
    return half(n, n)


@pytest.mark.parametrize("name,layout", CASES, ids=["%s-%s" % c for c in CASES])
def test_global_against_brute_force(pk, name, layout):
    obj, val = _build(pk, name)
    x, y, z, _, _, _ = obj._data_arrays()
    X = np.column_stack([x, y])
    groups = _groups(layout, X, X.shape[0])
    zz, ss = obj.leave_group_out(groups)
    _judge("%s-%s" % (name, layout), (zz, ss), _global_ref(obj, val, groups))


@pytest.mark.parametrize("n", [255, 256, 257, 513])
def test_tile_edges_and_gram_matrix(pk, n):
    """n = 255 .. 513 around the 64-row tiles of the Gram kernel: results against brute force, and G (debug tap 4)
    against scipy's inverse of the shifted covariance matrix."""
    X, val = _stations(50 + n, n, 2)
    obj = pk.UniversalKriging(X[:, 0], X[:, 1], val, drift_terms=["regional_linear"], **EXP)
    groups = blocks(X, 3)
    zz, ss = obj.leave_group_out(groups)
    _judge("uk_n%d_blocks" % n, (zz, ss), _global_ref(obj, val, groups))
    h = obj._kb_handle
    npad = (n + 255) // 256 * 256                                        # n_pad = ld: multiples of KB_BM = 256
    G = h.debug_fetch(4, npad * npad).reshape(npad, npad)[:n, :n]
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    c0 = h.debug_fetch(3, 10 ** 6)[-1]
    Gam = ko.variogram(fn, m, cdist(P, P))
    np.fill_diagonal(Gam, 0.0)
    ref = np.tril(scipy.linalg.inv(c0 - Gam))
    err = np.abs(np.tril(G) - ref).max() / np.abs(ref).max()
    WORST["gram_n%d" % n] = err
    assert err < 1e-10, err


def test_gauss_jordan_path(pk):
    """Hole-effect on dense scatter: C is indefinite (gform 1), G is the Gauss-Jordan inverse; small and large groups
    (the large one through the blocked Gauss-Jordan kernels)."""
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 25, (300, 2))
    val = rng.normal(size=300)
    obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, variogram_model="hole-effect", variogram_parameters=[1.0, 3.0, 0.0])
    for layout, groups in (("kfold5", kfold(300, 5, 1)), ("half", half(300, 2))):
        zz, ss = obj.leave_group_out(groups)
        _judge("gform1_%s" % layout, (zz, ss), _global_ref(obj, val, groups))


def test_full_size_config2(pk):
    """Config 2 (N = 5000) after a float64 execute(): five folds without a new factorisation, eight stations against
    brute-force solves of the reduced ~4000-station problems."""
    X, val = cases.synth_data(1002, 5000, 2)
    obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **EXP)
    obj.execute("points", X[:3, 0] + 0.5, X[:3, 1])
    h = obj._kb_handle
    h.reset_counters()
    groups = kfold(5000, 5, 7)
    zz, ss = obj.leave_group_out(groups)
    assert h.timings()["cholesky_ms"] == 0.0
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    idx = np.array([0, 1, 255, 256, 2047, 4095, 4998, 4999])
    zr, sr = np.zeros(idx.size), np.zeros(idx.size)
    for g in np.unique(groups[idx]):
        sel = idx[groups[idx] == g]
        keep = groups != g
        a = ko.kriging_matrix(P[keep], fn, m)
        z_, s_ = _refined_solve_many(a, P[keep], P[sel], val[keep], fn, m, exact, ())
        zr[groups[idx] == g], sr[groups[idx] == g] = z_, s_
    _judge("cfg2_n5000_5fold_8_stations", (zz[idx], ss[idx]), (zr, sr))


KNN = [("2d", 2), ("2d", 10), ("2d", 64), ("2d", 129), ("3d", 10), ("3d", 64), ("geo", 10), ("geo", 64),
       ("dups", 10), ("dups", 129)]


@pytest.mark.parametrize("kind,k", KNN, ids=["%s_k%d" % c for c in KNN])
def test_moving_window_against_oracle(pk, kind, k):
    n = 400
    if kind == "geo":
        rng = np.random.default_rng(23)
        X = np.column_stack([rng.uniform(-60, 60, n), rng.uniform(-45, 45, n)])
        val = 5 + np.sin(X[:, 0] / 20) + rng.normal(size=n) * 0.3
        obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, variogram_model="exponential",
                                 variogram_parameters=[1.0, 40.0, 0.05], coordinates_type="geographic")
    else:
        X, val = _stations(41, n, 3 if kind == "3d" else 2, dups=kind == "dups")
        obj = _obj(pk, "OrdinaryKriging3D" if kind == "3d" else "OrdinaryKriging", X, val, **EXP)
    for layout, groups in (("blocks", blocks(X, 3)), ("kfold", kfold(n, 4, k))):
        zz, ss = obj.leave_group_out(groups, n_closest_points=k)
        P, cols, fn, m, exact, geo = _reference_inputs(obj)
        ref = brute_force_lgo(P, val, fn, m, exact, groups, k=k, geo=geo, index_ties=kind == "dups")
        _judge("knn_%s_k%d_%s" % (kind, k, layout), (zz, ss), ref)


def test_bit_invariants(pk):
    """Field v equals a single-field call and does not depend on V or its position; sigma^2 is the same bits for any V;
    relabelled groups and a repeat give the same bits; singleton groups give leave_one_out()'s bits; execute() and
    leave_one_out() give the same bits before and after a leave_group_out()."""
    X, val = _stations(5, 700, 2, dups=True)
    F = 40.0 + 10.0 * np.random.default_rng(8).standard_normal((700, 64))
    groups = mixed(700, 3)
    relabel = np.array(["g%03d" % (997 - 3 * g) for g in groups])
    g = [np.linspace(50.0, 950.0, 7), np.linspace(80.0, 900.0, 5)]
    for kw in ({}, dict(n_closest_points=20)):
        uk = not kw
        mk = (lambda z: pk.UniversalKriging(X[:, 0], X[:, 1], z, drift_terms=["regional_linear"], **EXP)) if uk \
            else (lambda z: pk.OrdinaryKriging(X[:, 0], X[:, 1], z, **EXP))
        obj = mk(val)
        e0 = obj.execute("grid", *g, **kw)
        l0 = obj.leave_one_out(**kw)
        z64, s64 = obj.leave_group_out(groups, values=F, **kw)
        z3, s3 = obj.leave_group_out(groups, values=F[:, [5, 0, 63]], **kw)
        z1, s1 = obj.leave_group_out(groups, values=F[:, 63], **kw)
        np.testing.assert_array_equal(z3, z64[[5, 0, 63]])
        np.testing.assert_array_equal(z1, z64[63])
        for s in (s3, s1):
            np.testing.assert_array_equal(s, s64)
        zs, ss = mk(F[:, 0]).leave_group_out(groups, **kw)
        np.testing.assert_array_equal(zs, z64[0])
        np.testing.assert_array_equal(ss, s64)
        zr, sr = obj.leave_group_out(relabel, values=F, **kw)
        np.testing.assert_array_equal(zr, z64)
        np.testing.assert_array_equal(sr, s64)
        zb, sb = obj.leave_group_out(groups, values=F, **kw)
        np.testing.assert_array_equal(zb, z64)
        np.testing.assert_array_equal(sb, s64)
        zo, so = obj.leave_group_out(np.arange(700)[::-1], **kw)
        np.testing.assert_array_equal(zo, l0[0])
        np.testing.assert_array_equal(so, l0[1])
        e1 = obj.execute("grid", *g, **kw)
        l1 = obj.leave_one_out(**kw)
        for a, b in zip(e0 + l0, e1 + l1):
            np.testing.assert_array_equal(np.asarray(a), np.asarray(b))


def test_refusals_on_the_device(pk):
    from pykrige_b200 import _cabi
    X, val = _stations(9, 60, 2)
    groups = np.arange(60) % 4
    with pytest.raises(NotImplementedError):
        pk.OrdinaryKriging(X[:, 0], X[:, 1], val, pseudo_inv=True, **EXP).leave_group_out(groups)
    ok = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **EXP)
    for bad in (np.zeros(60), np.arange(59), np.zeros((60, 2))):
        with pytest.raises(ValueError):
            ok.leave_group_out(bad)
    with pytest.raises(ValueError, match="group 0"):
        ok.leave_group_out(groups, n_closest_points=46)
    rng = np.random.default_rng(9)
    t = rng.uniform(0, 100, 20)
    Xl = np.vstack([rng.uniform(0, 100, (6, 2)), np.column_stack([t, 0.5 * t + 3.0])])
    gl = np.r_[np.full(6, "edge"), np.array(["a", "b", "c"])[np.arange(20) % 3]]
    uk = pk.UniversalKriging(Xl[:, 0], Xl[:, 1], rng.normal(size=26), variogram_model="exponential",
                             variogram_parameters=[1.0, 40.0, 0.1], drift_terms=["regional_linear"])
    with pytest.raises(np.linalg.LinAlgError, match="group 'edge'"):
        uk.leave_group_out(gl)
    Xd = X.copy()
    Xd[:34] = Xd[0]                                     # 34 coincident stations; station 0 alone in group 9
    okd = pk.OrdinaryKriging(Xd[:, 0], Xd[:, 1], val, **EXP)
    gd = np.arange(60) % 4
    gd[0] = 9
    with pytest.raises(NotImplementedError, match="station 0"):
        okd.leave_group_out(gd)
    h = _cabi.Handle()
    args = (2, 0, X[:, 0], X[:, 1], None, val, [500.0, 500.0], np.eye(2), 3, [0.95, 300.0, 0.05], True, 1e-10)
    h.set_problem(*args)
    for g, ng in ((np.zeros(60), 1), (groups, 5), (groups - 1, 4)):
        with pytest.raises(ValueError):
            h.lgo(g, ng, 60)
    z, ss = h.lgo(groups, 4, 60)
    assert z.shape == (60,) and np.all(ss > 0)
    h.describe_problem(*args)
    h.blob_commit()
    with pytest.raises(_cabi.KrigeB200Error, match="blob_commit"):
        h.lgo(groups, 4, 60)
    h.close()
