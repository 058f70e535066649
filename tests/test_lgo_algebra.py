"""The leave-group-out formulation of DESIGN.md §5f, pinned in numpy, independent of any kernel.

From the covariance form the device holds (c0 search, rescaled drift basis, G = C^-1 = W^T W or the Gauss-Jordan
inverse, U, zeta, S^-1, phi), with P = G - U S^-1 U^T and alpha = zeta - U S^-1 phi, the stations of a group S are
    e_S = P_SS^-1 alpha_S,   zhat_S = Z_S - e_S,   sigma^2_S = diag(P_SS^-1),
plus, under exact_values, a correction from the stations of other groups within eps of a station (DESIGN.md §5f). This
file restates exactly that and compares it with brute-force reduced solves (tests/lgo_emulator.py) on the fuzz draws
with random k-fold and spatial-block groups, the geographic and duplicate draws, coincident stations inside one group
and across groups, the Gauss-Jordan variant and a drift left undetermined by one group."""
import numpy as np
import pytest
import scipy.linalg

import cases
from cv_emulator import CvEmulatedHandle as LgoEmulatedHandle, brute_force_lgo, near_pairs
from oracle import krige_oracle as ko
from test_loo_algebra import _c0, _rescale

TOL = 1e-9          # max|covariance form - brute force| / max|brute force|, z and sigma^2


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", LgoEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def covariance_form_lgo(P, fn, m, exact, drift_cols, n_rl, Zs, groups, geo=False, eps=ko.EPS):
    """Every station's leave-group-out (zhat [V, n], sigma^2 [n], gform, smallest |pivot| / scale over the groups)."""
    P = np.asarray(P, dtype=np.float64)
    n = P.shape[0]
    D = near_pairs(P, geo)
    Gam = ko.variogram(fn, m, D)
    np.fill_diagonal(Gam, 0.0)
    c0, unbounded = _c0(P, fn, m, geo)
    gform, L = 1, None
    for _ in range(5 if unbounded else 1):
        try:
            L = np.linalg.cholesky(c0 - Gam)
            gform = 0
            break
        except np.linalg.LinAlgError:
            c0 *= 2.0
    if gform:
        G = scipy.linalg.inv(_c0(P, fn, m, geo)[0] - Gam)
    else:
        W = scipy.linalg.solve_triangular(L, np.eye(n), lower=True)
        G = W.T @ W                                   # the Gram product of the lower-triangular W
    G = np.tril(G) + np.tril(G, -1).T                 # the device reads the lower triangle
    F = np.column_stack(_rescale(P, n_rl, drift_cols) + [np.ones(n)])
    Z = np.column_stack(Zs)
    U, zeta = G @ F, G @ Z
    S = F.T @ U
    Sinv = np.linalg.inv(0.5 * (S + S.T))
    usu = U @ Sinv @ U.T
    Pm = G - usu
    alpha = zeta - U @ Sinv @ (F.T @ zeta)
    zh, ss = np.zeros((Z.shape[1], n)), np.zeros(n)
    groups = np.asarray(groups)
    worst = np.inf
    for g in np.unique(groups):
        Sg = np.flatnonzero(groups == g)
        scale = np.maximum(np.abs(np.diag(G)[Sg]), np.abs(np.diag(usu)[Sg]))
        lu, piv = scipy.linalg.lu_factor(Pm[np.ix_(Sg, Sg)])
        worst = min(worst, float(np.min(np.abs(np.diag(lu)) / scale.max())))
        Q = np.linalg.inv(Pm[np.ix_(Sg, Sg)])
        e = Q @ alpha[Sg]
        zh[:, Sg] = (Z[Sg] - e).T
        ss[Sg] = np.diag(Q)
        if not exact:
            continue
        for a, i in enumerate(Sg):
            Dj = np.flatnonzero((np.abs(D[i]) <= eps) & (groups != g))
            if Dj.size == 0:
                continue
            dl = ko.variogram(fn, m, D[i, Dj])
            PjS = Pm[np.ix_(Dj, Sg)]
            zh[:, i] += dl @ (alpha[Dj] - PjS @ e)
            ss[i] += 2.0 * dl @ (PjS @ Q)[:, a] - dl @ (Pm[np.ix_(Dj, Dj)] - PjS @ Q @ PjS.T) @ dl
    return zh, ss, gform, worst


def _problem(obj):
    obj._ensure_problem("float64")
    p = obj._kb_handle.problem
    P = p["X"] if p["geo"] else p["P"]
    cols = ([P[:, c] for c in range(p["dim"])] if p["n_rl"] else []) + list(p["hd"])
    return p, P, cols


def _check(p, P, cols, groups, Zs=None, tol=TOL, min_pivot=0.0):
    """min_pivot: skip the comparison (return None) when some group's smallest pivot / scale is below it."""
    Zs = [p["values"]] if Zs is None else Zs
    zh, ss, gform, worst = covariance_form_lgo(P, p["fn"], p["m"], p["exact"], cols, p["dim"] if p["n_rl"] else 0, Zs,
                                               groups, geo=p["geo"])
    if worst < min_pivot:
        return None
    for v, Zv in enumerate(Zs):
        zr, sr = brute_force_lgo(P, Zv, p["fn"], p["m"], p["exact"], groups, cols, geo=p["geo"], refined=not p["geo"])
        assert np.abs(zh[v] - zr).max() <= tol * np.abs(zr).max(), np.abs(zh[v] - zr).max() / np.abs(zr).max()
        assert np.abs(ss - sr).max() <= tol * np.abs(sr).max(), np.abs(ss - sr).max() / np.abs(sr).max()
    return gform, worst


def kfold(n, k, seed):
    return np.random.default_rng(seed).permutation(np.arange(n) % k)


def blocks(P, nb):
    """Spatial blocks: an nb x nb grid over the bounding box of the first two coordinates."""
    lo, hi = P[:, :2].min(0), P[:, :2].max(0)
    c = np.minimum((nb * (P[:, :2] - lo) / np.maximum(hi - lo, 1e-300)).astype(int), nb - 1)
    return c[:, 0] * nb + c[:, 1]


GLOBAL_FUZZ = [t for t in range(cases.N_FUZZ) if cases.fuzz_config(t) is not None and cases.fuzz_config(t)["knn"] is None]


def test_fuzz_draws_match_brute_force(pk):
    """The global fuzz draws (all four classes, every drift kind, anisotropy, both exact_values) with 2, 5 and 10 random
    folds and 3 x 3 spatial blocks. A layout where some group leaves the drift nearly undetermined (smallest pivot
    below 1e-4 of its terms: both sides then lose digits to the conditioning) is not compared; there is one such
    layout (12 stations, four drift terms, two folds)."""
    done, worst, near = 0, [], 0
    for t in GLOBAL_FUZZ:
        c = cases.fuzz_config(t)
        obj = getattr(pk, c["cls"])(*c["data"], **c["kw"])
        p, P, cols = _problem(obj)
        n = P.shape[0]
        layouts = [kfold(n, (2, 5, 10)[t % 3], t), blocks(P, 3)]
        for groups in layouts:
            if np.unique(groups).size < 2:
                continue
            try:
                r = _check(p, P, cols, groups, min_pivot=1e-4)
            except np.linalg.LinAlgError:
                continue                    # drift undetermined without some group (a refusal, tested below)
            if r is None:
                near += 1
                continue
            worst.append(r[1])
            done += 1
    assert done >= 200 and near <= 2, (done, near)


def test_geographic_and_duplicate_draws(pk):
    """Geographic draws (great-circle distances) and exact duplicates with a nugget, with random folds: coincident
    stations fall both inside one group and across groups."""
    n_dup = 0
    for t in range(cases.N_KIND):
        c = cases.kind_config(t)
        if c["kind"] not in ("geo", "dups"):
            continue
        obj = getattr(pk, c["cls"])(*c["data"], **c["kw"])
        p, P, cols = _problem(obj)
        _check(p, P, cols, kfold(P.shape[0], 4, t))
        n_dup += c["kind"] == "dups"
    assert n_dup >= 20


@pytest.mark.parametrize("exact", [True, False])
def test_coincident_stations_inside_and_across_groups(pk, exact):
    """A coincident triple split over two groups, a coincident pair inside one group and a pair 1e-12 apart across
    groups; OK and UK (regional linear), two fields."""
    rng = np.random.default_rng(11)
    X = rng.uniform(0, 100, (60, 2))
    X[7] = X[3]
    X[21] = X[3]
    X[40] = X[12]
    X[30] = X[5] + np.array([1e-12, 0.0])
    groups = np.arange(60) % 6
    groups[[3, 7]] = 0
    groups[21] = 1
    groups[[12, 40]] = 2
    groups[5], groups[30] = 3, 4
    z = 5 + np.sin(X[:, 0] / 20) + rng.normal(size=60) * 0.3
    Zs = [z, rng.normal(size=60)]
    for cls, kw in (("OrdinaryKriging", {}), ("UniversalKriging", dict(drift_terms=["regional_linear"]))):
        obj = getattr(pk, cls)(X[:, 0], X[:, 1], z, variogram_model="exponential",
                               variogram_parameters=[1.2, 30.0, 0.1], exact_values=exact, **kw)
        p, P, cols = _problem(obj)
        _check(p, P, cols, groups, Zs)


def test_gauss_jordan_variant(pk):
    """Hole-effect on dense 2-D scatter: C is indefinite, G comes from the Gauss-Jordan inverse (gform 1)."""
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 10, (50, 2))
    z = rng.normal(size=50)
    for cls, kw in (("OrdinaryKriging", {}), ("UniversalKriging", dict(drift_terms=["regional_linear"]))):
        obj = getattr(pk, cls)(X[:, 0], X[:, 1], z, variogram_model="hole-effect", variogram_parameters=[1.0, 3.0, 0.0],
                               **kw)
        p, P, cols = _problem(obj)
        gform, _ = _check(p, P, cols, kfold(50, 5, 1), tol=1e-8)
        assert gform == 1


def test_singleton_groups_are_leave_one_out(pk):
    from test_loo_algebra import covariance_form_loo
    rng = np.random.default_rng(4)
    X = rng.uniform(0, 100, (30, 2))
    z = rng.normal(size=30)
    obj = pk.UniversalKriging(X[:, 0], X[:, 1], z, variogram_model="spherical", variogram_parameters=[1.0, 50.0, 0.1],
                              drift_terms=["regional_linear"])
    p, P, cols = _problem(obj)
    zg, sg, _, _ = covariance_form_lgo(P, p["fn"], p["m"], p["exact"], cols, 2, [z], np.arange(30))
    zl, sl, _, _ = covariance_form_loo(P, p["fn"], p["m"], p["exact"], cols, 2, [z])
    np.testing.assert_allclose(zg, zl, rtol=1e-10)
    np.testing.assert_allclose(sg, sl, rtol=1e-10)


def test_undetermined_drift_is_at_rounding_level(pk):
    """UK with a linear drift where every station outside group 0 lies on one line: without group 0 the drift is
    undetermined, P_SS of group 0 is singular to rounding, far below the 1e-10 threshold, and the brute force refuses."""
    rng = np.random.default_rng(9)
    t = rng.uniform(0, 100, 20)
    line = np.column_stack([t, 0.5 * t + 3.0])
    off = rng.uniform(0, 100, (6, 2))
    X = np.vstack([off, line])
    groups = np.r_[np.zeros(6, int), 1 + np.arange(20) % 3]
    z = rng.normal(size=26)
    obj = pk.UniversalKriging(X[:, 0], X[:, 1], z, variogram_model="exponential", variogram_parameters=[1.0, 40.0, 0.1],
                              drift_terms=["regional_linear"])
    p, P, cols = _problem(obj)
    _, _, _, worst = covariance_form_lgo(P, p["fn"], p["m"], p["exact"], cols, 2, [z], groups)
    assert worst < 1e-12, worst
    with pytest.raises(np.linalg.LinAlgError, match="group 0"):
        brute_force_lgo(P, z, p["fn"], p["m"], p["exact"], groups, cols)
