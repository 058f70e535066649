"""The leave-one-out formulation of DESIGN.md §5e, pinned in numpy, independent of any kernel.

The device computes every station's leave-one-out estimate and variance from the covariance form it already holds
(c0 search, rescaled drift basis, W = L^-1 or G = C^-1 on the indefinite fallback, U, zeta, S^-1, phi):
    P_ii = ||W[:, i]||^2 - u_i^T S^-1 u_i,   sigma^2_-i = 1 / P_ii,   zhat_-i = Z_i - alpha_i / P_ii,
    alpha = zeta - U S^-1 phi,
plus an exact-hit correction from P and alpha on {i} + D(i) when exact_values puts another station within eps. This
file restates exactly that in numpy and compares it with brute-force reduced solves (tests/loo_emulator.py) on the
fuzz draws of tests/cases.py (all four classes, every drift kind, anisotropy, both exact_values), the geographic and
duplicate draws, hand-made coincident stations and the Gauss-Jordan variant; the sequential statistics give a
cross-check for the last station."""
import numpy as np
import pytest
import scipy.linalg
from scipy.spatial.distance import cdist

import cases
from cv_emulator import CvEmulatedHandle as LooEmulatedHandle, brute_force_loo
from oracle import krige_oracle as ko

TOL = 1e-9          # max|covariance form - brute force| / max|brute force|, z and sigma^2


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", LooEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def _distances(P, geo):
    if geo:
        return ko.great_circle_distance(P[:, 0][:, None], P[:, 1][:, None], P[:, 0][None, :], P[:, 1][None, :])
    return cdist(P, P)


def _c0(P, fn, m, geo):
    """api.cu describe(): the sill for bounded models, gamma(bounding-box diagonal) (180 degrees geographic) else."""
    if fn in ("linear", "power") or callable(fn):
        if geo:
            d = 180.0
        else:
            d = float(np.sqrt(np.sum((P.max(0) - P.min(0)) ** 2)))
        if callable(fn):
            dd = np.linspace(0.0, d, 4097)
            c0 = float(np.max(ko.variogram(fn, m, dd)))
        else:
            c0 = float(ko.variogram(fn, m, np.array([d]))[0])
        return c0 if c0 > 0 else 1.0, True
    return float(m[0] + m[2]), False


def _rescale(P, n_rl, cols):
    """The device's change of drift basis: regional-linear about the bounding-box centre over the half width,
    host columns about their mean over the largest deviation (api.cu describe())."""
    out = []
    for c in range(n_rl):
        lo, hi = P[:, c].min(), P[:, c].max()
        half = 0.5 * (hi - lo)
        out.append((P[:, c] - 0.5 * (hi + lo)) * (1.0 / half if half > 0 else 1.0))
    for col in cols[n_rl:]:
        col = np.asarray(col, dtype=np.float64)
        mean = col.mean()
        amax = np.abs(col - mean).max()
        out.append((col - mean) * (1.0 / amax if amax > 0 else 1.0))
    return out


def covariance_form_loo(P, fn, m, exact, drift_cols, n_rl, Zs, geo=False, eps=ko.EPS):
    """Every station's leave-one-out (zhat [V, n], sigma^2 [n], gform, max ||W_i||^2 / P_ii) from the covariance form."""
    P = np.asarray(P, dtype=np.float64)
    n = P.shape[0]
    D = _distances(P, geo)
    Gam = ko.variogram(fn, m, D)
    np.fill_diagonal(Gam, 0.0)
    c0, unbounded = _c0(P, fn, m, geo)
    gform, L = 1, None
    for _ in range(5 if unbounded else 1):
        C = c0 - Gam
        try:
            L = np.linalg.cholesky(C)
            gform = 0
            break
        except np.linalg.LinAlgError:
            c0 *= 2.0
    if gform:
        c0 = _c0(P, fn, m, geo)[0]
        C = c0 - Gam
        Cinv = scipy.linalg.inv(C)
        diag = np.diag(Cinv).copy()
    else:
        W = scipy.linalg.solve_triangular(L, np.eye(n), lower=True)
        Cinv = W.T @ W
        diag = np.sum(W * W, axis=0)                      # column sums of squares of the lower-triangular W
    F = np.column_stack(_rescale(P, n_rl, drift_cols) + [np.ones(n)])
    Z = np.column_stack(Zs)
    U, zeta = Cinv @ F, Cinv @ Z
    S = F.T @ U
    Sinv = np.linalg.inv(0.5 * (S + S.T))
    phi = F.T @ zeta
    wt = U @ Sinv
    usu = np.sum(wt * U, axis=1)
    pii = diag - usu
    alpha = zeta - wt @ phi
    ss = 1.0 / pii
    zh = Z - alpha / pii[:, None]
    if exact:
        Pm = Cinv - U @ Sinv @ U.T
        for i in range(n):
            Dj = np.flatnonzero((np.abs(D[i]) <= eps) & (np.arange(n) != i))
            if Dj.size == 0:
                continue
            dl = ko.variogram(fn, m, D[i, Dj])
            pij = Pm[i, Dj]
            zh[i] += dl @ (alpha[Dj] - np.outer(pij / pii[i], alpha[i]))
            ss[i] += 2.0 * dl @ pij / pii[i] - dl @ (Pm[np.ix_(Dj, Dj)] - np.outer(pij, pij) / pii[i]) @ dl
    return zh.T, ss, gform, float(np.max(diag / np.abs(pii)))


def _problem(pk, obj):
    """The problem the class hands to the C ABI (the emulator records it): adjusted stations, drift columns, model."""
    obj._ensure_problem("float64")
    p = obj._kb_handle.problem
    P = p["X"] if p["geo"] else p["P"]
    cols = ([P[:, c] for c in range(p["dim"])] if p["n_rl"] else []) + list(p["hd"])
    return p, P, cols


def _check(p, P, cols, Zs=None, tol=TOL):
    Zs = [p["values"]] if Zs is None else Zs
    zh, ss, gform, ratio = covariance_form_loo(P, p["fn"], p["m"], p["exact"], cols, p["dim"] if p["n_rl"] else 0,
                                               Zs, geo=p["geo"])
    for v, Zv in enumerate(Zs):
        zr, sr = brute_force_loo(P, Zv, p["fn"], p["m"], p["exact"], cols, geo=p["geo"], refined=not p["geo"])
        scale = max(np.abs(zr).max(), 1e-300)
        assert np.abs(zh[v] - zr).max() <= tol * scale, (np.abs(zh[v] - zr).max() / scale)
        assert np.abs(ss - sr).max() <= tol * np.abs(sr).max(), (np.abs(ss - sr).max() / np.abs(sr).max())
    return gform, ratio


GLOBAL_FUZZ = [t for t in range(cases.N_FUZZ) if cases.fuzz_config(t) is not None and cases.fuzz_config(t)["knn"] is None]


def test_fuzz_draws_match_brute_force(pk):
    """The global fuzz draws: OK / UK / OK3D / UK3D, regional-linear, point_log, external_Z, specified and functional
    drift, anisotropy, both exact_values (several draws put a prediction point on a station; here every station)."""
    seen, ratios = set(), []
    for t in GLOBAL_FUZZ:
        c = cases.fuzz_config(t)
        obj = getattr(pk, c["cls"])(*c["data"], **c["kw"])
        p, P, cols = _problem(pk, obj)
        try:
            _, ratio = _check(p, P, cols)
        except np.linalg.LinAlgError:
            continue                   # drift undetermined without some station (a refusal, tested below)
        ratios.append(ratio)
        seen.add((c["cls"], tuple(c["kw"].get("drift_terms", ())), p["exact"]))
    assert len(ratios) >= 150, len(ratios)
    assert {s[0] for s in seen} == {"OrdinaryKriging", "UniversalKriging", "OrdinaryKriging3D", "UniversalKriging3D"}
    assert {e for s in seen for e in s[1]} == {"regional_linear", "point_log", "external_Z", "specified", "functional"}
    assert {s[2] for s in seen} == {True, False}
    # the refusal threshold of kb200_loo (|P_ii| <= 1e-10 of its terms) is far from every draw
    assert max(ratios) < 1e6, max(ratios)


def test_geographic_and_duplicate_draws(pk):
    """kind draws: geographic (great-circle distances) and exact duplicates with a nugget (exact-hit correction)."""
    n_dup = 0
    for t in range(cases.N_KIND):
        c = cases.kind_config(t)
        if c["kind"] not in ("geo", "dups"):
            continue
        obj = getattr(pk, c["cls"])(*c["data"], **c["kw"])
        p, P, cols = _problem(pk, obj)
        _check(p, P, cols)
        n_dup += c["kind"] == "dups"
    assert n_dup >= 20


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("model,params", [("exponential", [1.2, 30.0, 0.1]), ("spherical", [2.0, 45.0, 0.05]),
                                          ("gaussian", [1.5, 40.0, 0.02])])
def test_coincident_triple_and_near_pair(pk, exact, model, params):
    """A coincident triple and a pair 1e-12 apart (inside eps) with a nugget: the exact-hit correction covers every
    j != i within eps, not only earlier stations; OK and UK (regional linear), several fields."""
    rng = np.random.default_rng(11)
    X = rng.uniform(0, 100, (40, 2))
    X[7] = X[3]
    X[21] = X[3]
    X[30] = X[12] + np.array([1e-12, 0.0])
    z = 5 + np.sin(X[:, 0] / 20) + rng.normal(size=40) * 0.3
    Zs = [z, rng.normal(size=40)]
    for cls, kw in (("OrdinaryKriging", {}), ("UniversalKriging", dict(drift_terms=["regional_linear"]))):
        obj = getattr(pk, cls)(X[:, 0], X[:, 1], z, variogram_model=model, variogram_parameters=params,
                               exact_values=exact, **kw)
        p, P, cols = _problem(pk, obj)
        _check(p, P, cols, Zs)


def test_gauss_jordan_variant(pk):
    """Hole-effect on dense 2-D scatter: C is indefinite, the device inverts it by Gauss-Jordan (gform 1) and reads
    the diagonal of G instead of the column norms of W."""
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 10, (50, 2))
    z = rng.normal(size=50)
    for cls, kw in (("OrdinaryKriging", {}), ("UniversalKriging", dict(drift_terms=["regional_linear"]))):
        obj = getattr(pk, cls)(X[:, 0], X[:, 1], z, variogram_model="hole-effect", variogram_parameters=[1.0, 3.0, 0.0],
                               **kw)
        p, P, cols = _problem(pk, obj)
        gform, _ = _check(p, P, cols, tol=1e-8)
        assert gform == 1


def test_undetermined_drift_is_at_rounding_level(pk):
    """UK with regional-linear drift on three stations: without any one of them the drift is singular, and P_ii is
    rounding noise far below the 1e-10 threshold kb200_loo refuses at."""
    X = np.array([[0.0, 0.0], [10.0, 1.0], [3.0, 9.0]])
    obj = pk.UniversalKriging(X[:, 0], X[:, 1], np.array([1.0, 2.0, 0.5]), variogram_model="exponential",
                              variogram_parameters=[1.0, 20.0, 0.1], drift_terms=["regional_linear"])
    p, P, cols = _problem(pk, obj)
    with np.errstate(divide="ignore", invalid="ignore"):
        _, _, _, ratio = covariance_form_loo(P, p["fn"], p["m"], p["exact"], cols, 2, [p["values"]])
    assert ratio > 1e12, ratio
    with pytest.raises(np.linalg.LinAlgError, match="station 0"):
        brute_force_loo(P, p["values"], p["fn"], p["m"], p["exact"], cols)


def test_last_station_equals_the_sequential_statistic(pk):
    """core._find_statistics kriges station i from stations [0, i): for the last station that is its leave-one-out
    residual."""
    rng = np.random.default_rng(5)
    X = rng.uniform(0, 100, (30, 2))
    z = rng.normal(size=30)
    obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], z, variogram_model="spherical", variogram_parameters=[1.0, 50.0, 0.1])
    p, P, cols = _problem(pk, obj)
    zh, ss, _, _ = covariance_form_loo(P, p["fn"], p["m"], p["exact"], cols, 0, [z])
    delta, sigma, _ = ko.find_statistics(P, z, p["fn"], p["m"])
    np.testing.assert_allclose(z[-1] - zh[0, -1], delta[-1], rtol=1e-10)
    np.testing.assert_allclose(np.sqrt(ss[-1]), sigma[-1], rtol=1e-10)
