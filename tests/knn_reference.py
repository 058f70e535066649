"""Exact reference of one moving-window query (execute(n_closest_points=k), ok.py:722-758) — TEST INFRASTRUCTURE ONLY.

For each prediction point it gives
- the expected neighbour set: brute-force squared distances in the adjusted frame, ranked by (d^2, original index),
  the device's tie rule (cKDTree breaks ties its own way). Geographic data are ranked by chord length on the unit
  sphere (ok.py:936-960);
- an ambiguity flag: when stations other than exact ties lie within rounding of the k-th distance, the device's
  fma-contracted d^2 and numpy's may rank them differently, so any choice of them is accepted;
- the local weights lambda (k), z, sigma^2 and kappa_2 of the (k+1)^2 gamma-form system (ok.py:738-756, exact-hit rule
  ok.py:741-751), solved by fp64 LU plus refinement with np.longdouble residuals (cv_emulator.refined_solution), so
  that the result carries about kappa * 1e-19 instead of the kappa * eps of an fp64 solve. Geographic data are kriged
  with great-circle distances (ok.py:962-969).

The adjusted frame is the device's: (x - c) goes through the pre-multiplied anisotropy matrix of core.anisotropy_matrix
with every product and sum rounded separately (csrc/common.cuh kb_adjust), which numpy's element-wise arithmetic
reproduces bit for bit. It is the reference's map (oracle.krige_oracle.adjust_for_anisotropy) to a few ulp; using the
device's rounding keeps an ulp of a coordinate at a 5e6 offset out of the comparison of the search and the solve.

Also the host-side geometry of the launch: a mirror of kbk_knn_smem_per_warp (csrc/knn.cu), the points per CTA it
allows and the largest k check_knn (csrc/api.cu) accepts."""
import numpy as np
from scipy.spatial.distance import cdist

from cv_emulator import refined_solution
from oracle import krige_oracle as ko

KN_CAP = 512                    # candidate buffer per warp (knn.cu)
KN_SELECT_DOUBLES = 272         # selection scratch (knn.cu)
SMEM_PER_CTA = 226 * 1024       # dynamic shared memory one launch spreads over its warps (kbk_knn_solve)
SMEM_K_LIMIT = 200 * 1024       # check_knn: the LU footprint of k must stay below this
CHOL_K_MAX = 128                # the tiled Cholesky handles k <= 128, LU the rest


def smem_per_warp(k, chol, hasz, nv):
    """Bytes of shared memory one prediction point (one warp) of the moving-window kernel uses."""
    S = k | 1
    kp = (k + 7) & ~7 if chol else k
    nt, naug = kp // 8, (2 + nv + 7) // 8
    a = (nt * (nt + 1) // 2 + naug * nt + 1) * 64 if chol else k * S
    c = KN_CAP + KN_CAP // 2 + KN_SELECT_DOUBLES
    tail = (5 if hasz else 4) if chol else 7
    return (max(a, c) + tail * kp + 2) * 8


def points_per_cta(k, chol, hasz, nv):
    """wpc of kbk_knn_solve: prediction points (warps) per CTA."""
    return min(10, SMEM_PER_CTA // smem_per_warp(k, chol, hasz, nv))


def k_supported(k):
    return smem_per_warp(k, 0, 1, 1) <= SMEM_K_LIMIT


def device_frame(X, center, M):
    """Adjusted coordinates as kb_adjust computes them: c + M (x - c), every operation rounded on its own."""
    X = np.asarray(X, dtype=np.float64)
    c = np.asarray(center, dtype=np.float64)
    d = X - c[None, :]
    out = np.empty_like(d)
    for r in range(X.shape[1]):
        acc = M[r][0] * d[:, 0]
        for q in range(1, X.shape[1]):
            acc = acc + M[r][q] * d[:, q]
        out[:, r] = acc + c[r]
    return out


class Neighbours:
    """The expected neighbour set of one point. must: stations certainly among the k nearest; band: stations within
    rounding of the k-th distance, of which `need` are neighbours; sel: the set under the (d^2, index) rule; flagged:
    the band is ambiguous, so any `need` of it are accepted."""

    def __init__(self, must, band, need, sel, flagged):
        self.must, self.band, self.need, self.sel, self.flagged = must, band, need, sel, flagged

    def allowed(self):
        return np.union1d(self.must, self.band)

    def accepts(self, s):
        s = np.asarray(s)
        if not self.flagged:
            return np.array_equal(np.sort(s), np.sort(self.sel))
        return (s.size == self.must.size + self.need and np.all(np.isin(self.must, s))
                and np.all(np.isin(s, self.allowed())))


def neighbours(S, q, k, exclude=None, rel=1e-12):
    """The k nearest of the search coordinates S [n, d] to q [d] by (d^2, original index); exclude: stations that
    are never candidates (leave-one-out / leave-group-out). A station within rel * d_k^2 plus a few coordinate ulps
    of the k-th d^2 is in the band; a band that holds only exact ties of the k-th d^2 is decided by index."""
    S = np.asarray(S, dtype=np.float64)
    d2 = np.sum((S - q[None, :]) ** 2, axis=1)
    idx = np.arange(S.shape[0])
    ok = np.ones(S.shape[0], bool)
    if exclude is not None:
        ok[np.asarray(exclude, dtype=np.int64)] = False
    order = np.lexsort((idx[ok], d2[ok]))
    cand = idx[ok][order]
    sel = np.sort(cand[:k])
    dk = d2[cand[k - 1]]
    ulp = 8.0 * np.finfo(np.float64).eps * max(float(np.max(np.abs(S))), float(np.max(np.abs(q))))
    tol = rel * dk + 4.0 * np.sqrt(dk) * ulp + ulp * ulp
    e = d2[cand]
    must = np.sort(cand[e < dk - tol])
    band = np.sort(cand[np.abs(e - dk) <= tol])
    need = k - must.size
    exact_ties = np.all(d2[band] == dk)
    flagged = not exact_ties and band.size > need
    return Neighbours(must, band, need, sel, flagged)


def search_coords(P, geo):
    """Coordinates the device ranks by: adjusted x, y(, z), or unit vectors for lon/lat."""
    return ko._unit_sphere(P) if geo else P


def local_system(P, q, fn, m, exact, geo):
    """(a, b) of the local gamma-form system of the neighbours P [k, d] (lon/lat when geo) at the point q [d]."""
    k = P.shape[0]
    if geo:
        gc = lambda A, B: ko.great_circle_distance(A[:, 0][:, None], A[:, 1][:, None], B[:, 0][None, :],
                                                   B[:, 1][None, :])
        a = np.zeros((k + 1, k + 1))
        a[:k, :k] = -ko.variogram(fn, m, gc(P, P))
        np.fill_diagonal(a, 0.0)
        a[k, :k] = a[:k, k] = 1.0
        bd = gc(q[None, :], P)[0]
    else:
        a = ko.kriging_matrix(P, fn, m)
        bd = cdist(q[None, :], P)[0]
    b = np.zeros(k + 1)
    b[:k] = -ko.variogram(fn, m, bd)
    if exact:
        b[:k][np.absolute(bd) <= ko.EPS] = 0.0
    b[k] = 1.0
    return a, b


def local_solution(P, q, values, fn, m, exact, geo=False, kappa=True):
    """(lambda [k], z, sigma^2, kappa_2) of kriging q from the neighbours P [k, d] with values [k] (or [k, V]: z [V])
    in extended precision."""
    a, b = local_system(P, q, fn, m, exact, geo)
    X, BL = refined_solution(a, b[:, None])
    x = X[:, 0]
    k = P.shape[0]
    z = (np.asarray(values, dtype=np.longdouble).T @ x[:k]).astype(np.float64)
    ss = float(-np.sum(x * BL[:, 0]))
    return x[:k].astype(np.float64), z, ss, (float(np.linalg.cond(a)) if kappa else float("nan"))


def moving_window(P, Q, values, fn, m, k, exact=True, geo=False):
    """execute(n_closest_points=k) at the points Q: (z, sigma^2, kappa_2, flagged) per point, neighbours by the
    (d^2, index) rule."""
    S, SQ = search_coords(P, geo), search_coords(Q, geo)
    out = np.zeros((4, Q.shape[0]))
    for i in range(Q.shape[0]):
        nb = neighbours(S, SQ[i], k)
        _, z, ss, kap = local_solution(P[nb.sel], Q[i], values[nb.sel], fn, m, exact, geo)
        out[:, i] = z, ss, kap, nb.flagged
    return out[0], out[1], out[2], out[3].astype(bool)
