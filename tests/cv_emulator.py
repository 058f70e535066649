"""CPU emulation of kb200_loo / kb200_knn_loo / kb200_lgo / kb200_knn_lgo (include/krige_b200.h) — TEST INFRASTRUCTURE
ONLY.

`CvEmulatedHandle` is tests/fields_emulator.py's `FieldsEmulatedHandle` plus the four cross-validation entry points, all
by brute force: for every group the oracle kriges its stations from the stations outside it (a new matrix and solve per
group; leave-one-out: every station its own group), which is the definition the device's identities must meet. The
header's refusals are restated: pseudo-inverse, a problem received through kb200_blob_commit, bad group arrays, an
undetermined drift without a station or group, more than 32 stations of other groups within eps of one station, k
outside [2, n - 1] or above n - (largest group). When every group is one station, kb200_lgo is kb200_loo. Used by
tests/test_loo_host.py and tests/test_lgo_host.py; `brute_force_loo` and `brute_force_lgo` are also the references of
tests/test_loo_algebra.py, tests/test_lgo_algebra.py, tests/test_loo_gpu.py and tests/test_lgo_gpu.py."""
import re

import numpy as np
import scipy.linalg
from scipy.spatial.distance import cdist

from oracle import krige_oracle as ko
from fields_emulator import FieldsEmulatedHandle

MAXDUP = 32             # LOO_MAXDUP


def refined_solution(a, B, steps=2):
    """x = a^-1 B by oracle.krige_oracle.exec_vector_refined's scheme: one fp64 LU, then `steps` rounds of refinement
    with the residual B - a x formed and x held in np.longdouble. Returns (x, B) as np.longdouble arrays."""
    lu = scipy.linalg.lu_factor(a)
    A, BL = a.astype(np.longdouble), np.asarray(B).astype(np.longdouble)
    X = scipy.linalg.lu_solve(lu, B).astype(np.longdouble)
    for _ in range(steps):
        X += scipy.linalg.lu_solve(lu, (BL - A @ X).astype(np.float64)).astype(np.longdouble)
    return X, BL


def _refined_solve_many(a, P, Q, values, fn, m, exact, dp, steps=2):
    """oracle.krige_oracle.exec_vector_refined's scheme (fp64 LU, refinement with np.longdouble residuals, z and
    sigma^2 summed in np.longdouble) without its condition number, which costs an SVD per call, for several prediction
    points Q against one factorisation. dp: drift columns at the points."""
    n = P.shape[0]
    bd = cdist(Q, P)                                        # [q, n]
    B = np.zeros((a.shape[0], Q.shape[0]))
    B[:n] = -ko.variogram(fn, m, bd).T
    if exact:
        B[:n][np.absolute(bd.T) <= ko.EPS] = 0.0
    for c, col in enumerate(dp):
        B[n + c] = col
    B[-1] = 1.0
    X, BL = refined_solution(a, B, steps)
    z = (X[:n].T @ np.asarray(values, dtype=np.longdouble)).astype(np.float64)
    ss = (-np.sum(X * BL, axis=0)).astype(np.float64)
    return z, ss


def _refined_solve(a, P, q, values, fn, m, exact, dp, steps=2):
    """_refined_solve_many at the one point q [1, dim]; dp: drift columns at q. Returns (z, sigma^2) as floats."""
    z, ss = _refined_solve_many(a, P, q, values, fn, m, exact, dp, steps)
    return float(z[0]), float(ss[0])


def _moving_window_index_ties(P, q, values, fn, m, k, exact):
    """ok.py:722-758 at one point with the k nearest chosen by (d^2, original index), the device's tie rule; cKDTree
    breaks ties at the k-th distance its own way, which picks a different one of two coincident stations."""
    d2 = np.sum((P - q) ** 2, axis=1)
    sel = np.lexsort((np.arange(P.shape[0]), d2))[:k]
    bd = cdist(q, P[sel])[0]
    a = ko.kriging_matrix(P[sel], fn, m)
    b = np.zeros(k + 1)
    b[:k] = -ko.variogram(fn, m, bd)
    if exact:
        b[:k][np.absolute(bd) <= ko.EPS] = 0.0
    b[k] = 1.0
    x = scipy.linalg.solve(a, b)
    return np.array([x[:k] @ values[sel]]), np.array([-x @ b])


def near_pairs(P, geo, eps=ko.EPS):
    """Distances between stations as the device's pair scan sees them (|d| <= eps is a near pair)."""
    if geo:
        return ko.great_circle_distance(P[:, 0][:, None], P[:, 1][:, None], P[:, 0][None, :], P[:, 1][None, :])
    return cdist(P, P)


def brute_force_lgo(P, values, fn, m, exact, groups, drift_cols=(), k=None, geo=False, refined=False,
                    index_ties=False):
    """Every station kriged from the stations outside its group: P [n, dim] adjusted coordinates (lon/lat when geo),
    groups [n] labels, drift_cols the drift columns at the stations (regional-linear first), k the moving window.
    refined: extended-precision solves; index_ties: the moving window breaks distance ties by original index. Returns
    (z [n], sigmasq [n]); np.linalg.LinAlgError names the first group (in np.unique order) whose removal leaves the
    drift undetermined."""
    P = np.asarray(P, dtype=np.float64)
    values = np.asarray(values, dtype=np.float64)
    groups = np.asarray(groups)
    n = P.shape[0]
    z, ss = np.zeros(n), np.zeros(n)
    for g in np.unique(groups):
        S = np.flatnonzero(groups == g)
        keep = groups != g
        Q = P[S]
        if geo:
            zs, ss_ = ko.krige_geographic(P[keep], values[keep], fn, m, Q, exact_values=exact, n_closest_points=k)
        elif k is not None and index_ties:
            zs, ss_ = np.zeros(S.size), np.zeros(S.size)
            for t in range(S.size):
                a, b = _moving_window_index_ties(P[keep], Q[t:t + 1], values[keep], fn, m, int(k), exact)
                zs[t], ss_[t] = a[0], b[0]
        elif k is not None:
            zs, ss_ = ko.exec_moving_window(P[keep], Q, values[keep], fn, m, int(k), exact)
        else:
            dk = [np.asarray(c, dtype=np.float64)[keep] for c in drift_cols]
            F = np.column_stack(dk + [np.ones(int(keep.sum()))])
            if np.linalg.matrix_rank(F) < F.shape[1]:
                raise np.linalg.LinAlgError("leave-group-out: without group %s (lowest station %d) the drift terms "
                                            "are not determined" % (g, S[0]))
            a = ko.kriging_matrix(P[keep], fn, m, dk)
            dp = [np.asarray(c, dtype=np.float64)[S] for c in drift_cols]
            if refined:
                zs, ss_ = _refined_solve_many(a, P[keep], Q, values[keep], fn, m, exact, dp)
            else:
                zs, ss_ = ko.exec_vector(a, P[keep], Q, values[keep], fn, m, exact, dp)
        z[S], ss[S] = zs, ss_
    return z, ss


def brute_force_loo(P, values, fn, m, exact, drift_cols=(), k=None, geo=False, refined=False, index_ties=False):
    """brute_force_lgo with every station its own group: station i kriged from the other stations. Returns (z [n],
    sigmasq [n]); np.linalg.LinAlgError names the first station without which the drift is undetermined."""
    try:
        return brute_force_lgo(P, values, fn, m, exact, np.arange(np.shape(P)[0]), drift_cols, k, geo, refined,
                               index_ties)
    except np.linalg.LinAlgError as e:
        hit = re.search(r"lowest station (\d+)", str(e))
        if hit is None:
            raise
        raise np.linalg.LinAlgError("leave-one-out: without station %s the drift terms are not determined"
                                    % hit.group(1)) from None


def _check_groups(group, n_groups, n):
    group = np.asarray(group)
    if n_groups < 2 or group.shape != (n,) or group.min() < 0 or group.max() >= n_groups or \
            np.unique(group).size != n_groups:
        raise ValueError("leave-group-out: group must hold n indices in [0, n_groups), every group non-empty, "
                         "n_groups >= 2")
    return group


class CvEmulatedHandle(FieldsEmulatedHandle):
    from_blob = False

    def blob_commit(self):
        super().blob_commit()
        self.from_blob = True

    def set_problem(self, *args, **kwargs):
        self.from_blob = False
        super().set_problem(*args, **kwargs)

    def _fields_or_values(self):
        p = self.problem
        return [p["values"]] if self.fields is None else list(self.fields)

    def _global(self, what, n):
        """The refusals of the global path (kb200_loo / kb200_lgo); returns the problem."""
        from pykrige_b200 import _cabi
        p = self.problem
        if p is None or p["knn"] or not getattr(self, "ready", False):
            raise _cabi.KrigeB200Error("no factored problem: call kb200_set_problem first")
        if p["pinv"]:
            raise NotImplementedError("%s has no pseudo-inverse form" % what)
        if self.from_blob:
            raise _cabi.KrigeB200Error("the factorisation is not on this handle (problem received through "
                                       "kb200_blob_commit)")
        assert int(n) == p["X"].shape[0]
        return p

    def _brute_force(self, group, k=None):
        """brute_force_lgo (group None: brute_force_loo) of every value field on the held problem; on the moving window
        a LinAlgError is the solver's 'Singular matrix'."""
        p = self.problem
        P = p["X"] if p["geo"] else p["P"]
        cols = [] if p["geo"] or k is not None else \
            ([P[:, c] for c in range(p["dim"])] if p["n_rl"] else []) + list(p["hd"])

        def one(v):
            if group is None:
                return brute_force_loo(P, v, p["fn"], p["m"], p["exact"], cols, k=k, geo=p["geo"])
            return brute_force_lgo(P, v, p["fn"], p["m"], p["exact"], group, cols, k=k, geo=p["geo"])
        try:
            out = [one(v) for v in self._fields_or_values()]
        except np.linalg.LinAlgError:
            if k is None:
                raise
            raise ValueError("Singular matrix")
        return np.concatenate([o[0] for o in out]), out[0][1]

    def loo(self, n):
        self.calls.append("loo")
        self._global("leave-one-out", n)
        return self._brute_force(None)

    def knn_loo(self, k, n):
        self.calls.append("knn_loo")
        p = self.problem
        assert p is not None and p["knn"], "kb200_set_problem_knn first"
        assert int(n) == p["X"].shape[0]
        if not 2 <= int(k) <= int(n) - 1:
            raise ValueError("leave-one-out: n_closest_points must be in [2, n - 1]")
        return self._brute_force(None, int(k))

    def lgo(self, group, n_groups, n):
        self.calls.append("lgo")
        p = self._global("leave-group-out", n)
        group = _check_groups(group, n_groups, int(n))
        if int(n_groups) == int(n):
            return self.loo(n)
        if p["exact"]:
            D = near_pairs(p["X"] if p["geo"] else p["P"], p["geo"])
            near = (np.abs(D) <= ko.EPS) & (group[:, None] != group[None, :])
            if near.sum(axis=1).max() > MAXDUP:
                raise NotImplementedError("leave-group-out: station %d has more than %d stations of other groups "
                                          "within eps" % (int(np.argmax(near.sum(axis=1))), MAXDUP))
        return self._brute_force(group)

    def knn_lgo(self, k, group, n_groups, n):
        self.calls.append("knn_lgo")
        p = self.problem
        assert p is not None and p["knn"], "kb200_set_problem_knn first"
        group = _check_groups(group, n_groups, int(n))
        if not 2 <= int(k) <= int(n) - np.bincount(group).max():
            raise ValueError("leave-group-out: n_closest_points must be at most n - (size of the largest group)")
        return self._brute_force(group, int(k))
