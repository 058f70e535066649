"""CPU emulation of kb200_lgo / kb200_knn_lgo (include/krige_b200.h) — TEST INFRASTRUCTURE ONLY.

`LgoEmulatedHandle` is tests/loo_emulator.py's `LooEmulatedHandle` plus the two leave-group-out entry points, both by
brute force: for every group the oracle kriges its stations from the stations outside it (a new matrix and solve per
group), which is the definition the device's identities must meet. The header's refusals are restated: bad group
arrays, an undetermined drift without a group, more than 32 stations of other groups within eps of one station, k above
n - (largest group). When every group is one station, kb200_lgo is kb200_loo. Used by tests/test_lgo_host.py;
`brute_force_lgo` is also the reference of tests/test_lgo_algebra.py and tests/test_lgo_gpu.py."""
import numpy as np
import scipy.linalg
from scipy.spatial.distance import cdist

from oracle import krige_oracle as ko
from loo_emulator import LooEmulatedHandle, _moving_window_index_ties

MAXDUP = 32             # LOO_MAXDUP


def _refined_solve_many(a, P, Q, values, fn, m, exact, dp, steps=2):
    """loo_emulator._refined_solve for several prediction points against one factorisation: fp64 LU, refinement with
    np.longdouble residuals, z and sigma^2 summed in np.longdouble. dp: drift columns at the points."""
    n = P.shape[0]
    bd = cdist(Q, P)                                        # [q, n]
    B = np.zeros((a.shape[0], Q.shape[0]))
    B[:n] = -ko.variogram(fn, m, bd).T
    if exact:
        B[:n][np.absolute(bd.T) <= ko.EPS] = 0.0
    for c, col in enumerate(dp):
        B[n + c] = col
    B[-1] = 1.0
    lu = scipy.linalg.lu_factor(a)
    A, BL = a.astype(np.longdouble), B.astype(np.longdouble)
    X = scipy.linalg.lu_solve(lu, B).astype(np.longdouble)
    for _ in range(steps):
        X += scipy.linalg.lu_solve(lu, (BL - A @ X).astype(np.float64)).astype(np.longdouble)
    z = (X[:n].T @ np.asarray(values, dtype=np.longdouble)).astype(np.float64)
    ss = (-np.sum(X * BL, axis=0)).astype(np.float64)
    return z, ss


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


def _check_groups(group, n_groups, n):
    group = np.asarray(group)
    if n_groups < 2 or group.shape != (n,) or group.min() < 0 or group.max() >= n_groups or \
            np.unique(group).size != n_groups:
        raise ValueError("leave-group-out: group must hold n indices in [0, n_groups), every group non-empty, "
                         "n_groups >= 2")
    return group


class LgoEmulatedHandle(LooEmulatedHandle):

    def lgo(self, group, n_groups, n):
        from pykrige_b200 import _cabi
        self.calls.append("lgo")
        p = self.problem
        if p is None or p["knn"] or not getattr(self, "ready", False):
            raise _cabi.KrigeB200Error("no factored problem: call kb200_set_problem first")
        if p["pinv"]:
            raise NotImplementedError("leave-group-out has no pseudo-inverse form")
        if self.from_blob:
            raise _cabi.KrigeB200Error("the factorisation is not on this handle (problem received through "
                                       "kb200_blob_commit)")
        group = _check_groups(group, n_groups, int(n))
        if int(n_groups) == int(n):
            return self.loo(n)
        P = p["X"] if p["geo"] else p["P"]
        if p["exact"]:
            D = near_pairs(P, p["geo"])
            near = (np.abs(D) <= ko.EPS) & (group[:, None] != group[None, :])
            if near.sum(axis=1).max() > MAXDUP:
                raise NotImplementedError("leave-group-out: station %d has more than %d stations of other groups "
                                          "within eps" % (int(np.argmax(near.sum(axis=1))), MAXDUP))
        cols = [] if p["geo"] else ([P[:, c] for c in range(p["dim"])] if p["n_rl"] else []) + list(p["hd"])
        out = [brute_force_lgo(P, v, p["fn"], p["m"], p["exact"], group, cols, geo=p["geo"])
               for v in self._fields_or_values()]
        return np.concatenate([o[0] for o in out]), out[0][1]

    def knn_lgo(self, k, group, n_groups, n):
        self.calls.append("knn_lgo")
        p = self.problem
        assert p is not None and p["knn"], "kb200_set_problem_knn first"
        group = _check_groups(group, n_groups, int(n))
        if not 2 <= int(k) <= int(n) - np.bincount(group).max():
            raise ValueError("leave-group-out: n_closest_points must be at most n - (size of the largest group)")
        P = p["X"] if p["geo"] else p["P"]
        try:
            out = [brute_force_lgo(P, v, p["fn"], p["m"], p["exact"], group, k=int(k), geo=p["geo"])
                   for v in self._fields_or_values()]
        except np.linalg.LinAlgError:
            raise ValueError("Singular matrix")
        return np.concatenate([o[0] for o in out]), out[0][1]
