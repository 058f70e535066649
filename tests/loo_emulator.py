"""CPU emulation of kb200_loo / kb200_knn_loo (include/krige_b200.h) — TEST INFRASTRUCTURE ONLY.

`LooEmulatedHandle` is tests/fields_emulator.py's `FieldsEmulatedHandle` plus the two leave-one-out entry points, both
by brute force: for every station the oracle kriges it from the other n - 1 stations (a new matrix and inverse per
station), which is the definition the device's one-pass identities must meet. The header's refusals are restated:
pseudo-inverse, a problem received through kb200_blob_commit, an undetermined drift without a station, k outside
[2, n - 1]. Used by tests/test_loo_host.py; `brute_force_loo` is also the reference of tests/test_loo_algebra.py and
tests/test_loo_gpu.py."""
import numpy as np
import scipy.linalg
from scipy.spatial.distance import cdist

from oracle import krige_oracle as ko
from fields_emulator import FieldsEmulatedHandle


def _refined_solve(a, P, q, values, fn, m, exact, dp, steps=2):
    """The one-point form of oracle.krige_oracle.exec_vector_refined (fp64 LU, refinement with np.longdouble
    residuals, z and sigma^2 summed in np.longdouble) without its condition number, which costs an SVD per call."""
    n = P.shape[0]
    bd = cdist(q, P)[0]
    b = np.zeros(a.shape[0])
    b[:n] = -ko.variogram(fn, m, bd)
    if exact:
        b[:n][np.absolute(bd) <= ko.EPS] = 0.0
    for c, col in enumerate(dp):
        b[n + c] = col[0]
    b[-1] = 1.0
    lu = scipy.linalg.lu_factor(a)
    A, B = a.astype(np.longdouble), b.astype(np.longdouble)
    x = scipy.linalg.lu_solve(lu, b).astype(np.longdouble)
    for _ in range(steps):
        x += scipy.linalg.lu_solve(lu, (B - A @ x).astype(np.float64)).astype(np.longdouble)
    return float(x[:n] @ np.asarray(values, dtype=np.longdouble)), float(-(x @ B))


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


def brute_force_loo(P, values, fn, m, exact, drift_cols=(), k=None, geo=False, refined=False, index_ties=False):
    """Station i kriged from the other stations: P [n, dim] adjusted coordinates (lon/lat when geo), drift_cols the
    drift columns at the stations in the reference's order (regional-linear first), k the moving window. refined:
    extended-precision solves (exec_vector_refined's scheme) instead of exec_vector. index_ties: the moving window
    breaks distance ties by original index (as the device does) instead of cKDTree's order. Returns (z [n],
    sigmasq [n])."""
    P = np.asarray(P, dtype=np.float64)
    values = np.asarray(values, dtype=np.float64)
    n = P.shape[0]
    z, ss = np.zeros(n), np.zeros(n)
    for i in range(n):
        keep = np.arange(n) != i
        Q = P[i:i + 1]
        if geo:
            zi, si = ko.krige_geographic(P[keep], values[keep], fn, m, Q, exact_values=exact, n_closest_points=k)
        elif k is not None and index_ties:
            zi, si = _moving_window_index_ties(P[keep], Q, values[keep], fn, m, int(k), exact)
        elif k is not None:
            zi, si = ko.exec_moving_window(P[keep], Q, values[keep], fn, m, int(k), exact)
        else:
            dk = [np.asarray(c, dtype=np.float64)[keep] for c in drift_cols]
            F = np.column_stack(dk + [np.ones(n - 1)])
            if np.linalg.matrix_rank(F) < F.shape[1]:
                raise np.linalg.LinAlgError("leave-one-out: without station %d the drift terms are not determined" % i)
            a = ko.kriging_matrix(P[keep], fn, m, dk)
            dp = [np.asarray(c, dtype=np.float64)[i:i + 1] for c in drift_cols]
            if refined:
                zi, si = (np.array([v]) for v in _refined_solve(a, P[keep], Q, values[keep], fn, m, exact, dp))
            else:
                zi, si = ko.exec_vector(a, P[keep], Q, values[keep], fn, m, exact, dp)
        z[i], ss[i] = zi[0], si[0]
    return z, ss


class LooEmulatedHandle(FieldsEmulatedHandle):
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

    def loo(self, n):
        from pykrige_b200 import _cabi
        self.calls.append("loo")
        p = self.problem
        if p is None or p["knn"] or not getattr(self, "ready", False):
            raise _cabi.KrigeB200Error("no factored problem: call kb200_set_problem first")
        if p["pinv"]:
            raise NotImplementedError("leave-one-out has no pseudo-inverse form")
        if self.from_blob:
            raise _cabi.KrigeB200Error("the factorisation is not on this handle (problem received through "
                                       "kb200_blob_commit)")
        assert int(n) == p["X"].shape[0]
        if p["geo"]:
            P, cols = p["X"], []
        else:
            P = p["P"]
            cols = ([P[:, c] for c in range(p["dim"])] if p["n_rl"] else []) + list(p["hd"])
        out = [brute_force_loo(P, v, p["fn"], p["m"], p["exact"], cols, geo=p["geo"]) for v in self._fields_or_values()]
        return np.concatenate([o[0] for o in out]), out[0][1]

    def knn_loo(self, k, n):
        self.calls.append("knn_loo")
        p = self.problem
        assert p is not None and p["knn"], "kb200_set_problem_knn first"
        assert int(n) == p["X"].shape[0]
        if not 2 <= int(k) <= int(n) - 1:
            raise ValueError("leave-one-out: n_closest_points must be in [2, n - 1]")
        P = p["X"] if p["geo"] else p["P"]
        try:
            out = [brute_force_loo(P, v, p["fn"], p["m"], p["exact"], k=int(k), geo=p["geo"])
                   for v in self._fields_or_values()]
        except np.linalg.LinAlgError:
            raise ValueError("Singular matrix")
        return np.concatenate([o[0] for o in out]), out[0][1]
