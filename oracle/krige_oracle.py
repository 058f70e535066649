"""CPU oracle for the kriging execute() hot path — TEST INFRASTRUCTURE ONLY.

A plain numpy/scipy restatement of the reference's algorithm (GeoStat-Framework/PyKrige
v1.7.3, commit 5e896fb), one function per reference step, each citing the file:line it follows.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module; the product path (pykrige_b200) never does.

Parity pinning: this oracle is checked in tests/test_oracle.py against
  * the reference's own golden vectors (KT3D_H2O / KT3D answers of tests/test_core.py:490-507,
    707-725, 1957-1989, stored in tests/golden/reference_goldens.npz), and
  * outputs of the imported reference itself (backend='vectorized' / 'loop'), generated here by
    tests/golden/make_golden.py and stored in tests/golden/*.npz, and
  * the reference's own compiled native twins (lib/cok.pyx) built into oracle/_ref by
    oracle/build_ref.py and driven by oracle/ref_native.py (same inputs, fresh seeds).

The arithmetic deliberately stays in the reference's form (gamma-form matrix with zero diagonal,
explicit inverse, inverse x RHS) — NOT the covariance/Cholesky form the CUDA path uses — so that
the comparison is between two independent formulations.
"""
import numpy as np
import scipy.linalg
from scipy.spatial import cKDTree
from scipy.spatial.distance import cdist

EPS = 1.0e-10  # ok.py:177


# ---- variogram models: variogram_models.py:25-81 ------------------------------------
def variogram(model, m, d):
    d = np.asarray(d, dtype=np.float64)
    if callable(model):          # variogram_model='custom': user callable f(params, d), ok.py:247-253
        return np.asarray(model(m, d), dtype=np.float64)
    if model == "linear":        # variogram_models.py:25-29
        return float(m[0]) * d + float(m[1])
    if model == "power":         # :32-37
        return float(m[0]) * d ** float(m[1]) + float(m[2])
    psill, rng, nugget = float(m[0]), float(m[1]), float(m[2])
    if model == "gaussian":      # :40-45
        return psill * (1.0 - np.exp(-(d**2.0) / (rng * 4.0 / 7.0) ** 2.0)) + nugget
    if model == "exponential":   # :48-53
        return psill * (1.0 - np.exp(-d / (rng / 3.0))) + nugget
    if model == "spherical":     # :56-70
        out = np.full(d.shape, psill + nugget)
        s = d <= rng
        out[s] = psill * ((3.0 * d[s]) / (2.0 * rng) - (d[s] ** 3.0) / (2.0 * rng**3.0)) + nugget
        return out
    if model == "hole-effect":   # :73-81
        return psill * (1.0 - (1.0 - d / (rng / 3.0)) * np.exp(-d / (rng / 3.0))) + nugget
    raise ValueError(model)


def stored_parameters(model, plist):
    """List input [FULL sill, range, nugget] -> stored [psill, range, nugget] (core.py:345-357)."""
    if model in ("gaussian", "spherical", "exponential", "hole-effect"):
        return [plist[0] - plist[2], plist[1], plist[2]]
    return list(plist)


# ---- geographic distances: core.py:36-97 -----------------------------------------------
def great_circle_distance(lon1, lat1, lon2, lat2):
    lat1 = np.array(lat1) * np.pi / 180.0
    lat2 = np.array(lat2) * np.pi / 180.0
    dlon = (lon1 - lon2) * np.pi / 180.0
    c1, s1, c2, s2, cd = np.cos(lat1), np.sin(lat1), np.cos(lat2), np.sin(lat2), np.cos(dlon)
    return 180.0 / np.pi * np.arctan2(np.sqrt((c2 * np.sin(dlon)) ** 2 + (c1 * s2 - s1 * c2 * cd) ** 2),
                                      s1 * s2 + c1 * c2 * cd)


def _unit_sphere(lonlat):
    """lon/lat degrees -> 3-D unit vectors, the kd-tree coordinates of ok.py:936-956."""
    lon = lonlat[:, 0] * np.pi / 180.0
    lat = lonlat[:, 1] * np.pi / 180.0
    return np.column_stack((np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)))


def krige_geographic(data_lonlat, values, model, plist_stored, points, *, exact_values=True, n_closest_points=None):
    """coordinates_type='geographic' (OrdinaryKriging only; ok.py:634-640, 930-969, 990-996): great-circle
    distances in degrees, no anisotropy; the moving window ranks neighbours by chord length on the unit
    sphere and then uses great-circle distances."""
    P = np.asarray(data_lonlat, dtype=np.float64)
    Q = np.asarray(points, dtype=np.float64)
    vals = np.asarray(values, dtype=np.float64)
    n = P.shape[0]
    def gmat(A, B):
        return great_circle_distance(A[:, 0][:, None], A[:, 1][:, None], B[:, 0][None, :], B[:, 1][None, :])
    if n_closest_points is None:
        a = np.zeros((n + 1, n + 1))
        a[:n, :n] = -variogram(model, plist_stored, gmat(P, P))
        np.fill_diagonal(a, 0.0)
        a[n, :n] = 1.0
        a[:n, n] = 1.0
        a_inv = scipy.linalg.inv(a)
        bd = gmat(Q, P)
        b = np.ones((Q.shape[0], n + 1))
        b[:, :n] = -variogram(model, plist_stored, bd)
        if exact_values:
            b[:, :n][np.absolute(bd) <= EPS] = 0.0
        x = a_inv @ b.T
        return x[:n, :].T @ vals, np.sum(x.T * -b, axis=1)
    k = n_closest_points
    tree = cKDTree(_unit_sphere(P))
    _, idx_all = tree.query(_unit_sphere(Q), k=k, eps=0.0)
    z = np.zeros(Q.shape[0])
    ss = np.zeros(Q.shape[0])
    for i in range(Q.shape[0]):
        sel = idx_all[i]
        S = P[sel]
        a = np.zeros((k + 1, k + 1))
        a[:k, :k] = -variogram(model, plist_stored, gmat(S, S))
        np.fill_diagonal(a, 0.0)
        a[k, :k] = 1.0
        a[:k, k] = 1.0
        bd = great_circle_distance(Q[i, 0], Q[i, 1], S[:, 0], S[:, 1])
        b = np.ones(k + 1)
        b[:k] = -variogram(model, plist_stored, bd)
        if exact_values:
            b[:k][np.absolute(bd) <= EPS] = 0.0
        x = scipy.linalg.solve(a, b)
        z[i] = x[:k].dot(vals[sel])
        ss[i] = -x.dot(b)
    return z, ss


# ---- anisotropy: core.py:120-193 -----------------------------------------------------
def adjust_for_anisotropy(X, center, scaling, angle):
    X = np.array(X, dtype=np.float64, copy=True)
    center = np.asarray(center, dtype=np.float64)[None, :]
    ang = np.asarray(angle, dtype=np.float64) * np.pi / 180.0
    X -= center
    nd = X.shape[1]
    if nd == 2:
        stretch = np.array([[1.0, 0.0], [0.0, scaling[0]]])
        rot = np.array([[np.cos(-ang[0]), -np.sin(-ang[0])], [np.sin(-ang[0]), np.cos(-ang[0])]])
    else:
        stretch = np.diag([1.0, scaling[0], scaling[1]])
        rx = np.array([[1, 0, 0], [0, np.cos(-ang[0]), -np.sin(-ang[0])], [0, np.sin(-ang[0]), np.cos(-ang[0])]])
        ry = np.array([[np.cos(-ang[1]), 0, np.sin(-ang[1])], [0, 1, 0], [-np.sin(-ang[1]), 0, np.cos(-ang[1])]])
        rz = np.array([[np.cos(-ang[2]), -np.sin(-ang[2]), 0], [np.sin(-ang[2]), np.cos(-ang[2]), 0], [0, 0, 1]])
        rot = rz @ (ry @ rx)
    return (stretch @ (rot @ X.T)).T + center


# ---- kriging matrix: ok.py:626-648, uk.py:861-920, ok3d.py:603-622, uk3d.py:688-737 ----
def kriging_matrix(P, model, m, drift_cols=()):
    """P: [n, dim] adjusted data coordinates; drift_cols: list of length-n arrays (in the
    reference's column order). Returns the (n+K+1)^2 matrix with the unbiasedness border."""
    n = P.shape[0]
    K = len(drift_cols)
    a = np.zeros((n + K + 1, n + K + 1))
    a[:n, :n] = -variogram(model, m, cdist(P, P, "euclidean"))
    np.fill_diagonal(a, 0.0)                      # ok.py:644
    for i, col in enumerate(drift_cols):          # uk.py:876-910
        a[:n, n + i] = col
        a[n + i, :n] = col
    a[n + K, :n] = 1.0                            # ok.py:645-647 / uk.py:915-918
    a[:n, n + K] = 1.0
    a[n:, n:] = 0.0
    return a


# ---- global solve: ok.py:650-683, uk.py:922-1009 --------------------------------------
def exec_vector(a, P, Q, values, model, m, exact_values=True, drift_pts=(), pseudo_inv=None):
    """Q: [npt, dim] adjusted prediction points; drift_pts: list of length-npt arrays.
    Returns (zvalues, sigmasq): inverse x RHS exactly as the reference's 'vectorized' backend."""
    n = P.shape[0]
    K = len(drift_pts)
    npt = Q.shape[0]
    if pseudo_inv:                                # ok.py:660-661: P_INV[pseudo_inv_type](a), core.py:33
        a_inv = {"pinv": scipy.linalg.pinv, "pinvh": scipy.linalg.pinvh}[pseudo_inv](a)
    else:
        a_inv = scipy.linalg.inv(a)               # ok.py:663
    bd = cdist(Q, P, "euclidean")                 # ok.py:989
    b = np.zeros((npt, n + K + 1))
    b[:, :n] = -variogram(model, m, bd)           # ok.py:670
    if exact_values:
        b[:, :n][np.absolute(bd) <= EPS] = 0.0    # ok.py:665-672
    for i, col in enumerate(drift_pts):           # uk.py:949-979
        b[:, n + i] = col
    b[:, n + K] = 1.0                             # ok.py:673
    x = a_inv @ b.T                               # ok.py:679
    z = np.sum(x[:n, :].T * values, axis=1)       # ok.py:680
    ss = np.sum(x.T * -b, axis=1)                 # ok.py:681
    return z, ss


def exec_vector_refined(a, P, Q, values, model, m, exact_values=True, drift_pts=(), bd=None, steps=3):
    """The exact solution of the system exec_vector solves: the same matrix `a` and the same RHS (exact-hit zeroing,
    drift columns, unbiasedness row; ok.py:665-681, uk.py:922-1009), solved to extended precision instead of through
    the fp64 inverse. One fp64 LU factorisation, then `steps` rounds of iterative refinement with the residual
    b - A x formed and x held in np.longdouble (64-bit mantissa on x86-64); z = x[:n].Z and sigma^2 = -x.b are summed
    in np.longdouble and rounded to fp64 once. The result carries about kappa * 1e-19 relative error instead of the
    kappa * eps of an fp64 solve, so it can judge kernels that are themselves accurate to ~1e-12.
    bd: [npt, n] data-to-point distances when they are not Euclidean (geographic great-circle degrees).
    Returns (zvalues, sigmasq, kappa_2(a))."""
    n = P.shape[0]
    K = len(drift_pts)
    npt = Q.shape[0]
    if bd is None:
        bd = cdist(Q, P, "euclidean")
    b = np.zeros((npt, n + K + 1))
    b[:, :n] = -variogram(model, m, bd)
    if exact_values:
        b[:, :n][np.absolute(bd) <= EPS] = 0.0
    for i, col in enumerate(drift_pts):
        b[:, n + i] = col
    b[:, n + K] = 1.0
    lu = scipy.linalg.lu_factor(a)
    A = a.astype(np.longdouble)
    B = b.T.astype(np.longdouble)
    x = scipy.linalg.lu_solve(lu, b.T).astype(np.longdouble)
    for _ in range(steps):
        r = B - A @ x
        x += scipy.linalg.lu_solve(lu, r.astype(np.float64)).astype(np.longdouble)
    z = (x[:n, :].T @ np.asarray(values, dtype=np.longdouble)).astype(np.float64)
    ss = (-np.sum(x * B, axis=0)).astype(np.float64)
    return z, ss, float(np.linalg.cond(a))


# ---- moving window: ok.py:722-758, 957-960; cok.pyx:98-193 -----------------------------
def exec_moving_window(P, Q, values, model, m, k, exact_values=True):
    """Never builds the N x N matrix (SURVEY F4): the local (k+1)^2 system is assembled from the
    neighbour coordinates, which is what gathering from the full matrix yields (cok.pyx:138-147)."""
    tree = cKDTree(P)
    bd_all, idx_all = tree.query(Q, k=k, eps=0.0)  # ok.py:957-960
    npt = Q.shape[0]
    z = np.zeros(npt)
    ss = np.zeros(npt)
    for i in range(npt):
        sel = idx_all[i]
        bd = bd_all[i]
        a = kriging_matrix(P[sel], model, m)       # == a_all[sel+[n]][:, sel+[n]] (ok.py:738-739)
        b = np.zeros(k + 1)
        b[:k] = -variogram(model, m, bd)
        if exact_values:
            b[:k][np.absolute(bd) <= EPS] = 0.0    # ok.py:741-751
        b[k] = 1.0
        x = scipy.linalg.solve(a, b)               # ok.py:753
        z[i] = x[:k].dot(values[sel])              # ok.py:755
        ss[i] = -x.dot(b)                          # ok.py:756
    return z, ss


# ---- point set-up: ok.py:862-885, ok3d.py:860-898 ---------------------------------------
def grid_points(axes):
    """2-D: meshgrid(x, y) flattened (x fastest, ok.py:864-866); 3-D: meshgrid(z, y, x, 'ij')
    flattened (ok3d.py:863-866). Returns [npt, dim] in (x, y[, z]) column order."""
    if len(axes) == 2:
        gx, gy = np.meshgrid(axes[0], axes[1])
        return np.column_stack((gx.ravel(), gy.ravel()))
    gz, gy, gx = np.meshgrid(axes[2], axes[1], axes[0], indexing="ij")
    return np.column_stack((gx.ravel(), gy.ravel(), gz.ravel()))


def krige(data_xyz, values, model, plist_stored, points, *, scaling=None, angle=None,
          regional_linear=False, data_drift=(), point_drift=(), exact_values=True, n_closest_points=None,
          pseudo_inv=None):
    """End-to-end oracle for one execute() call on explicit points (original coordinates).
    pseudo_inv: None | "pinv" | "pinvh" (ignored by the moving window, like ok.py:753).

    data_xyz [n, dim], points [npt, dim]; centre = (max+min)/2 of the data (ok.py:278-279);
    regional-linear drift uses the adjusted coordinates in x, y[, z] order (uk.py:877-883,
    uk3d.py:708-717, 767-773). data_drift / point_drift: extra host drift columns.
    """
    data_xyz = np.asarray(data_xyz, dtype=np.float64)
    points = np.asarray(points, dtype=np.float64)
    dim = data_xyz.shape[1]
    center = (data_xyz.max(axis=0) + data_xyz.min(axis=0)) / 2.0
    if scaling is None:
        scaling = [1.0] * (dim - 1)
    if angle is None:
        angle = [0.0] * (2 * dim - 3)
    P = adjust_for_anisotropy(data_xyz, center, scaling, angle)
    Q = adjust_for_anisotropy(points, center, scaling, angle)
    if n_closest_points is not None:
        return exec_moving_window(P, Q, np.asarray(values, float), model, plist_stored, n_closest_points, exact_values)
    dcols, pcols = [], []
    if regional_linear:
        for c in range(dim):
            dcols.append(P[:, c])
            pcols.append(Q[:, c])
    dcols += [np.asarray(c, float) for c in data_drift]
    pcols += [np.asarray(c, float) for c in point_drift]
    a = kriging_matrix(P, model, plist_stored, dcols)
    return exec_vector(a, P, Q, np.asarray(values, float), model, plist_stored, exact_values, pcols, pseudo_inv)


class PreparedKriging:
    """The reference's global path with the set-up (matrix + scipy.linalg.inv, ok.py:626-648,663) done once and
    the inverse x RHS step (ok.py:665-681) applied to any number of point slabs — what one execute() call does,
    cut so that M x N never materialises (SURVEY F3/F7). Used by krige_chunked and by bench.py's CPU arm."""

    def __init__(self, data_xyz, values, model, plist_stored, *, scaling=None, angle=None, regional_linear=False,
                 exact_values=True):
        data_xyz = np.asarray(data_xyz, dtype=np.float64)
        self.dim = data_xyz.shape[1]
        self.center = (data_xyz.max(axis=0) + data_xyz.min(axis=0)) / 2.0
        self.scaling = scaling or [1.0] * (self.dim - 1)
        self.angle = angle or [0.0] * (2 * self.dim - 3)
        self.exact = exact_values
        self.model, self.m = model, plist_stored
        self.P = adjust_for_anisotropy(data_xyz, self.center, self.scaling, self.angle)
        dcols = [self.P[:, c] for c in range(self.dim)] if regional_linear else []
        self.K = len(dcols)
        self.vals = np.asarray(values, float)
        self.a_inv = scipy.linalg.inv(kriging_matrix(self.P, model, plist_stored, dcols))

    def krige(self, points):
        n, K = self.P.shape[0], self.K
        Q = adjust_for_anisotropy(np.asarray(points, dtype=np.float64), self.center, self.scaling, self.angle)
        bd = cdist(Q, self.P, "euclidean")
        b = np.ones((Q.shape[0], n + K + 1))
        b[:, :n] = -variogram(self.model, self.m, bd)
        if self.exact:
            b[:, :n][np.absolute(bd) <= EPS] = 0.0
        for c in range(K):
            b[:, n + c] = Q[:, c]
        x = self.a_inv @ b.T
        return x[:n, :].T @ self.vals, -np.einsum("ij,ji->i", b, x)


def krige_chunked(data_xyz, values, model, plist_stored, points, chunk=20000, **kw):
    """Same as krige() for the global path but inverts once and streams the points in chunks, so
    large M never materialises M x N (SURVEY F3/F7). Used by bench.py's CPU baseline."""
    points = np.asarray(points, dtype=np.float64)
    pk = PreparedKriging(data_xyz, values, model, plist_stored, scaling=kw.get("scaling"), angle=kw.get("angle"),
                         regional_linear=bool(kw.get("regional_linear")), exact_values=kw.get("exact_values", True))
    z = np.empty(points.shape[0])
    ss = np.empty(points.shape[0])
    for s in range(0, points.shape[0], chunk):
        z[s:s + chunk], ss[s:s + chunk] = pk.krige(points[s:s + chunk])
    return z, ss


# ---- constructor side (SURVEY.md §8f next-2) ---------------------------------------------
def experimental_variogram(X, y, nlags, coordinates_type="euclidean"):
    """Binned experimental semivariogram, core.py:432-505: every pair's distance and half squared
    value difference, nlags equal-width bins from dmin to dmax (last edge dmax + 0.001), per-bin means,
    empty bins dropped. Materialises the full pair list like the reference does (small cases only)."""
    from scipy.spatial.distance import pdist

    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if coordinates_type == "euclidean":              # core.py:432-434
        d = pdist(X, metric="euclidean")
        g = 0.5 * pdist(y[:, None], metric="sqeuclidean")
    elif coordinates_type == "geographic":           # core.py:440-453 (strict lower triangle)
        if X.shape[1] != 2:
            raise ValueError("Geographic coordinate type only supported for 2D datasets.")
        D = great_circle_distance(X[:, 0][None, :], X[:, 1][None, :], X[:, 0][:, None], X[:, 1][:, None])
        G = 0.5 * (y[None, :] - y[:, None]) ** 2.0
        low = np.tril(np.ones(D.shape, dtype=bool), -1)
        d, g = D[low], G[low]
    else:
        raise ValueError("Specified coordinate type '%s' is not supported." % coordinates_type)
    dmax, dmin = np.amax(d), np.amin(d)              # core.py:471-476
    dd = (dmax - dmin) / nlags
    bins = [dmin + n * dd for n in range(nlags)]
    bins.append(dmax + 0.001)
    lags, semi = [], []
    for n in range(nlags):                           # core.py:493-505
        sel = (d >= bins[n]) & (d < bins[n + 1])
        if np.any(sel):
            lags.append(np.mean(d[sel]))
            semi.append(np.mean(g[sel]))
    return np.array(lags), np.array(semi)


def krige_one(X, y, coords, model, m, coordinates_type="euclidean"):
    """core._krige, core.py:654-756: one ordinary-kriging estimate and variance at `coords`."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    if coordinates_type == "euclidean":
        d = cdist(X, X)
        bd = cdist(X, np.asarray(coords, dtype=np.float64)[None, :]).ravel()
    else:
        d = great_circle_distance(X[:, 0][None, :], X[:, 1][None, :], X[:, 0][:, None], X[:, 1][:, None])
        bd = great_circle_distance(X[:, 0], X[:, 1], coords[0] * np.ones(n), coords[1] * np.ones(n))
    a = np.zeros((n + 1, n + 1))
    a[:n, :n] = -variogram(model, m, d)
    np.fill_diagonal(a, 0.0)
    a[n, :] = 1.0
    a[:, n] = 1.0
    a[n, n] = 0.0
    b = np.zeros(n + 1)
    b[:n] = -variogram(model, m, bd)
    if np.any(np.absolute(bd) <= 1e-10):             # core.py:729-731, 748-749
        b[int(np.flatnonzero(bd <= 1e-10)[0])] = 0.0
    b[n] = 1.0
    res = np.linalg.solve(a, b)
    return float(np.sum(res[:n] * y)), float(np.sum(res * -b))


def find_statistics(X, y, model, m, coordinates_type="euclidean"):
    """core._find_statistics, core.py:759-836: point i kriged from points [0, i); near-zero variances
    are skipped. Returns (delta, sigma, epsilon)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    delta = np.zeros(y.shape)
    sigma = np.zeros(y.shape)
    for i in range(1, y.shape[0]):
        k, ss = krige_one(X[:i, :], y[:i], X[i, :], model, m, coordinates_type)
        if np.absolute(ss) < EPS:
            continue
        delta[i] = y[i] - k
        sigma[i] = np.sqrt(ss)
    keep = sigma > EPS
    delta, sigma = delta[keep], sigma[keep]
    return delta, sigma, delta / sigma
