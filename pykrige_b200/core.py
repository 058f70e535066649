"""Host-side helpers of the H100 kriging backend (numpy/scipy, constructor-time only).

Mirrors the behaviour of the reference's ``src/pykrige/core.py`` for the pieces the
kriging classes need around ``execute()``; none of this is on the hot path:

* anisotropy affine map                      core.py:120-193
* variogram parameter normalisation          core.py:196-376  (list form = FULL sill -> psill)
* experimental variogram + model fit         core.py:379-651
* cross-validation statistics (lazy here)    core.py:654-851
"""
import numpy as np
from scipy.optimize import least_squares
from scipy.spatial.distance import pdist

eps = 1.0e-10

_BOUNDED = ("gaussian", "spherical", "exponential", "hole-effect")


def great_circle_distance(lon1, lat1, lon2, lat2):
    """Great-circle distance in DEGREES between points given as lon/lat degrees, numpy broadcasting
    semantics (core.py:36-97: the arctan form, stable for small and near-antipodal separations)."""
    lat1 = np.asarray(lat1, dtype=float) * np.pi / 180.0
    lat2 = np.asarray(lat2, dtype=float) * np.pi / 180.0
    dlon = (np.asarray(lon1, dtype=float) - np.asarray(lon2, dtype=float)) * np.pi / 180.0
    c1, s1, c2, s2, cd = np.cos(lat1), np.sin(lat1), np.cos(lat2), np.sin(lat2), np.cos(dlon)
    num = np.sqrt((c2 * np.sin(dlon)) ** 2 + (c1 * s2 - s1 * c2 * cd) ** 2)
    return 180.0 / np.pi * np.arctan2(num, s1 * s2 + c1 * c2 * cd)


def euclid3_to_great_circle(euclid3_distance):
    """Chord length on the unit sphere -> great-circle distance in degrees (core.py:100-117)."""
    e = np.minimum(np.asarray(euclid3_distance, dtype=float), 2.0)
    return 180.0 - 360.0 / np.pi * np.arccos(0.5 * e)


def anisotropy_matrix(ndim, scaling, angle):
    """Return Mt = stretch @ rot (ndim x ndim) of the reference's anisotropy map.

    2-D: rot = R(-angle), stretch = diag(1, s).  3-D: rot = Rz @ Ry @ Rx (each by the
    negated angle), stretch = diag(1, s_y, s_z).  (core.py:148-189)
    """
    rot, stretch = _rotation_and_stretch(ndim, scaling, angle)
    return stretch @ rot


def _rotation_and_stretch(ndim, scaling, angle):
    """(rot, stretch) of the reference's anisotropy map, see anisotropy_matrix."""
    ang = -np.asarray(angle, dtype=float) * np.pi / 180.0
    if ndim == 2:
        c, s = np.cos(ang[0]), np.sin(ang[0])
        return np.array([[c, -s], [s, c]]), np.diag([1.0, float(scaling[0])])
    if ndim == 3:
        cx, sx = np.cos(ang[0]), np.sin(ang[0])
        cy, sy = np.cos(ang[1]), np.sin(ang[1])
        cz, sz = np.cos(ang[2]), np.sin(ang[2])
        rx = np.array([[1.0, 0.0, 0.0], [0.0, cx, -sx], [0.0, sx, cx]])
        ry = np.array([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]])
        rz = np.array([[cz, -sz, 0.0], [sz, cz, 0.0], [0.0, 0.0, 1.0]])
        return np.dot(rz, np.dot(ry, rx)), np.diag([1.0, float(scaling[0]), float(scaling[1])])
    if ndim == 1:
        raise NotImplementedError("1-D anisotropy is not implemented")
    raise ValueError("anisotropy adjustment supports 2-D and 3-D only")


def _adjust_for_anisotropy(X, center, scaling, angle):
    """X_adj = stretch (rot (X - c)) + c   (core.py:120-193).  X is [n, ndim]; not modified.
    Rotation first, stretch second, as two products — the association the reference uses, so that X_ADJUSTED (and
    with it the experimental variogram and the automatic fit) carries the same bits; the device applies the
    pre-multiplied matrix of anisotropy_matrix (csrc/common.cuh kb_adjust), which is inside the parity tolerance."""
    X = np.asarray(X, dtype=float)
    c = np.asarray(center, dtype=float)[None, :]
    rot, stretch = _rotation_and_stretch(X.shape[1], scaling, angle)
    return np.dot(stretch, np.dot(rot, (X - c).T)).T + c


def _make_variogram_parameter_list(variogram_model, variogram_model_parameters):
    """User parameters (None | dict | list) -> stored list (core.py:196-376).

    linear [slope, nugget]; power [scale, exponent, nugget]; bounded models
    [psill, range, nugget] — a *list* gives the FULL sill first (core.py:345-357), a dict
    may give either 'sill' or 'psill' (core.py:286-299).
    """
    p = variogram_model_parameters
    if p is None:
        return None
    known = ("linear", "power") + _BOUNDED + ("custom",)
    if variogram_model not in known:
        raise ValueError(
            "Specified variogram model must be one of the following: 'linear', 'power', "
            "'gaussian', 'spherical', 'exponential', 'hole-effect', 'custom'."
        )
    if type(p) is dict:
        if variogram_model == "custom":
            raise TypeError("For user-specified custom variogram model, parameters must be specified in a list, not a dict.")
        if variogram_model == "linear":
            if "slope" not in p or "nugget" not in p:
                raise KeyError("'linear' variogram model requires 'slope' and 'nugget' specified in variogram model parameter dictionary.")
            return [p["slope"], p["nugget"]]
        if variogram_model == "power":
            if "scale" not in p or "exponent" not in p or "nugget" not in p:
                raise KeyError("'power' variogram model requires 'scale', 'exponent', and 'nugget' specified in variogram model parameter dictionary.")
            return [p["scale"], p["exponent"], p["nugget"]]
        if "range" not in p or "nugget" not in p:
            raise KeyError("'%s' variogram model requires 'range', 'nugget', and either 'sill' or 'psill' specified in variogram model parameter dictionary." % variogram_model)
        if "sill" in p:
            return [p["sill"] - p["nugget"], p["range"], p["nugget"]]
        if "psill" in p:
            return [p["psill"], p["range"], p["nugget"]]
        raise KeyError("'%s' variogram model requires either 'sill' or 'psill' specified in variogram model parameter dictionary." % variogram_model)
    if type(p) is list:
        if variogram_model == "custom":
            return p
        want = 2 if variogram_model == "linear" else 3
        if len(p) != want:
            raise ValueError(
                "Variogram model parameter list must have exactly %s entries when variogram model set to '%s'."
                % ("two" if want == 2 else "three", variogram_model)
            )
        if variogram_model in _BOUNDED:
            return [p[0] - p[2], p[1], p[2]]
        return p
    raise TypeError("Variogram model parameters must be provided in either a list or a dict when they are explicitly specified.")


def _device_available():
    from . import _cabi
    return _cabi.device_available()


def _pair_distances(XA, XB, coordinates_type):
    if coordinates_type == "geographic":
        return great_circle_distance(XA[:, 0][:, None], XA[:, 1][:, None], XB[:, 0][None, :], XB[:, 1][None, :])
    from scipy.spatial.distance import cdist
    return cdist(XA, XB)


def _experimental_variogram(X, y, nlags, block=2048, coordinates_type="euclidean", device="auto"):
    """Equal-width binned semivariogram (core.py:432-505).

    Same bins as the reference (nlags equal bins from dmin to dmax, last edge dmax + 0.001; lag = mean
    distance and semivariance = mean 0.5*(dy)^2 of the pairs in the bin; empty bins dropped).
    device=True / "auto" with a CUDA device: the pair pass runs on the GPU
    (kb200_experimental_variogram, csrc/variogram.cu — 5e9 pairs at N = 1e5 in well under a second).
    device=False / "auto" without a device: host numpy accumulated over row blocks, so that the O(N^2)
    pair list never exists (the reference's pdist needs 80 GB at N = 1e5)."""
    n = X.shape[0]
    if coordinates_type == "geographic" and X.shape[1] != 2:
        raise ValueError("Geographic coordinate type only supported for 2D datasets.")
    small = n * (n - 1) // 2 <= 20_000_000
    # "auto": the pdist route below reproduces the reference's lags bit for bit (same summation order), which the
    # least-squares fit needs; it is cheap up to ~6300 points. Beyond that only the device can hold the pair pass.
    if device is True or (device == "auto" and n >= 2 and not small and _device_available()):
        from . import _cabi
        cnt, sd, sg, _, _ = _cabi.aux_handle().experimental_variogram(
            X, y, nlags, geographic=(coordinates_type == "geographic"))
        keep = cnt > 0
        return sd[keep] / cnt[keep], sg[keep] / cnt[keep]
    if small:
        if coordinates_type == "geographic":
            # the reference's pair list (core.py:444-451): strictly-lower-triangle pairs (i > j) in row-major order,
            # point j in the first argument slot of the (bitwise asymmetric) great-circle formula
            i, j = np.tril_indices(n, -1)
            d = great_circle_distance(X[j, 0], X[j, 1], X[i, 0], X[i, 1])
            g = 0.5 * (y[j] - y[i]) ** 2.0
        else:
            d = pdist(X, metric="euclidean")
            g = 0.5 * pdist(y[:, None], metric="sqeuclidean")
        dmax, dmin = np.amax(d), np.amin(d)
        dd = (dmax - dmin) / nlags
        edges = np.array([dmin + k * dd for k in range(nlags)] + [dmax + 0.001])
        # per-bin np.mean over the selected pairs, exactly the reference's expression (core.py:493-505): the same
        # pairwise summation order, so that the least-squares fit (which amplifies 1e-14 differences of the lags
        # to ~1e-4 in the fitted parameters) starts from bit-identical inputs
        lags, semi = [], []
        for k in range(nlags):
            sel = (d >= edges[k]) & (d < edges[k + 1])
            if np.any(sel):
                lags.append(np.mean(d[sel]))
                semi.append(np.mean(g[sel]))
        return np.array(lags), np.array(semi)
    else:
        dmin, dmax = np.inf, 0.0
        for s in range(0, n, block):
            D = _pair_distances(X[s:s + block], X[s:], coordinates_type)
            iu = np.triu_indices(D.shape[0], 1, D.shape[1])
            dv = D[iu]
            if dv.size:
                dmin, dmax = min(dmin, dv.min()), max(dmax, dv.max())
        dd = (dmax - dmin) / nlags
        edges = np.array([dmin + k * dd for k in range(nlags)] + [dmax + 0.001])
        cnt = np.zeros(nlags)
        sd = np.zeros(nlags)
        sg = np.zeros(nlags)
        for s in range(0, n, block):
            D = _pair_distances(X[s:s + block], X[s:], coordinates_type)
            iu = np.triu_indices(D.shape[0], 1, D.shape[1])
            dv = D[iu]
            gv = 0.5 * (y[s:s + block, None] - y[None, s:])[iu] ** 2
            which = np.searchsorted(edges, dv, side="right") - 1
            ok = (which >= 0) & (which < nlags)
            cnt += np.bincount(which[ok], minlength=nlags)
            sd += np.bincount(which[ok], weights=dv[ok], minlength=nlags)
            sg += np.bincount(which[ok], weights=gv[ok], minlength=nlags)
    keep = cnt > 0
    return sd[keep] / cnt[keep], sg[keep] / cnt[keep]


def _variogram_residuals(params, x, y, variogram_function, weight):
    """Residuals for the fit, with the reference's optional logistic lag weights (core.py:538-579)."""
    if weight:
        drange = np.amax(x) - np.amin(x)
        k = 2.1972 / (0.1 * drange)
        x0 = 0.7 * drange + np.amin(x)
        w = 1.0 / (1.0 + np.exp(-k * (x0 - x)))
        w /= np.sum(w)
        return (variogram_function(params, x) - y) * w
    return variogram_function(params, x) - y


def _calculate_variogram_model(lags, semivariance, variogram_model, variogram_function, weight):
    """soft-L1 least squares with the reference's start values and bounds (core.py:582-651)."""
    smax, smin = np.amax(semivariance), np.amin(semivariance)
    lmax, lmin = np.amax(lags), np.amin(lags)
    if variogram_model == "linear":
        x0 = [(smax - smin) / (lmax - lmin), smin]
        bnds = ([0.0, 0.0], [np.inf, smax])
    elif variogram_model == "power":
        x0 = [(smax - smin) / (lmax - lmin), 1.1, smin]
        bnds = ([0.0, 0.001, 0.0], [np.inf, 1.999, smax])
    else:
        x0 = [smax - smin, 0.25 * lmax, smin]
        bnds = ([0.0, 0.0, 0.0], [10.0 * smax, lmax, smax])
    res = least_squares(
        _variogram_residuals, x0, bounds=bnds, loss="soft_l1",
        args=(lags, semivariance, variogram_function, weight),
    )
    return res.x


def _initialize_variogram_model(X, y, variogram_model, variogram_model_parameters,
                                variogram_function, nlags, weight, coordinates_type, lazy=False):
    """Returns (lags, semivariance, parameters) (core.py:379-535). With lazy=True and explicit
    parameters the experimental variogram (an O(N^2) pass that execute() never needs) is returned as
    a zero-argument callable instead of arrays."""
    if coordinates_type not in ("euclidean", "geographic"):
        raise ValueError("Specified coordinate type '%s' is not supported." % coordinates_type)
    p = variogram_model_parameters
    deferred = None
    if lazy and p is not None:
        def deferred():
            return (_experimental_variogram(X, y, nlags, coordinates_type=coordinates_type)
                    if X.shape[0] > 1 else (np.zeros(0), np.zeros(0)))
        lags, semivariance = None, None
    elif X.shape[0] > 1:
        lags, semivariance = _experimental_variogram(X, y, nlags, coordinates_type=coordinates_type)
    else:
        lags, semivariance = np.zeros(0), np.zeros(0)
    if p is not None:
        if variogram_model == "linear" and len(p) != 2:
            raise ValueError("Exactly two parameters required for linear variogram model.")
        if variogram_model in ("power",) + _BOUNDED and len(p) != 3:
            raise ValueError("Exactly three parameters required for %s variogram model" % variogram_model)
    else:
        if variogram_model == "custom":
            raise ValueError("Variogram parameters must be specified when implementing custom variogram model.")
        p = _calculate_variogram_model(lags, semivariance, variogram_model, variogram_function, weight)
    if deferred is not None:
        return deferred, None, p
    return lags, semivariance, p


def _krige(X, y, coords, variogram_function, variogram_model_parameters, coordinates_type="euclidean",
           pseudo_inv=False):
    """One ordinary-kriging estimate at ``coords`` from data (X, y) (core.py:654-756); host numpy, used by the
    cross-validation statistics when there is no device route. Same numerical primitives as the reference
    (pdist/cdist distances, numpy's gesv / gelsd drivers on an (n+1, 1) right-hand side, only the FIRST coincident
    data point zeroed), so that delta / sigma / epsilon carry the reference's bits."""
    from scipy.spatial.distance import cdist, squareform

    n = X.shape[0]
    coords = np.asarray(coords, dtype=float)
    if coordinates_type == "geographic":
        # d[i, j]: point j in the first argument slot of the (bitwise asymmetric) great-circle formula (core.py:689-691)
        d = great_circle_distance(X[None, :, 0], X[None, :, 1], X[:, 0, None], X[:, 1, None])
        bd = great_circle_distance(X[:, 0], X[:, 1], coords[0] * np.ones(n), coords[1] * np.ones(n))
    elif coordinates_type == "euclidean":
        d = squareform(pdist(X, metric="euclidean"))
        bd = cdist(X, coords[None, :], metric="euclidean").ravel()
    else:
        raise ValueError("Specified coordinate type '%s' is not supported." % coordinates_type)
    a = np.zeros((n + 1, n + 1))
    a[:n, :n] = -variogram_function(variogram_model_parameters, d)
    np.fill_diagonal(a, 0.0)
    a[n, :n] = 1.0
    a[:n, n] = 1.0
    b = np.zeros((n + 1, 1))
    b[:n, 0] = -variogram_function(variogram_model_parameters, bd)
    if np.any(np.absolute(bd) <= 1e-10):
        b[int(np.flatnonzero(bd <= 1e-10)[0]), 0] = 0.0
    b[n, 0] = 1.0
    res = np.linalg.lstsq(a, b, rcond=None)[0] if pseudo_inv else np.linalg.solve(a, b)
    return np.sum(res[:n, 0] * y), np.sum(res[:, 0] * -b[:, 0])


def _find_statistics(X, y, variogram_function, variogram_model_parameters, coordinates_type="euclidean",
                     pseudo_inv=False):
    """Sequential cross-validation residuals (core.py:759-836): delta, sigma, epsilon."""
    n = y.shape[0]
    delta = np.zeros(n)
    sigma = np.zeros(n)
    for i in range(1, n):                 # the first point has nothing to be estimated from
        k, ss = _krige(X[:i, :], y[:i], X[i, :], variogram_function, variogram_model_parameters,
                       coordinates_type, pseudo_inv)
        if np.absolute(ss) < eps:
            continue
        delta[i] = y[i] - k
        sigma[i] = np.sqrt(ss)
    delta = delta[sigma > eps]
    sigma = sigma[sigma > eps]
    return delta, sigma, delta / sigma


def calcQ1(epsilon):
    """core.py:839-841"""
    return abs(np.sum(epsilon) / (epsilon.shape[0] - 1))


def calcQ2(epsilon):
    """core.py:844-846"""
    return np.sum(epsilon**2) / (epsilon.shape[0] - 1)


def calc_cR(Q2, sigma):
    """core.py:849-851"""
    return Q2 * np.exp(np.sum(np.log(sigma**2)) / sigma.shape[0])
