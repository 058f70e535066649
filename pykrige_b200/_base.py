"""Shared host logic of the four kriging classes (not part of the reference's API surface).

The reference repeats this logic in ok.py / uk.py / ok3d.py / uk3d.py; here it lives once:
variogram model selection (ok.py:208-253), the ``backend='cuda'`` dispatch that replaces the
``backend`` string switch of ``execute`` (ok.py:971-1010), point-list / grid / mask handling
(ok.py:842-900, ok3d.py:833-898) and output shaping (ok.py:1012-1020).
"""
import warnings
import numpy as np

from . import variogram_models
from . import core
from . import _cabi


class KrigeBase:
    eps = 1.0e-10  # cutoff for comparison to zero (ok.py:177)
    variogram_dict = {
        "linear": variogram_models.linear_variogram_model,
        "power": variogram_models.power_variogram_model,
        "gaussian": variogram_models.gaussian_variogram_model,
        "spherical": variogram_models.spherical_variogram_model,
        "exponential": variogram_models.exponential_variogram_model,
        "hole-effect": variogram_models.hole_effect_variogram_model,
    }
    _ndim = 2

    # ---- variogram model selection (ok.py:208-253; GSTools models arrive as 'custom') ----
    def _select_variogram(self, variogram_model, variogram_function, gstools_dim_ok):
        self.variogram_model = variogram_model
        self.model = None
        overrides = {}
        if hasattr(self.variogram_model, "pykrige_kwargs"):
            self.model = self.variogram_model
            gstools_dim_ok(self.model)
            self.variogram_model = "custom"
            variogram_function = self.model.pykrige_vario
            overrides["variogram_parameters"] = []
            overrides["gstools"] = self.model
        if self.variogram_model not in self.variogram_dict.keys() and self.variogram_model != "custom":
            raise ValueError("Specified variogram model '%s' is not supported." % variogram_model)
        elif self.variogram_model == "custom":
            if variogram_function is None or not callable(variogram_function):
                raise ValueError("Must specify callable function for custom variogram model.")
            self.variogram_function = variogram_function
        else:
            self.variogram_function = self.variogram_dict[self.variogram_model]
        return overrides

    def _print_variogram(self):
        p = self.variogram_model_parameters
        if self.variogram_model == "linear":
            print("Using '%s' Variogram Model" % "linear")
            print("Slope:", p[0])
            print("Nugget:", p[1], "\n")
        elif self.variogram_model == "power":
            print("Using '%s' Variogram Model" % "power")
            print("Scale:", p[0])
            print("Exponent:", p[1])
            print("Nugget:", p[2], "\n")
        elif self.variogram_model == "custom":
            print("Using Custom Variogram Model")
        else:
            print("Using '%s' Variogram Model" % self.variogram_model)
            print("Partial Sill:", p[0])
            print("Full Sill:", p[0] + p[2])
            print("Range:", p[1])
            print("Nugget:", p[2], "\n")

    # ---- experimental variogram: computed on first access when the parameters were given explicitly
    #      (the reference always runs the O(N^2) pdist in the constructor, core.py:432-436) -------------
    def _get_lags(self):
        if callable(self._lags):
            self._lags, self._semivariance = self._lags()
        return self._lags

    def _set_lags(self, v):
        self._lags = v

    def _get_semivariance(self):
        self._get_lags()
        return self._semivariance

    def _set_semivariance(self, v):
        if v is not None or not callable(getattr(self, "_lags", None)):
            self._semivariance = v

    lags = property(_get_lags, _set_lags)
    semivariance = property(_get_semivariance, _set_semivariance)

    # ---- cross-validation statistics: lazy (the reference runs this O(N^4) loop in the
    #      constructor of OK3D/UK/UK3D, ok3d.py:352, uk.py:380, uk3d.py:380; SURVEY F5) -----
    def _stats_inputs(self):
        raise NotImplementedError

    def _device_statistics(self):
        """delta, sigma, epsilon from the Cholesky factor of the device problem (kb200_statistics,
        csrc/variogram.cu: O(N) after the factorisation instead of the reference's N solves). Returns
        None when this problem has no device twin (custom variogram, pseudo_inv, indefinite
        covariance form, no CUDA device) — the caller then runs the reference's loop on the host."""
        if not _cabi.device_available() or getattr(self, "pseudo_inv", False):
            return None                          # core._krige solves with lstsq under pseudo_inv (core.py:749-750)
        try:
            key = getattr(self, "_kb_key", None)
            if key is not None and key[1] is False and key == self._problem_signature(key[0], False):
                h = self._cuda_handle()           # the factor of the last global execute() is still there
            else:
                h = self._ensure_problem("float64")
            delta, sigma = h.statistics(len(self._stats_inputs()[1]))
        except (NotImplementedError, _cabi.KrigeB200Error, np.linalg.LinAlgError, ValueError, MemoryError):
            return None
        keep = (sigma * sigma >= core.eps) & (sigma > core.eps)      # core.py:818-819, 829-831
        delta, sigma = delta[keep], sigma[keep]
        return delta, sigma, delta / sigma

    def _compute_statistics(self, device="auto"):
        X, y = self._stats_inputs()
        res = self._device_statistics() if device in ("auto", True) else None
        if res is None:
            if device is True:
                raise _cabi.KrigeB200Error("cross-validation statistics: this problem has no device route")
            res = core._find_statistics(
                X, y, self.variogram_function, self.variogram_model_parameters,
                getattr(self, "coordinates_type", "euclidean"), getattr(self, "pseudo_inv", False),
            )
        self._delta, self._sigma, self._epsilon = res
        self._Q1 = core.calcQ1(self._epsilon)
        self._Q2 = core.calcQ2(self._epsilon)
        self._cR = core.calc_cR(self._Q2, self._sigma)
        self._stats_state = "done"

    def _statistics_policy(self, policy):
        """End of the constructors / update_variogram_model. policy 'off' (OrdinaryKriging without enable_statistics:
        every statistic is None), 'eager' (enable_statistics=True) or 'lazy' (the other three classes and every
        update_variogram_model: the reference computes the statistics right here, ok3d.py:352, uk.py:380, uk3d.py:380,
        ok.py:539 — an O(N^4) loop, SURVEY F5; here they are computed on first access). verbose=True prints what the
        reference prints at this point (ok.py:358-375), which for 'lazy' means computing them now."""
        if self.verbose:
            print("Calculating statistics on variogram model fit...")
        self._stats_state = "lazy" if policy == "eager" else policy
        if policy == "eager" or (policy == "lazy" and self.verbose):
            self._compute_statistics()
            if self.verbose:
                print("Q1 =", self.Q1)
                print("Q2 =", self.Q2)
                print("cR =", self.cR, "\n")

    def _stat(self, name):
        state = getattr(self, "_stats_state", "off")
        if state == "off":
            return None
        if state == "lazy":
            self._compute_statistics()
        return getattr(self, "_" + name)

    delta = property(lambda self: self._stat("delta"))
    sigma = property(lambda self: self._stat("sigma"))
    epsilon = property(lambda self: self._stat("epsilon"))
    Q1 = property(lambda self: self._stat("Q1"))
    Q2 = property(lambda self: self._stat("Q2"))
    cR = property(lambda self: self._stat("cR"))

    # ---- small public helpers kept from the reference API (ok.py:555-624) ---------------
    def display_variogram_model(self):
        """Displays variogram model with the actual binned data."""
        import matplotlib.pyplot as plt

        fig = plt.figure()
        ax = fig.add_subplot(111)
        ax.plot(self.lags, self.semivariance, "r*")
        ax.plot(self.lags, self.variogram_function(self.variogram_model_parameters, self.lags), "k-")
        plt.show()

    def get_variogram_points(self):
        """Returns both the lags and the variogram function evaluated at each of them."""
        return self.lags, self.variogram_function(self.variogram_model_parameters, self.lags)

    def switch_verbose(self):
        self.verbose = not self.verbose

    def switch_plotting(self):
        self.enable_plotting = not self.enable_plotting

    def get_epsilon_residuals(self):
        return self.epsilon

    def plot_epsilon_residuals(self):
        import matplotlib.pyplot as plt

        fig = plt.figure()
        ax = fig.add_subplot(111)
        ax.scatter(range(self.epsilon.size), self.epsilon, c="k", marker="*")
        ax.axhline(y=0.0)
        plt.show()

    def get_statistics(self):
        return self.Q1, self.Q2, self.cR

    def print_statistics(self):
        print("Q1 =", self.Q1)
        print("Q2 =", self.Q2)
        print("cR =", self.cR)

    # ---- the backend='cuda' arm ---------------------------------------------------------
    TABLE_MODEL_ID = 6          # KB200_VG_TABLE
    TABLE_NODES = (1 << 20) + 1

    def _device_model(self):
        """model id + stored parameters for the device. Built-in models run as closed forms; a 'custom'
        callable or a GSTools model (which the reference's native 'C' backend refuses,
        variogram_models.pyx:20-21) is tabulated by the host and interpolated on the device
        (KB200_VG_TABLE, include/krige_b200.h: kb200_set_variogram_table)."""
        name = getattr(self.variogram_function, "__name__", None)
        mid = variogram_models.DEVICE_MODEL_IDS.get(name)
        if mid is None or self.variogram_function is not self.variogram_dict.get(self.variogram_model):
            if not callable(self.variogram_function):
                raise NotImplementedError("backend='cuda' needs a built-in variogram model or a callable f(params, d)")
            return self.TABLE_MODEL_ID, []
        return mid, [float(v) for v in self.variogram_model_parameters]

    def _adjusted_corners(self, lo, hi):
        """Corners of the axis-aligned box [lo, hi] (original coordinates) in the adjusted frame."""
        nd = self._ndim
        x, y, z, v, center, Mt = self._data_arrays()
        Mt = np.asarray(Mt, dtype=float).reshape(nd, nd)
        c = np.asarray(center, dtype=float)
        corners = np.array(np.meshgrid(*[[lo[k], hi[k]] for k in range(nd)], indexing="ij")).reshape(nd, -1).T
        return (corners - c) @ Mt.T + c

    def _table_dmax(self, pred_lo=None, pred_hi=None):
        """Upper bound of every distance the device will evaluate: data-data and data-prediction (the
        distance between two boxes is largest at a pair of corners; the affine anisotropy map keeps them
        corners), with head-room for the moving window's local shift gamma(2 d_k)."""
        if getattr(self, "coordinates_type", "euclidean") == "geographic":
            return 360.0
        x, y, z = self._data_arrays()[:3]
        cols = [x, y] + ([z] if self._ndim == 3 else [])
        dlo = [float(np.min(c)) for c in cols]
        dhi = [float(np.max(c)) for c in cols]
        D = self._adjusted_corners(dlo, dhi)
        pts = D if pred_lo is None else np.vstack([D, self._adjusted_corners(pred_lo, pred_hi)])
        span = np.sqrt(((pts[:, None, :] - D[None, :, :]) ** 2).sum(axis=2)).max()
        need = 2.2 * max(float(span), 1e-300)
        have = getattr(self, "_kb_table_dmax", 0.0)
        if need > have:                       # grow geometrically so that moving prediction windows do not re-tabulate
            self._kb_table_dmax = need if have == 0.0 else max(need, 2.0 * have)
        return self._kb_table_dmax

    def _variogram_table(self, dmax):
        """gamma at the sqrt-spaced nodes d_i = dmax (i/(n-1))^2, cached per (callable, parameters, dmax)."""
        key = (id(self.variogram_function), tuple(np.ravel(np.asarray(self.variogram_model_parameters, dtype=float))),
               float(dmax))
        cached = getattr(self, "_kb_table", None)
        if cached is not None and cached[0] == key:
            return cached[1]
        n = self.TABLE_NODES
        d = dmax * (np.arange(n, dtype=np.float64) / (n - 1)) ** 2
        with np.errstate(all="ignore"):
            g = np.asarray(self.variogram_function(self.variogram_model_parameters, d), dtype=np.float64)
        if g.shape != d.shape:
            g = np.broadcast_to(g, d.shape).copy()
        if not np.all(np.isfinite(g)):
            raise ValueError("the custom variogram function must be finite on [0, %g]" % dmax)
        self._kb_table = (key, g)
        return g

    def _data_arrays(self):
        """(x, y, z|None, values, center, Mt) in ORIGINAL coordinates."""
        raise NotImplementedError

    def _drift_spec(self):
        """(n_rl, [host drift data columns])"""
        return 0, []

    def _cuda_handle(self, n_gpus=None):
        """The C-ABI executor of this model: one kb200 handle (default) or, for n_gpus > 1, a kb200_group of
        handles on devices 0..n_gpus-1 driven by this host thread."""
        if n_gpus is not None and int(n_gpus) > 1:
            g = getattr(self, "_kb_group", None)
            if g is None or g.size != int(n_gpus):
                if g is not None:
                    g.close()
                g = _cabi.Group(int(n_gpus))
                self._kb_group = g
                self._kb_gkey = None
            return g
        h = getattr(self, "_kb_handle", None)
        if h is None:
            h = _cabi.Handle()
            self._kb_handle = h
            self._kb_key = None
        return h

    def _content_digest(self):
        """Cheap content hash of everything the device problem is built from (coordinates, values, host drift
        columns), so that in-place edits of the data arrays invalidate the cached factorisation."""
        import hashlib
        x, y, z, v, center, Mt = self._data_arrays()
        n_rl, cols = self._drift_spec()
        hsh = hashlib.blake2b(digest_size=16)
        for a in (x, y, z, v) + tuple(cols):
            if a is not None:
                hsh.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
        return hsh.hexdigest()

    def _problem_signature(self, dtype, knn, fields=None):
        x, y, z, v, center, Mt = self._data_arrays()
        mid, vp = self._device_model()
        n_rl, cols = self._drift_spec()
        if mid == self.TABLE_MODEL_ID:      # the table itself is part of the problem
            vp = ("table", id(self.variogram_function), getattr(self, "_kb_table_dmax", 0.0)) + tuple(
                np.ravel(np.asarray(self.variogram_model_parameters, dtype=float)))
        return (dtype, knn, mid, tuple(vp), bool(self.exact_values), tuple(np.ravel(Mt)), tuple(center),
                n_rl, len(cols), x.size, getattr(self, "coordinates_type", "euclidean"),
                bool(getattr(self, "pseudo_inv", False)), self._device_drift_signature(), self._content_digest(),
                self._fields_signature(fields))

    @staticmethod
    def _fields_signature(fields):
        """(V, digest) of the value fields a problem kriges instead of the constructor's values; (0, None) without."""
        if fields is None:
            return 0, None
        import hashlib
        return fields.shape[0], hashlib.blake2b(np.ascontiguousarray(fields).tobytes(), digest_size=16).hexdigest()

    def _device_drift_signature(self):
        return ()

    def _configure_device_drift(self, h):
        """Hook for drift terms evaluated on the device (UniversalKriging: point_log, external_Z)."""
        h.set_device_drift(None, None)

    def _ensure_problem(self, dtype="float64", knn=False, n_gpus=None, fields=None):
        name = dtype if isinstance(dtype, str) and dtype in _cabi.DTYPES else str(np.dtype(dtype))
        dt = _cabi.DTYPES.get(name)
        if dt is None:
            raise ValueError("dtype must be one of %s" % ", ".join(repr(k) for k in _cabi.DTYPES))
        h = self._cuda_handle(n_gpus)
        grouped = isinstance(h, _cabi.Group)
        if self._device_model()[0] == self.TABLE_MODEL_ID:
            self._table_dmax()                  # fixes the tabulated range before it enters the signature
        key = self._problem_signature(dt, knn, fields)
        if (self._kb_gkey if grouped else self._kb_key) == key:
            return h
        x, y, z, v, center, Mt = self._data_arrays()
        mid, vp = self._device_model()
        n_rl, cols = self._drift_spec()
        if grouped:
            self._kb_gkey = None
        else:
            self._kb_key = None
        if knn and bool(getattr(self, "pseudo_inv", False)):
            warnings.warn("pseudo_inv is ignored by the moving window (n_closest_points), as in the reference "
                          "(ok.py:753 always calls scipy.linalg.solve).", UserWarning)
        h.set_coordinates(getattr(self, "coordinates_type", "euclidean") == "geographic")
        h.set_pseudo_inverse(bool(getattr(self, "pseudo_inv", False)) and not knn)
        if mid == self.TABLE_MODEL_ID:
            dmax = self._table_dmax()
            h.set_variogram_table(self._variogram_table(dmax), dmax)
        if fields is not None or getattr(h, "n_fields", 0):
            h.set_values(fields)
        if knn:
            h.set_problem_knn(self._ndim, x, y, z, v, center, Mt, mid, vp, self.exact_values, self.eps)
        else:
            self._configure_device_drift(h)
            h.set_problem(self._ndim, dt, x, y, z, v, center, Mt, mid, vp, self.exact_values, self.eps,
                          n_rl=n_rl, drift_data=cols if cols else None)
        if grouped:
            self._kb_gkey = key
        else:
            self._kb_key = key
        return h

    # ---- execute(): argument handling shared by the four classes ---------------------------------
    _MASK_DIM_MSG = {2: "Mask is not two-dimensional.", 3: "Mask is not three-dimensional."}
    _POINTS_MSG = {
        2: "xpoints and ypoints must have same dimensions when treated as listing discrete points.",
        3: "xpoints, ypoints, and zpoints must have same dimensions when treated as listing discrete points.",
    }

    def _prepare_points(self, style, coords, mask):
        """style / mask / point-list validation of execute() (ok.py:834-874, uk.py:1169-1215, ok3d.py:833-876,
        uk3d.py:981-1024), once for 2-D and 3-D. coords = (xpoints, ypoints[, zpoints]).
        Returns (axes: list of 1-D float64 arrays, sizes (nx, ny[, nz]), flat_mask or None); the mask is
        returned in the reference's flattened order (x fastest; 3-D: (z, y, x))."""
        nd = self._ndim
        if style != "grid" and style != "masked" and style != "points":
            raise ValueError("style argument must be 'grid', 'points', or 'masked'")
        axes = [np.atleast_1d(np.squeeze(np.array(c, copy=True))) for c in coords]
        sizes = tuple(a.size for a in axes)
        flat_mask = None
        if style == "masked":
            if mask is None:
                raise IOError("Must specify boolean masking array when style is 'masked'.")
            if mask.ndim != nd:
                raise ValueError(self._MASK_DIM_MSG[nd])
            want = sizes[::-1]                        # (ny, nx) / (nz, ny, nx)
            if tuple(mask.shape) != want:
                if tuple(mask.shape) == sizes:        # given as (nx, ny[, nz]): transpose (ok.py:855-859)
                    mask = mask.T if nd == 2 else mask.swapaxes(0, 2)
                else:
                    raise ValueError("Mask dimensions do not match specified grid dimensions.")
            flat_mask = np.asarray(mask, dtype=bool).flatten()
        elif style == "points":
            bad = (sizes[0] != sizes[1]) if nd == 2 else (sizes[0] != sizes[1] and sizes[1] != sizes[2])
            if bad:
                raise ValueError(self._POINTS_MSG[nd])
        return [a.astype(np.float64) for a in axes], sizes, flat_mask

    def _specified_drift_grids(self, style, specified_drift_arrays, sizes, npoints, cls_name):
        """'specified' drift arrays at the prediction points: validation of uk.py:1217-1274 / uk3d.py:1040-1098.
        Returns the list of arrays in the reference's orientation ((ny, nx) / (nz, ny, nx) or (n,))."""
        nd = self._ndim
        if specified_drift_arrays is None:
            specified_drift_arrays = []
        grids = []
        if self.specified_drift:
            if len(specified_drift_arrays) == 0:
                raise ValueError("Must provide drift values for kriging points when using 'specified' drift capability.")
            if type(specified_drift_arrays) is not list:
                raise TypeError("Arrays for specified drift terms must be encapsulated in a list.")
            want = sizes[::-1]
            for spec in specified_drift_arrays:
                if style in ["grid", "masked"]:
                    if spec.ndim < nd:
                        raise ValueError("Dimensions of drift values array do not match specified grid dimensions.")
                    elif tuple(spec.shape[:nd]) != want:
                        if tuple(spec.shape[:nd]) == sizes:
                            grids.append(np.squeeze(spec.T if nd == 2 else spec.swapaxes(0, 2)))
                        else:
                            raise ValueError("Dimensions of drift values array do not match specified grid dimensions.")
                    else:
                        grids.append(np.squeeze(spec))
                elif style == "points":
                    if spec.ndim != 1:
                        raise ValueError("Dimensions of drift values array do not match specified grid dimensions.")
                    elif spec.shape[0] != npoints:
                        raise ValueError("Number of supplied drift values in array do not match specified number of kriging points.")
                    else:
                        grids.append(np.squeeze(spec))
            if len(grids) != len(self.specified_drift_data_arrays):
                raise ValueError("Inconsistent number of specified drift terms supplied.")
        elif len(specified_drift_arrays) != 0:
            warnings.warn(
                "Provided specified drift values, but 'specified' drift was not initialized during "
                "instantiation of %s class." % cls_name, RuntimeWarning,
            )
        return grids

    @staticmethod
    def _shape_output(style, z, ss, sizes, flat_mask):
        """Masked wrap + reshape of execute() (ok.py:1012-1020, ok3d.py:924-932). z may carry a leading field
        axis (execute(values=...)); the grid mask is broadcast over it."""
        if style == "masked":
            zmask = flat_mask if np.ndim(z) == 1 else np.broadcast_to(flat_mask, np.shape(z)).copy()
            z = np.ma.array(z, mask=zmask)
            ss = np.ma.array(ss, mask=flat_mask)
        if style in ["masked", "grid"]:
            z = z.reshape(np.shape(z)[:-1] + tuple(sizes[::-1]))
            ss = ss.reshape(sizes[::-1])
        return z, ss

    # ---- execute(values=...): several value fields through one factorisation ---------------------------------
    @staticmethod
    def _fields_kw(fields):
        """Keyword for _run_cuda: without fields the call is the single-field call, unchanged."""
        return {} if fields is None else {"fields": fields}

    def _check_values(self, values, dtype, n_closest_points, n_gpus):
        """Validates the values= keyword of execute() after the reference's own argument checks. Returns
        (fields as a (V, N) float64 array, whether values was 1-D), or (None, False) for values=None."""
        if values is None:
            return None, False
        v = np.asarray(values)
        n = np.size(self._data_arrays()[3])
        if v.ndim not in (1, 2):
            raise ValueError("values must have shape (N,) or (N, V), got %d dimensions" % v.ndim)
        if v.shape[0] != n:
            raise ValueError("values has %d rows; it needs one row per data point (N = %d), shape (N, V)"
                             % (v.shape[0], n))
        one = v.ndim == 1
        v = v.reshape(n, -1).astype(np.float64)
        if v.shape[1] == 0:
            raise ValueError("values has no fields (V = 0)")
        if not np.all(np.isfinite(v)):
            raise ValueError("values must be finite")
        name = dtype if isinstance(dtype, str) else str(np.dtype(dtype))
        if name != "float64":
            raise NotImplementedError("execute(values=...) runs in dtype='float64' only")
        if bool(getattr(self, "pseudo_inv", False)) and n_closest_points is None:
            raise NotImplementedError("execute(values=...) is not supported with pseudo_inv=True")
        if n_gpus is not None and int(n_gpus) > 1:
            raise NotImplementedError("execute(values=...) runs on one GPU (n_gpus > 1 is not supported)")
        return np.ascontiguousarray(v.T), one

    # ---- the device run: plan (what to compute) -> run (one contiguous block of it) -> scatter ----
    def _plan(self, style, axes, mask, drift_at=None):
        """What one execute() computes, as a flat work list that can be cut into contiguous blocks (one per
        GPU): kind 'grid' (points generated on the device from the axes, 0 bytes/point of input) or 'points'
        (explicit coordinates; 'masked' keeps only the unmasked cells, host-supplied drift forces a list)."""
        nd = self._ndim
        if style == "points":
            pts = [np.ascontiguousarray(a, dtype=np.float64) for a in axes]
            return {"kind": "points", "pts": pts, "idx": None, "npt": pts[0].size, "count": pts[0].size,
                    "scatter": False}
        sizes = [a.size for a in axes[:nd]]
        npt = int(np.prod(sizes))
        if mask is None and drift_at is None:
            return {"kind": "grid", "axes": axes, "npt": npt, "count": npt, "scatter": False}
        idx = np.flatnonzero(~mask) if mask is not None else np.arange(npt)
        nx, ny = sizes[0], sizes[1]
        pts = [np.asarray(axes[0], dtype=np.float64)[idx % nx], np.asarray(axes[1], dtype=np.float64)[(idx // nx) % ny]]
        if nd == 3:
            pts.append(np.asarray(axes[2], dtype=np.float64)[idx // (nx * ny)])
        return {"kind": "points", "pts": pts, "idx": idx, "npt": npt, "count": idx.size, "scatter": mask is not None}

    def _run_block(self, h, plan, first, count, n_closest_points=None, drift_at=None):
        """Krige items [first, first+count) of the plan's work list on handle (or device group) `h`."""
        nd = self._ndim
        knn = n_closest_points is not None
        if count <= 0:
            return np.zeros(0), np.zeros(0)
        if plan["kind"] == "grid":
            ax = plan["axes"]
            gz = ax[2] if nd == 3 else None
            if knn:
                return h.execute_knn_grid(n_closest_points, ax[0], ax[1], gz, first, count)
            return h.execute_grid(ax[0], ax[1], gz, None, first, count)
        sl = slice(first, first + count)
        pts = [p[sl] for p in plan["pts"]]
        idx = plan["idx"][sl] if plan["idx"] is not None else None
        if idx is None and (first != 0 or count != plan["count"]):
            idx = np.arange(first, first + count)      # 'points' style: position in the caller's arrays
        dv = drift_at(pts, idx) if drift_at is not None else None
        if knn:
            return h.execute_knn_points(n_closest_points, pts[0], pts[1], pts[2] if nd == 3 else None)
        return h.execute_points(pts[0], pts[1], pts[2] if nd == 3 else None, dv)

    @staticmethod
    def _scatter(plan, z, ss):
        if not plan["scatter"]:
            return z, ss
        zf = np.zeros(np.shape(z)[:-1] + (plan["npt"],))
        sf = np.zeros(plan["npt"])
        zf[..., plan["idx"]] = z
        sf[plan["idx"]] = ss
        return zf, sf

    def _run_cuda(self, style, axes, mask, n_closest_points=None, drift_at=None, dtype="float64", n_gpus=None,
                  fields=None):
        """axes: list of 1-D coordinate arrays [x, y(, z)] (grid axes or point lists, original coords).
        mask: flattened bool mask (True = skip) or None.  drift_at: callable(pts list, idx) -> [n_hd, m]
        host-supplied drift values at the given points, or None.  n_gpus: None/1 = this handle's device;
        G > 1 = single-process multi-GPU (one host thread, kb200_group_*: device 0 factors, peer copies of the
        factor blob, contiguous blocks of the work list, results gathered in the reference's order).
        fields: (V, N) value fields kriged instead of the constructor's values, or None.
        Returns flat (z, ss) of length npt in the reference's flattened order; z is (V, npt) with fields.
        More than _cabi.MAX_FIELDS fields run as chunks of that many, each its own problem (factorisation) and
        execute; every field's result is independent of the chunk it is in."""
        knn = n_closest_points is not None
        nd = self._ndim
        if self._device_model()[0] == self.TABLE_MODEL_ID and all(np.size(a) for a in axes[:nd]):
            self._table_dmax([float(np.min(a)) for a in axes[:nd]], [float(np.max(a)) for a in axes[:nd]])
        if fields is None:
            h = self._ensure_problem(dtype, knn, n_gpus=n_gpus)
            plan = self._plan(style, axes, mask, drift_at)
            z, ss = self._run_block(h, plan, 0, plan["count"], n_closest_points, drift_at)
            return self._scatter(plan, z, ss)
        plan = self._plan(style, axes, mask, drift_at)
        zs = []
        for c0 in range(0, fields.shape[0], _cabi.MAX_FIELDS):
            chunk = fields[c0:c0 + _cabi.MAX_FIELDS]
            h = self._ensure_problem(dtype, knn, n_gpus=n_gpus, fields=chunk)
            z, ss = self._run_block(h, plan, 0, plan["count"], n_closest_points, drift_at)
            zs.append(np.reshape(z, (chunk.shape[0], -1)))
        return self._scatter(plan, np.concatenate(zs), ss)

    # ---- leave_one_out(): cross-validation of every station --------------------------------------------------
    def _leave_one_out(self, n_closest_points, values, backend, what):
        """(zvalues, sigmasq) of kriging every station from the other N - 1 with this object's fixed variogram
        (DESIGN.md §5e): the global path from the factorisation the last float64 execute() left on the handle (or a
        new one, which a later execute() reuses), the moving window with n_closest_points neighbours. values as in
        execute(values=...): zvalues is (V, N) for a 2-D values, (N,) otherwise; sigmasq is (N,)."""
        self._check_backend(backend, what)
        n = int(np.size(self._data_arrays()[3]))
        if n < 2:
            raise ValueError("leave-one-out needs at least two data points, got %d" % n)
        knn = n_closest_points is not None
        if knn and not 2 <= n_closest_points <= n - 1:
            raise ValueError("leave-one-out: n_closest_points must be in [2, N - 1] = [2, %d], got %r"
                             % (n - 1, n_closest_points))
        if not knn and bool(getattr(self, "pseudo_inv", False)):
            raise NotImplementedError("leave_one_out() has no pseudo_inv=True form on the global path: the "
                                      "leave-one-out identities need the inverse of the kriging matrix")
        fields, one = self._check_values(values, "float64", n_closest_points, None)

        def run(h):
            return h.knn_loo(int(n_closest_points), n) if knn else h.loo(n)
        if fields is None:
            return run(self._ensure_problem("float64", knn))
        zs = []
        for c0 in range(0, fields.shape[0], _cabi.MAX_FIELDS):
            chunk = fields[c0:c0 + _cabi.MAX_FIELDS]
            z, ss = run(self._ensure_problem("float64", knn, fields=chunk))
            zs.append(np.reshape(z, (chunk.shape[0], n)))
        z = np.concatenate(zs)
        return (z[0] if one else z), ss

    @staticmethod
    def _check_backend(backend, what):
        if backend != "cuda":
            raise ValueError(
                "Specified backend {} is not supported for {}: this package implements backend='cuda' only "
                "(the reference's 'vectorized'/'loop'/'C' CPU paths live in PyKrige).".format(backend, what)
            )
