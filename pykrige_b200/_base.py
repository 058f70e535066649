"""Shared host logic of the four kriging classes (not part of the reference's API surface).

The reference repeats this logic in ok.py / uk.py / ok3d.py / uk3d.py; here it lives once, for 2-D and 3-D alike:
the constructor and update_variogram_model (ok.py:208-553, uk.py:246-790, ok3d.py:221-520, uk3d.py:239-660),
variogram model selection (ok.py:208-253), the ``backend='cuda'`` dispatch that replaces the ``backend`` string switch
of ``execute`` (ok.py:971-1010), point-list / grid / mask handling (ok.py:842-900, ok3d.py:833-898), the 'specified'
and 'functional' drift terms of the universal classes and output shaping (ok.py:1012-1020). What differs between the
dimensions and the classes is data: the class attributes of Krige2D / Krige3D and of the four classes.
"""
import hashlib
import re
import warnings
from collections import namedtuple

import numpy as np

from . import variogram_models
from . import core
from . import _cabi
from .core import _adjust_for_anisotropy, _make_variogram_parameter_list, _initialize_variogram_model

P_INV_TYPES = ("pinv", "pinvh")
GEO_ANISOTROPY_WARNING = "Anisotropy is not compatible with geographic coordinates. Ignoring user set anisotropy."

# What the device problem on a handle was built from. digest covers every input array (coordinates, values, host drift
# columns, device drift arrays, value fields), so that an in-place edit of any of them invalidates the factorisation.
ProblemKey = namedtuple("ProblemKey", "dtype knn model params exact_values aniso center n_rl geographic pseudo_inv "
                                      "n_fields digest")


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
    # per dimension (Krige2D / Krige3D): coordinate letters (X_ORIG, XCENTER, X_ADJUSTED, ...), the attribute of the
    # values, the anisotropy attributes (scalings, then angles: the order of the constructor's arguments)
    _ndim = None
    _AXES = None
    _VALUES = None
    _SCALINGS = ()
    _ANGLES = ()
    # per class: the name in the backend error, drift terms (the universal classes), whether n_closest_points is checked
    # before the point lists (OrdinaryKriging), the "Coordinates type" line (OrdinaryKriging, ok.py:333)
    _KIND = None
    _universal = False
    _k_before_points = False
    _prints_coordinates_type = False

    # ---- variogram model selection (ok.py:208-253; GSTools models arrive as 'custom') ----
    def _select_variogram(self, variogram_model, variogram_function, variogram_parameters, anisotropy, check_latlon):
        """Returns the (variogram_parameters, anisotropy) that apply: a GSTools CovModel brings its own callable and
        anisotropy (ok.py:224-239)."""
        self.variogram_model = variogram_model
        self.model = None
        if hasattr(self.variogram_model, "pykrige_kwargs"):
            from .compat_gstools import validate_gstools

            self.model = self.variogram_model
            validate_gstools(self.model)
            if self._ndim == 2 and self.model.field_dim == 3:
                raise ValueError("GSTools: model dim is not 1 or 2")
            if self._ndim == 3 and self.model.field_dim < 3:
                raise ValueError("GSTools: model dim is not 3")
            if check_latlon and self.model.latlon and self.coordinates_type == "euclidean":
                raise ValueError("GSTools: latlon models require geographic coordinates")
            self.variogram_model = "custom"
            variogram_function = self.model.pykrige_vario
            variogram_parameters = []
            anisotropy = tuple(getattr(self.model, a.replace("anisotropy_scaling", "pykrige_anis")
                                       .replace("anisotropy_angle", "pykrige_angle"))
                               for a in self._SCALINGS + self._ANGLES)
        if self.variogram_model not in self.variogram_dict.keys() and self.variogram_model != "custom":
            raise ValueError("Specified variogram model '%s' is not supported." % variogram_model)
        elif self.variogram_model == "custom":
            if variogram_function is None or not callable(variogram_function):
                raise ValueError("Must specify callable function for custom variogram model.")
            self.variogram_function = variogram_function
        else:
            self.variogram_function = self.variogram_dict[self.variogram_model]
        return variogram_parameters, anisotropy

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

    # ---- constructor and update_variogram_model ------------------------------------------------------------------
    def _init_model(self, coords, values, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                    anisotropy, verbose, enable_plotting, exact_values, pseudo_inv, pseudo_inv_type,
                    coordinates_type="euclidean", statistics="lazy"):
        """The constructor body: option checks, GSTools hand-over, float64 copies of the data, anisotropy of the data,
        variogram initialisation, statistics policy. coords = (x, y[, z]); anisotropy = the values of the anisotropy
        attributes in argument order. statistics: 'off' (OrdinaryKriging default), 'eager' (enable_statistics=True) or
        'lazy' (the other classes: the reference computes them in the constructor, uk.py:380; here on first access)."""
        self.pseudo_inv = bool(pseudo_inv)
        self.pseudo_inv_type = str(pseudo_inv_type)
        if self.pseudo_inv_type not in P_INV_TYPES:
            raise ValueError("pseudo inv type not valid: " + str(pseudo_inv_type))
        if not isinstance(exact_values, bool):
            raise ValueError("exact_values has to be boolean True or False")
        if coordinates_type not in ("euclidean", "geographic"):
            raise ValueError("Only 'euclidean' and 'geographic' are valid values for coordinates-keyword.")
        self.exact_values = exact_values
        self.coordinates_type = coordinates_type
        self.verbose = verbose
        self.enable_plotting = enable_plotting
        variogram_parameters, anisotropy = self._select_variogram(
            variogram_model, variogram_function, variogram_parameters, anisotropy, check_latlon=self._ndim == 2)

        # 1-D float64 copies of the inputs (ok.py:262-268)
        copies = [np.atleast_1d(np.squeeze(np.array(a, copy=True, dtype=np.float64))) for a in tuple(coords) + (values,)]
        for name, a in zip([c + "_ORIG" for c in self._AXES] + [self._VALUES], copies):
            setattr(self, name, a)
        if self.enable_plotting and self.verbose:
            print("Plotting Enabled\n")

        if coordinates_type == "geographic":
            # lon/lat in degrees (2-D only); anisotropy is ambiguous on the sphere and ignored (ok.py:292-306)
            if anisotropy[0] != 1.0:
                warnings.warn(GEO_ANISOTROPY_WARNING, UserWarning)
            self.XCENTER = self.YCENTER = 0.0
            self.anisotropy_scaling, self.anisotropy_angle = 1.0, 0.0
            self.X_ADJUSTED, self.Y_ADJUSTED = self.X_ORIG, self.Y_ORIG
        else:
            for c in self._AXES:
                orig = getattr(self, c + "_ORIG")
                setattr(self, c + "CENTER", (np.amax(orig) + np.amin(orig)) / 2.0)
            self._set_anisotropy(anisotropy)

        if self.verbose:
            print("Initializing variogram model...")
        self._fit_variogram(variogram_parameters, nlags, weight)
        self._statistics_policy(statistics)

    def _update_variogram_model(self, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                                anisotropy):
        variogram_parameters, anisotropy = self._select_variogram(
            variogram_model, variogram_function, variogram_parameters, anisotropy, check_latlon=False)
        if self.coordinates_type == "geographic":
            if anisotropy[0] != 1.0:
                warnings.warn(GEO_ANISOTROPY_WARNING, UserWarning)
        elif tuple(anisotropy) != tuple(getattr(self, a) for a in self._SCALINGS + self._ANGLES):
            self._set_anisotropy(anisotropy)
        if self.verbose:
            print("Updating variogram mode...")
        self._fit_variogram(variogram_parameters, nlags, weight)
        self._statistics_policy("lazy")

    def _set_anisotropy(self, anisotropy):
        """Sets the anisotropy attributes and moves the data to the adjusted frame (X_ADJUSTED, ...)."""
        if self.verbose:
            print("Adjusting data for anisotropy...")
        for name, v in zip(self._SCALINGS + self._ANGLES, anisotropy):
            setattr(self, name, v)
        adjusted = self._adjust(*[getattr(self, c + "_ORIG") for c in self._AXES])
        for c, a in zip(self._AXES, adjusted):
            setattr(self, c + "_ADJUSTED", a)

    def _adjust(self, *coords):
        """This object's anisotropy applied to points given as coordinate arrays in the original frame: the adjusted
        coordinate arrays, stacked [ndim, n] (core.py:120-193)."""
        center, scalings, angles = self._anisotropy()
        return _adjust_for_anisotropy(np.vstack(coords).T, center, scalings, angles).T

    def _anisotropy(self):
        """(center, scalings, angles) as lists."""
        return ([getattr(self, c + "CENTER") for c in self._AXES], [getattr(self, a) for a in self._SCALINGS],
                [getattr(self, a) for a in self._ANGLES])

    def _fit_variogram(self, variogram_parameters, nlags, weight):
        self._nlags = nlags                     # the experimental variogram of data added later (add_data)
        X, values = self._stats_inputs()
        vp = _make_variogram_parameter_list(self.variogram_model, variogram_parameters)
        self.lags, self.semivariance, self.variogram_model_parameters = _initialize_variogram_model(
            X, values, self.variogram_model, vp, self.variogram_function, nlags, weight, self.coordinates_type,
            lazy=True)
        if self.verbose:
            if self._prints_coordinates_type:
                print("Coordinates type: '%s'" % self.coordinates_type, "\n")
            self._print_variogram()
        if self.enable_plotting:
            self.display_variogram_model()

    def _stats_inputs(self):
        """(adjusted data coordinates [n, ndim], values)"""
        return np.vstack([getattr(self, c + "_ADJUSTED") for c in self._AXES]).T, getattr(self, self._VALUES)

    def _data_arrays(self):
        """(x, y, z|None, values, center, Mt) in ORIGINAL coordinates."""
        center, scalings, angles = self._anisotropy()
        x, y, z = [getattr(self, c + "_ORIG") for c in self._AXES] + [None] * (3 - self._ndim)
        return x, y, z, getattr(self, self._VALUES), center, core.anisotropy_matrix(self._ndim, scalings, angles)

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
    def _device_statistics(self):
        """delta, sigma, epsilon from the Cholesky factor of the device problem (kb200_statistics,
        csrc/variogram.cu: O(N) after the factorisation instead of the reference's N solves). Returns
        None when this problem has no device twin (custom variogram, pseudo_inv, indefinite
        covariance form, no CUDA device) — the caller then runs the reference's loop on the host."""
        if not _cabi.device_available() or getattr(self, "pseudo_inv", False):
            return None                          # core._krige solves with lstsq under pseudo_inv (core.py:749-750)
        try:
            key = getattr(self, "_kb_key", None)
            if key is not None and not key.knn and key == self._problem_key(key.dtype, False):
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

    def _cover_prediction_points(self, axes):
        """A tabulated variogram must reach every data-prediction distance: extends its range to the box of the
        prediction points, axes = [x, y(, z)] grid axes or point lists (the same on every rank of a sharded run)."""
        nd = self._ndim
        if self._device_model()[0] == self.TABLE_MODEL_ID and all(np.size(a) for a in axes[:nd]):
            self._table_dmax([float(np.min(a)) for a in axes[:nd]], [float(np.max(a)) for a in axes[:nd]])

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

    def _drift_spec(self):
        """(n_rl, [host drift data columns])"""
        return 0, []

    def _device_drift(self):
        """(wells, ext) of the drift terms evaluated on the device (UniversalKriging: point_log, external_Z)."""
        return None, None

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

    def _problem_key(self, dtype, knn, fields=None):
        x, y, z, v, center, Mt = self._data_arrays()
        mid, vp = self._device_model()
        n_rl, cols = self._drift_spec()
        if mid == self.TABLE_MODEL_ID:      # the table itself is part of the problem
            vp = ("table", id(self.variogram_function), getattr(self, "_kb_table_dmax", 0.0)) + tuple(
                np.ravel(np.asarray(self.variogram_model_parameters, dtype=float)))
        wells, ext = self._device_drift()
        hsh = hashlib.blake2b(digest_size=16)
        for a in [x, y, z, v] + list(cols) + [wells] + list(ext or (None,)) + [fields]:
            if a is None:
                hsh.update(b"-")
            else:
                a = np.ascontiguousarray(a, dtype=np.float64)
                hsh.update(repr(a.shape).encode())
                hsh.update(a.tobytes())
        return ProblemKey(dtype, knn, mid, tuple(vp), bool(self.exact_values), tuple(np.ravel(Mt)), tuple(center), n_rl,
                          getattr(self, "coordinates_type", "euclidean") == "geographic",
                          bool(getattr(self, "pseudo_inv", False)), 0 if fields is None else fields.shape[0],
                          hsh.hexdigest())

    def _ensure_problem(self, dtype="float64", knn=False, n_gpus=None, fields=None):
        dt = _cabi.dtype_code(dtype)
        h = self._cuda_handle(n_gpus)
        slot = "_kb_gkey" if isinstance(h, _cabi.Group) else "_kb_key"
        if self._device_model()[0] == self.TABLE_MODEL_ID:
            self._table_dmax()                  # fixes the tabulated range before it enters the key
        key = self._problem_key(dt, knn, fields)
        if getattr(self, slot) == key:
            return h
        setattr(self, slot, None)
        self._set_up_problem(h, dt, knn, fields)
        setattr(self, slot, key)
        return h

    def _set_up_problem(self, h, dt, knn=False, fields=None, describe_only=False):
        """Configures handle (or group) h for this object's problem, then hands the problem over: kb200_set_problem
        (assemble and factor), kb200_set_problem_knn (the moving window) or, with describe_only, kb200_describe_problem
        (record it and allocate the factor blob that a broadcast fills, multigpu.prepare_sharded)."""
        x, y, z, v, center, Mt = self._data_arrays()
        mid, vp = self._device_model()
        if knn and bool(getattr(self, "pseudo_inv", False)):
            warnings.warn("pseudo_inv is ignored by the moving window (n_closest_points), as in the reference "
                          "(ok.py:753 always calls scipy.linalg.solve).", UserWarning)
        h.set_coordinates(getattr(self, "coordinates_type", "euclidean") == "geographic")
        h.set_pseudo_inverse(bool(getattr(self, "pseudo_inv", False)) and not knn)
        if mid == self.TABLE_MODEL_ID:          # 'custom' callable: every rank of a sharded run tabulates it itself
            dmax = self._table_dmax()
            h.set_variogram_table(self._variogram_table(dmax), dmax)
        if fields is not None or getattr(h, "n_fields", 0):
            h.set_values(fields)
        if knn:
            h.set_problem_knn(self._ndim, x, y, z, v, center, Mt, mid, vp, self.exact_values, self.eps)
            return
        h.set_device_drift(*self._device_drift())
        n_rl, cols = self._drift_spec()
        hand_over = h.describe_problem if describe_only else h.set_problem
        hand_over(self._ndim, dt, x, y, z, v, center, Mt, mid, vp, self.exact_values, self.eps, n_rl=n_rl,
                  drift_data=cols if cols else None)

    # ---- execute(): argument handling shared by the four classes ---------------------------------
    _MASK_DIM_MSG = {2: "Mask is not two-dimensional.", 3: "Mask is not three-dimensional."}
    _POINTS_MSG = {
        2: "xpoints and ypoints must have same dimensions when treated as listing discrete points.",
        3: "xpoints, ypoints, and zpoints must have same dimensions when treated as listing discrete points.",
    }

    @staticmethod
    def _check_style(style):
        if style != "grid" and style != "masked" and style != "points":
            raise ValueError("style argument must be 'grid', 'points', or 'masked'")

    @staticmethod
    def _check_n_closest_points(n_closest_points):
        if n_closest_points is not None and n_closest_points <= 1:
            raise ValueError("n_closest_points has to be at least two!")

    def _prepare_points(self, style, coords, mask):
        """style / mask / point-list validation of execute() (ok.py:834-874, uk.py:1169-1215, ok3d.py:833-876,
        uk3d.py:981-1024), once for 2-D and 3-D. coords = (xpoints, ypoints[, zpoints]).
        Returns (axes: list of 1-D float64 arrays, sizes (nx, ny[, nz]), flat_mask or None); the mask is
        returned in the reference's flattened order (x fastest; 3-D: (z, y, x))."""
        nd = self._ndim
        self._check_style(style)
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

    def _specified_drift_grids(self, style, specified_drift_arrays, sizes, npoints):
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
                "instantiation of %s class." % ("UniversalKriging" if nd == 2 else "UniversalKriging3D"), RuntimeWarning,
            )
        return grids

    def _check_drift_domain(self, axes):
        """Hook: UniversalKriging checks that its external-Z raster covers the prediction points."""

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

    def _execute(self, style, coords, mask, backend, n_closest_points=None, specified_drift_arrays=None,
                 dtype="float64", n_gpus=None, values=None):
        """The body of the four execute() methods, each class's checks in the order the reference makes them."""
        if self.verbose:
            print("Executing %s Kriging...\n" % ("Universal" if self._universal else "Ordinary"))
        if self._k_before_points:
            self._check_style(style)
            self._check_n_closest_points(n_closest_points)
        axes, sizes, flat_mask = self._prepare_points(style, coords, mask)
        self._check_n_closest_points(n_closest_points)
        drift_at = None
        if self._universal:
            drift_at = self._host_drift_at(self._specified_drift_grids(style, specified_drift_arrays, sizes,
                                                                       axes[0].size))
        self._check_backend(backend, self._KIND)
        self._check_drift_domain(axes)
        fields, one = self._check_values(values, dtype, n_closest_points, n_gpus)
        z, ss = self._run_cuda(style, axes, flat_mask, n_closest_points=n_closest_points, drift_at=drift_at,
                               dtype=dtype, n_gpus=n_gpus, fields=fields)
        return self._shape_output(style, z[0] if one else z, ss, sizes, flat_mask)

    # ---- 'specified' and 'functional' drift terms of the universal classes ---------------------------------------
    def _init_host_drift_terms(self, drift_terms, specified_drift, functional_drift):
        """The 'specified' (uk.py:476-494) and 'functional' (uk.py:496-510) drift terms of the constructor."""
        if specified_drift is None:
            specified_drift = []
        if functional_drift is None:
            functional_drift = []
        if "specified" in drift_terms:
            if type(specified_drift) is not list:
                raise TypeError("Arrays for specified drift terms must be encapsulated in a list.")
            if len(specified_drift) == 0:
                raise ValueError("Must provide at least one drift-value array when using the 'specified' drift capability.")
            self.specified_drift = True
            self.specified_drift_data_arrays = []
            for term in specified_drift:
                specified = np.squeeze(np.array(term, copy=True))
                if specified.size != self.X_ORIG.size:
                    raise ValueError("Must specify the drift values for each data point when using the 'specified' drift capability.")
                self.specified_drift_data_arrays.append(specified)
        else:
            self.specified_drift = False
        # functional drift: callables evaluated with the adjusted coordinates
        if "functional" in drift_terms:
            if type(functional_drift) is not list:
                raise TypeError("Callables for functional drift terms must be encapsulated in a list.")
            if len(functional_drift) == 0:
                raise ValueError("Must provide at least one callable object when using the 'functional' drift capability.")
            self.functional_drift = True
            self.functional_drift_terms = functional_drift
        else:
            self.functional_drift = False

    def _host_drift_at(self, spec_drift_grids):
        """The drift_at callback of a run (see _run_cuda): the 'specified' and 'functional' drift values at the
        prediction points (uk.py:972-979, uk3d.py:1100-1110), or None without such terms."""
        if not (self.specified_drift or self.functional_drift):
            return None

        def drift_at(pts, idx):
            cols = []
            for g in spec_drift_grids:
                flat = np.asarray(g, dtype=float).flatten()
                cols.append(flat if idx is None else flat[idx])
            if self.functional_drift:
                adjusted = self._adjust(*pts)
                for func in self.functional_drift_terms:
                    cols.append(np.asarray(func(*adjusted), dtype=float) * np.ones(adjusted[0].shape))
            return np.ascontiguousarray(np.vstack(cols), dtype=np.float64)
        return drift_at

    # ---- execute(values=...): several value fields through one factorisation ---------------------------------
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
        if _cabi.dtype_name(dtype) != "float64":
            raise NotImplementedError("execute(values=...) runs in dtype='float64' only")
        if bool(getattr(self, "pseudo_inv", False)) and n_closest_points is None:
            raise NotImplementedError("execute(values=...) is not supported with pseudo_inv=True")
        if n_gpus is not None and int(n_gpus) > 1:
            raise NotImplementedError("execute(values=...) runs on one GPU (n_gpus > 1 is not supported)")
        return np.ascontiguousarray(v.T), one

    @staticmethod
    def _per_chunk(fields, run):
        """run(chunk) -> (z, ss) once with chunk None (no fields) or once per chunk of at most _cabi.MAX_FIELDS
        fields, each its own problem (factorisation); z then is (V, m): every field's result is independent of the
        chunk it is in."""
        if fields is None:
            return run(None)
        zs = []
        for c0 in range(0, fields.shape[0], _cabi.MAX_FIELDS):
            chunk = fields[c0:c0 + _cabi.MAX_FIELDS]
            z, ss = run(chunk)
            zs.append(np.reshape(z, (chunk.shape[0], -1)))
        return np.concatenate(zs), ss

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
        fields: (V, N) value fields kriged instead of the constructor's values, or None (see _per_chunk).
        Returns flat (z, ss) of length npt in the reference's flattened order; z is (V, npt) with fields."""
        knn = n_closest_points is not None
        self._cover_prediction_points(axes)
        plan = self._plan(style, axes, mask, drift_at)

        def run(chunk):
            h = self._ensure_problem(dtype, knn, n_gpus=n_gpus, fields=chunk)
            return self._run_block(h, plan, 0, plan["count"], n_closest_points, drift_at)
        z, ss = self._per_chunk(fields, run)
        return self._scatter(plan, z, ss)

    # ---- leave_one_out() and leave_group_out(): cross-validation of every station ----------------------------------
    def _cross_validate(self, groups, n_closest_points, values, backend):
        """(zvalues, sigmasq) of kriging every station from the stations outside its group with this object's fixed
        variogram: groups=None holds out each station alone (leave-one-out, DESIGN.md §5e), else groups holds N labels of
        any type np.unique sorts and the errors name the user's label (leave-group-out, §5f). The global path runs from
        the factorisation the last float64 execute() left on the handle (or a new one, which a later execute() reuses),
        the moving window with n_closest_points neighbours. values as in execute(values=...): zvalues is (V, N) for a
        2-D values, (N,) otherwise; sigmasq is (N,)."""
        self._check_backend(backend, self._KIND)
        n = int(np.size(self._data_arrays()[3]))
        knn = n_closest_points is not None
        if groups is None:
            what = "leave-one-out"
            if n < 2:
                raise ValueError("leave-one-out needs at least two data points, got %d" % n)
            if knn and not 2 <= n_closest_points <= n - 1:
                raise ValueError("leave-one-out: n_closest_points must be in [2, N - 1] = [2, %d], got %r"
                                 % (n - 1, n_closest_points))
        else:
            what = "leave-group-out"
            g = np.asarray(groups)
            if g.ndim != 1 or g.shape[0] != n:
                raise ValueError("groups must have shape (N,) = (%d,), one label per data point, got shape %s"
                                 % (n, g.shape))
            labels, dense, sizes = np.unique(g, return_inverse=True, return_counts=True)
            if labels.size < 2:
                raise ValueError("leave-group-out needs at least two distinct groups, got %d" % labels.size)
            dense = np.ascontiguousarray(dense.reshape(-1), dtype=np.int32)
            big = int(np.argmax(sizes))
            if knn and not 2 <= n_closest_points <= n - int(sizes[big]):
                raise ValueError("leave-group-out: n_closest_points must be in [2, N - %d] = [2, %d] (group %r has %d "
                                 "stations), got %r" % (sizes[big], n - sizes[big], labels[big].item(), sizes[big],
                                                        n_closest_points))
        if not knn and bool(getattr(self, "pseudo_inv", False)):
            raise NotImplementedError("%s() has no pseudo_inv=True form on the global path: the %s identities need the "
                                      "inverse of the kriging matrix" % (what.replace("-", "_"), what))
        fields, one = self._check_values(values, "float64", n_closest_points, None)

        def run(chunk):
            h = self._ensure_problem("float64", knn, fields=chunk)
            if groups is None:
                return h.knn_loo(int(n_closest_points), n) if knn else h.loo(n)
            try:
                if knn:
                    return h.knn_lgo(int(n_closest_points), dense, labels.size, n)
                return h.lgo(dense, labels.size, n)
            except np.linalg.LinAlgError as e:
                msg = re.sub(r"group (\d+)", lambda m: "group %r" % (labels[int(m.group(1))].item(),), str(e))
                if labels.size == n:            # every group one station: the leave-one-out message names the station
                    msg = re.sub(r"station (\d+)", lambda m: "station %s (group %r)" % (
                        m.group(1), labels[dense[int(m.group(1))]].item()), msg)
                raise np.linalg.LinAlgError(msg) from None
        z, ss = self._per_chunk(fields, run)
        return (z[0] if one else z), ss

    # ---- add_data(): new stations for the held problem ---------------------------------------------------------
    def _add_data(self, coords, values, specified_drift=None):
        """The body of add_data() of the four classes. coords = (x, y[, z]) of the new stations in the original frame.
        Afterwards every public result equals that of an object built with the same arguments, the current variogram
        as fixed parameters, on the old stations followed by the new ones (DESIGN.md §5g)."""
        new = [np.atleast_1d(np.squeeze(np.array(a, copy=True, dtype=np.float64))) for a in tuple(coords) + (values,)]
        m = new[0].size
        if m == 0 or any(a.ndim != 1 or a.size != m for a in new):
            raise ValueError("add_data: %s and the values must be 1-D arrays of the same non-zero length, got sizes %s"
                             % (", ".join(c.lower() for c in self._AXES), [a.size for a in new]))
        if not all(np.all(np.isfinite(a)) for a in new):
            raise ValueError("add_data: coordinates and values must be finite")
        extra = self._new_drift_data(new[:self._ndim], m, specified_drift)

        key = getattr(self, "_kb_key", None)
        h = getattr(self, "_kb_handle", None)
        fast = (h is not None and key is not None and not key.knn and key.n_fields == 0 and not key.pseudo_inv
                and key == self._problem_key(key.dtype, False))
        frame = self._anisotropy()[0]
        dmax = getattr(self, "_kb_table_dmax", 0.0)

        names = [c + "_ORIG" for c in self._AXES] + [self._VALUES]
        for name, a in zip(names, new):
            setattr(self, name, np.concatenate([getattr(self, name), a]))
        if self.coordinates_type == "geographic":
            self.X_ADJUSTED, self.Y_ADJUSTED = self.X_ORIG, self.Y_ORIG
        else:
            for c in self._AXES:
                orig = getattr(self, c + "_ORIG")
                setattr(self, c + "CENTER", (np.amax(orig) + np.amin(orig)) / 2.0)
            self._set_anisotropy([getattr(self, a) for a in self._SCALINGS + self._ANGLES])
        self._append_drift_data(extra)

        # the variogram stays; the experimental variogram and the statistics belong to the data
        X, vals = self._stats_inputs()
        self.lags, self.semivariance, _ = _initialize_variogram_model(
            X, vals, self.variogram_model, list(self.variogram_model_parameters), self.variogram_function, self._nlags,
            False, self.coordinates_type, lazy=True)
        if getattr(self, "_stats_state", "off") == "done":
            self._stats_state = "lazy"

        self._kb_key = None
        if getattr(self, "_kb_group", None) is not None:
            self._kb_gkey = None
        if fast and getattr(self, "functional_drift", False) and self._anisotropy()[0] != frame:
            # the callables see the adjusted coordinates: unless the map is the identity, a new centre moves them
            _, _, _, _, _, Mt = self._data_arrays()
            fast = np.array_equal(np.asarray(Mt, dtype=float).reshape(self._ndim, self._ndim), np.eye(self._ndim))
        if fast and self._device_model()[0] == self.TABLE_MODEL_ID:
            fast = self._table_dmax() == dmax      # a longer table is a new problem
        if not fast:
            return
        _, cols = self._drift_spec()
        try:
            h.append_data(*(new[:self._ndim] + [None] * (3 - self._ndim)), new[-1], [np.asarray(c, dtype=np.float64)[-m:] for c in cols] or None)
        except (NotImplementedError, np.linalg.LinAlgError):
            return                              # the next execute() sets the problem up from scratch
        self._kb_key = self._problem_key(key.dtype, False)

    def _new_drift_data(self, coords, m, specified_drift):
        """Checks the drift data of m new stations before anything changes (the constructor's messages) and returns
        what _append_drift_data needs: here the 'specified' arrays."""
        if not getattr(self, "specified_drift", False):
            if specified_drift:
                warnings.warn("Provided specified drift values, but 'specified' drift was not initialized during "
                              "instantiation of %s class." % type(self).__name__, RuntimeWarning)
            return {}
        if specified_drift is None:
            specified_drift = []
        if type(specified_drift) is not list:
            raise TypeError("Arrays for specified drift terms must be encapsulated in a list.")
        if len(specified_drift) == 0:
            raise ValueError("Must provide at least one drift-value array when using the 'specified' drift capability.")
        arrays = [np.atleast_1d(np.squeeze(np.array(term, copy=True))) for term in specified_drift]
        if len(arrays) != len(self.specified_drift_data_arrays):
            raise ValueError("Inconsistent number of specified drift terms supplied.")
        if any(a.size != m for a in arrays):
            raise ValueError("Must specify the drift values for each data point when using the 'specified' drift capability.")
        return {"specified": arrays}

    def _append_drift_data(self, extra):
        if "specified" in extra:
            self.specified_drift_data_arrays = [np.concatenate([np.ravel(old), np.ravel(a)])
                                                for old, a in zip(self.specified_drift_data_arrays, extra["specified"])]

    @staticmethod
    def _check_backend(backend, what):
        if backend != "cuda":
            raise ValueError(
                "Specified backend {} is not supported for {}: this package implements backend='cuda' only "
                "(the reference's 'vectorized'/'loop'/'C' CPU paths live in PyKrige).".format(backend, what)
            )


class Krige2D(KrigeBase):
    """OrdinaryKriging and UniversalKriging: data X_ORIG, Y_ORIG with values Z; geographic coordinates exist here."""
    _ndim = 2
    _AXES = "XY"
    _VALUES = "Z"
    _SCALINGS = ("anisotropy_scaling",)
    _ANGLES = ("anisotropy_angle",)

    def update_variogram_model(self, variogram_model, variogram_parameters=None, variogram_function=None, nlags=6,
                               weight=False, anisotropy_scaling=1.0, anisotropy_angle=0.0):
        """Change the variogram model and/or its parameters (ok.py:379-553, uk.py:630-790). The statistics are
        recomputed on their next access (the reference recomputes them here)."""
        self._update_variogram_model(variogram_model, variogram_parameters, variogram_function, nlags, weight,
                                     (anisotropy_scaling, anisotropy_angle))


    def add_data(self, x, y, z, specified_drift=None):
        """Adds stations at (x, y) with values z after the existing ones (monitoring networks that gain stations while
        the variogram stays). ``specified_drift`` (UniversalKriging with a 'specified' drift term): the list of drift
        arrays at the new stations, one per array of the constructor; the external_Z, point_log and functional drift
        values at the new stations are computed as the constructor computes them.

        The variogram is NOT refitted, even for an object built with an automatic fit: the current model and parameters
        stay, as if a new object were built with them given as fixed parameters. Everything that depends on the data
        follows the extended data exactly as a new object built on the old stations followed by the new ones (in that
        order) would: the original and adjusted coordinates, the centre of the anisotropy, the experimental variogram
        (``lags``, ``semivariance``), the statistics (recomputed on their next access), the drift data and every
        result of execute(), leave_one_out() and leave_group_out().

        When the handle holds the positive definite global factorisation of this object's current problem (after a
        global execute() in any dtype, or a cross-validation), the factorisation is extended on the device instead of
        being redone: one new block row of L and L^-1, about 2 m n^2 flops for m new stations, and the next execute()
        in the same dtype uses it. Otherwise the stations are only recorded and the next call sets the problem up
        from scratch, as for a new object: nothing held yet, a moving-window (n_closest_points) problem,
        ``pseudo_inv=True``, the indefinite fallback (a variogram that is not valid in this dimension), a problem of
        execute(values=...), ``n_gpus > 1``, a 'custom' variogram whose tabulated range no longer covers the data,
        'functional' drift terms with anisotropy when the centre moves (the callables see the adjusted coordinates),
        and an extended matrix that is singular (the new problem then raises as a new object would).
        """
        self._add_data((x, y), z, specified_drift)


class Krige3D(KrigeBase):
    """OrdinaryKriging3D and UniversalKriging3D: data X_ORIG, Y_ORIG, Z_ORIG with values VALUES."""
    _ndim = 3
    _AXES = "XYZ"
    _VALUES = "VALUES"
    _SCALINGS = ("anisotropy_scaling_y", "anisotropy_scaling_z")
    _ANGLES = ("anisotropy_angle_x", "anisotropy_angle_y", "anisotropy_angle_z")

    def update_variogram_model(self, variogram_model, variogram_parameters=None, variogram_function=None,
                               nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0,
                               anisotropy_angle_x=0.0, anisotropy_angle_y=0.0, anisotropy_angle_z=0.0):
        """Change the variogram model and/or its parameters (ok3d.py:354-520)."""
        self._update_variogram_model(variogram_model, variogram_parameters, variogram_function, nlags, weight,
                                     (anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x,
                                      anisotropy_angle_y, anisotropy_angle_z))

    def add_data(self, x, y, z, val, specified_drift=None):
        """Adds stations at (x, y, z) with values val after the existing ones; ``specified_drift`` as in
        UniversalKriging.add_data (UniversalKriging3D with a 'specified' drift term; functional drift values at the new
        stations are computed as the constructor computes them).

        The variogram is NOT refitted, even for an object built with an automatic fit: the current model and parameters
        stay, as if a new object were built with them given as fixed parameters. Everything that depends on the data
        follows the extended data exactly as a new object built on the old stations followed by the new ones (in that
        order) would: the original and adjusted coordinates, the centre of the anisotropy, the experimental variogram
        (``lags``, ``semivariance``), the statistics (recomputed on their next access), the drift data and every
        result of execute(), leave_one_out() and leave_group_out().

        When the handle holds the positive definite global factorisation of this object's current problem (after a
        global execute() in any dtype, or a cross-validation), the factorisation is extended on the device instead of
        being redone: one new block row of L and L^-1, about 2 m n^2 flops for m new stations, and the next execute()
        in the same dtype uses it. Otherwise the stations are only recorded and the next call sets the problem up
        from scratch, as for a new object: nothing held yet, a moving-window (n_closest_points) problem,
        ``pseudo_inv=True``, the indefinite fallback (a variogram that is not valid in this dimension), a problem of
        execute(values=...), ``n_gpus > 1``, a 'custom' variogram whose tabulated range no longer covers the data,
        'functional' drift terms with anisotropy when the centre moves (the callables see the adjusted coordinates),
        and an extended matrix that is singular (the new problem then raises as a new object would).
        """
        self._add_data((x, y, z), val, specified_drift)
