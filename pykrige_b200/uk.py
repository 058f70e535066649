"""UniversalKriging (2-D) with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/uk.py:220-1328). Regional-linear drift is built
on the device from the adjusted coordinates. The DATA-side columns of the other drift kinds
(uk.py:884-910) are evaluated once on the host and enter the device system as extra columns;
at the PREDICTION points point-log and external-Z (uk.py:955-971) are evaluated inside the solve
kernels (kb200_set_device_drift), only specified / functional values (uk.py:972-979) are shipped.
"""
import numpy as np

from ._base import Krige2D, P_INV_TYPES  # noqa: F401


def _first_last_index(axis, v):
    """(index of the first node >= v, index of the last node <= v) for every v — the node
    selection rule of the reference's bilinear sampler (uk.py:556-559)."""
    axis = np.asarray(axis, dtype=float)
    ge = axis[None, :] >= v[:, None]
    le = axis[None, :] <= v[:, None]
    i2 = np.argmax(ge, axis=1)
    i1 = axis.size - 1 - np.argmax(le[:, ::-1], axis=1)
    return i1, i2


class UniversalKriging(Krige2D):
    """Two-dimensional universal kriging; arguments as in the reference docstring (uk.py:40-205)."""

    UNBIAS = True  # the unbiasedness row is always present on the device path (uk.py:208)
    _KIND = "2D universal kriging"
    _universal = True

    def __init__(self, x, y, z, variogram_model="linear", variogram_parameters=None, variogram_function=None, nlags=6,
                 weight=False, anisotropy_scaling=1.0, anisotropy_angle=0.0, drift_terms=None, point_drift=None,
                 external_drift=None, external_drift_x=None, external_drift_y=None, specified_drift=None,
                 functional_drift=None, verbose=False, enable_plotting=False, exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        if drift_terms is None:
            drift_terms = []
        # no drift term exists yet: the statistics the common body may compute (verbose=True) are those of the
        # ordinary-kriging system, as in the reference, where they precede the drift initialisation (uk.py:380-394)
        self.regional_linear_drift = self.external_Z_drift = self.point_log_drift = False
        self.specified_drift = self.functional_drift = False
        self._init_model((x, y), z, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                         (anisotropy_scaling, anisotropy_angle), verbose, enable_plotting, exact_values, pseudo_inv,
                         pseudo_inv_type)

        if self.verbose:
            print("Initializing drift terms...")
        self.regional_linear_drift = "regional_linear" in drift_terms
        if self.regional_linear_drift and self.verbose:
            print("Implementing regional linear drift.")

        # external Z drift: sampled with the ORIGINAL coordinates (uk.py:413-446)
        if "external_Z" in drift_terms:
            if external_drift is None:
                raise ValueError("Must specify external Z drift terms.")
            if external_drift_x is None or external_drift_y is None:
                raise ValueError("Must specify coordinates of external Z drift terms.")
            self.external_Z_drift = True
            if external_drift.shape[0] != external_drift_y.shape[0] or external_drift.shape[1] != external_drift_x.shape[0]:
                if external_drift.shape[0] == external_drift_x.shape[0] and external_drift.shape[1] == external_drift_y.shape[0]:
                    self.external_Z_array = np.array(external_drift.T)
                else:
                    raise ValueError("External drift dimensions do not match provided x- and y-coordinate dimensions.")
            else:
                self.external_Z_array = np.array(external_drift)
            self.external_Z_array_x = np.array(external_drift_x).flatten()
            self.external_Z_array_y = np.array(external_drift_y).flatten()
            self.z_scalars = self._calculate_data_point_zscalars(self.X_ORIG, self.Y_ORIG)
            if self.verbose:
                print("Implementing external Z drift.")
        else:
            self.external_Z_drift = False

        # point-logarithmic drift: well coordinates go to the adjusted frame (uk.py:448-474)
        if "point_log" in drift_terms:
            if point_drift is None:
                raise ValueError("Must specify location(s) and strength(s) of point drift terms.")
            self.point_log_drift = True
            point_log = np.atleast_2d(np.squeeze(np.array(point_drift, copy=True)))
            self.point_log_array = np.zeros(point_log.shape)
            self.point_log_array[:, 2] = point_log[:, 2]
            self.point_log_array[:, :2] = self._adjust(point_log[:, 0], point_log[:, 1]).T
            self._point_log_orig = point_log[:, :2].copy()      # the wells move with the adjusted frame (add_data)
            if self.verbose:
                print("Implementing external point-logarithmic drift; number of points =",
                      self.point_log_array.shape[0], "\n")
        else:
            self.point_log_drift = False

        self._init_host_drift_terms(drift_terms, specified_drift, functional_drift)

    def _new_drift_data(self, coords, m, specified_drift):
        extra = super()._new_drift_data(coords, m, specified_drift)
        if self.external_Z_drift:       # the constructor's domain check, before anything changes
            extra["z_scalars"] = self._calculate_data_point_zscalars(coords[0], coords[1])
        return extra

    def _append_drift_data(self, extra):
        super()._append_drift_data(extra)
        if "z_scalars" in extra:
            self.z_scalars = np.concatenate([np.ravel(self.z_scalars), extra["z_scalars"]])
        if self.point_log_drift:        # as the constructor places the wells, in the moved frame
            wells = self.point_log_array.copy()
            wells[:, :2] = self._adjust(self._point_log_orig[:, 0], self._point_log_orig[:, 1]).T
            self.point_log_array = wells

    def _calculate_data_point_zscalars(self, x, y, type_="array"):
        """Bilinear sample of the external-Z grid at (x, y) (uk.py:512-628), vectorised; node
        selection, degenerate (on-node / on-line) cases and the domain check follow the reference."""
        xs = np.atleast_1d(np.asarray(x, dtype=float))
        ys = np.atleast_1d(np.asarray(y, dtype=float))
        shape = xs.shape
        xs = xs.ravel()
        ys = ys.ravel()
        ax, ay, Zg = self.external_Z_array_x, self.external_Z_array_y, self.external_Z_array
        if (np.any(xs > np.amax(ax)) or np.any(xs < np.amin(ax)) or np.any(ys > np.amax(ay)) or np.any(ys < np.amin(ay))):
            raise ValueError("External drift array does not cover specified kriging domain.")
        out = np.empty(xs.size)
        step = max(1, 4_000_000 // max(ax.size, ay.size))
        for s in range(0, xs.size, step):
            xn, yn = xs[s:s + step], ys[s:s + step]
            x1, x2 = _first_last_index(ax, xn)
            y1, y2 = _first_last_index(ay, yn)
            dx = ax[x2] - ax[x1]
            dy = ay[y2] - ay[y1]
            same_x = x1 == x2
            same_y = y1 == y2
            with np.errstate(divide="ignore", invalid="ignore"):
                full = (Zg[y1, x1] * (ax[x2] - xn) * (ay[y2] - yn) + Zg[y1, x2] * (xn - ax[x1]) * (ay[y2] - yn)
                        + Zg[y2, x1] * (ax[x2] - xn) * (yn - ay[y1]) + Zg[y2, x2] * (xn - ax[x1]) * (yn - ay[y1])) / (dx * dy)
                along_x = (Zg[y1, x1] * (ax[x2] - xn) + Zg[y2, x2] * (xn - ax[x1])) / dx
                along_y = (Zg[y1, x1] * (ay[y2] - yn) + Zg[y2, x2] * (yn - ay[y1])) / dy
            z = np.where(same_y, np.where(same_x, Zg[y1, x1], along_x), np.where(same_x, along_y, full))
            out[s:s + step] = z
        if type_ == "scalar":
            return out[0]
        return out.reshape(shape)

    def _point_log_column(self, well, xa, ya):
        """-strength * log(distance to the well), log(0) clamped to -100 (uk.py:885-896, 955-966)."""
        with np.errstate(divide="ignore"):
            ld = np.log(np.sqrt((xa - self.point_log_array[well, 0]) ** 2 + (ya - self.point_log_array[well, 1]) ** 2))
        ld = np.where(np.isinf(ld), -100.0, ld)
        return -self.point_log_array[well, 2] * ld

    def _drift_spec(self):
        """Host-evaluated drift columns at the data, in the reference's order (uk.py:884-910)."""
        cols = []
        if self.point_log_drift:
            for w in range(self.point_log_array.shape[0]):
                cols.append(self._point_log_column(w, self.X_ADJUSTED, self.Y_ADJUSTED))
        if self.external_Z_drift:
            cols.append(np.asarray(self.z_scalars, dtype=float))
        if self.specified_drift:
            for arr in self.specified_drift_data_arrays:
                cols.append(np.asarray(arr, dtype=float))
        if self.functional_drift:
            for func in self.functional_drift_terms:
                cols.append(np.asarray(func(self.X_ADJUSTED, self.Y_ADJUSTED), dtype=float))
        return (2 if self.regional_linear_drift else 0), cols

    def _device_drift(self):
        """point_log wells and the external-Z raster are evaluated at the prediction points by the solve kernels
        themselves (kb200_set_device_drift)."""
        wells = self.point_log_array if self.point_log_drift else None
        ext = ((self.external_Z_array_x, self.external_Z_array_y, self.external_Z_array)
               if self.external_Z_drift else None)
        return wells, ext

    def _check_drift_domain(self, axes):
        xpts, ypts = axes
        if self.external_Z_drift and xpts.size and ypts.size:
            ax, ay = self.external_Z_array_x, self.external_Z_array_y      # domain check of uk.py:545-551
            if (np.amax(xpts) > np.amax(ax) or np.amin(xpts) < np.amin(ax)
                    or np.amax(ypts) > np.amax(ay) or np.amin(ypts) < np.amin(ay)):
                raise ValueError("External drift array does not cover specified kriging domain.")

    def execute(self, style, xpoints, ypoints, mask=None, backend="cuda", specified_drift_arrays=None,
                dtype="float64", n_gpus=None, values=None):
        """Calculates a kriged grid and the associated variance (uk.py:1090-1328); ``backend='cuda'``.
        point_log and external_Z drift terms are evaluated at the prediction points on the device
        (uk.py:955-971, bilinear sampler uk.py:512-628); 'specified' and 'functional' terms are host
        arrays / host callables by definition and are shipped as columns.

        ``values`` (shape ``(N, V)``, row i for data point i of the constructor) kriges V value fields with this
        object's variogram, anisotropy, drift terms, ``exact_values`` and coordinate type through one factorisation;
        the constructor's values are neither used nor changed, and the variogram is never refitted to ``values``.
        ``zvalues`` then gets a leading field axis (``(V, ...)``; for 'masked' the mask is broadcast over it) and
        ``sigmasq`` keeps its shape, since it does not depend on the values. A 1-D ``values`` of shape ``(N,)``
        returns the usual shapes. float64 only, one GPU, not with ``pseudo_inv=True`` on the global path. Above
        ``KB200_MAX_FIELDS`` (64) fields the call runs in chunks of 64, each with its own factorisation.
        """
        return self._execute(style, (xpoints, ypoints), mask, backend, specified_drift_arrays=specified_drift_arrays,
                             dtype=dtype, n_gpus=n_gpus, values=values)

    def leave_one_out(self, values=None, backend="cuda"):
        """Leave-one-out cross-validation: every station kriged from the other N - 1 stations with this object's fixed
        variogram, anisotropy, ``exact_values`` and drift terms (the drift values at a held-out station are its own row
        of the drift data; the variogram is not refitted per fold). Returns ``(zvalues, sigmasq)`` in station order:
        ``zvalues`` (N,), or (V, N) for a 2-D ``values``; ``sigmasq`` (N,).

        Reads the factorisation the last float64 execute() left on the device (or makes one, which a later execute()
        reuses): O(N^2) on top of it, not N factorisations. ``values`` (shape (N,) or (N, V)) as in
        execute(values=...). Raises ``numpy.linalg.LinAlgError`` naming the station when leaving it out leaves the
        drift terms undetermined, and NotImplementedError with ``pseudo_inv=True``.
        """
        return self._cross_validate(None, None, values, backend)

    def leave_group_out(self, groups, values=None, backend="cuda"):
        """Leave-group-out cross-validation: every station kriged from the stations outside its group, with this
        object's fixed variogram, anisotropy, drift terms and ``exact_values`` (the variogram is not refitted per
        fold). ``groups`` is one label per station (N labels of any type ``numpy.unique`` sorts: k random folds,
        spatial blocks, ...); stations of the same group are held out together. Returns ``(zvalues, sigmasq)`` in station order, shaped as
        leave_one_out(): ``zvalues`` (N,), or (V, N) for a 2-D ``values``; ``sigmasq`` (N,).

        Reads the factorisation the last float64 execute() left on the device (or makes one, which a later execute()
        reuses) and forms C^-1 once: O(N^3 / 3) plus one small solve per group, not one factorisation per group.
        ``values`` as in execute(values=...). Raises ``numpy.linalg.LinAlgError`` naming the group when leaving it
        out leaves the drift terms undetermined, and NotImplementedError with ``pseudo_inv=True``.
        """
        return self._cross_validate(groups, None, values, backend)
