"""UniversalKriging (2-D) with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/uk.py:220-1328). Regional-linear drift is built
on the device from the adjusted coordinates. The DATA-side columns of the other drift kinds
(uk.py:884-910) are evaluated once on the host and enter the device system as extra columns;
at the PREDICTION points point-log and external-Z (uk.py:955-971) are evaluated inside the solve
kernels (kb200_set_device_drift), only specified / functional values (uk.py:972-979) are shipped.
"""
import numpy as np

from ._base import KrigeBase
from ._krige2d import Krige2DMixin, P_INV_TYPES  # noqa: F401
from .core import _adjust_for_anisotropy


def _first_last_index(axis, v):
    """(index of the first node >= v, index of the last node <= v) for every v — the node
    selection rule of the reference's bilinear sampler (uk.py:556-559)."""
    axis = np.asarray(axis, dtype=float)
    ge = axis[None, :] >= v[:, None]
    le = axis[None, :] <= v[:, None]
    i2 = np.argmax(ge, axis=1)
    i1 = axis.size - 1 - np.argmax(le[:, ::-1], axis=1)
    return i1, i2


class UniversalKriging(Krige2DMixin, KrigeBase):
    """Two-dimensional universal kriging; arguments as in the reference docstring (uk.py:40-205)."""

    UNBIAS = True  # the unbiasedness row is always present on the device path (uk.py:208)

    def __init__(self, x, y, z, variogram_model="linear", variogram_parameters=None, variogram_function=None, nlags=6,
                 weight=False, anisotropy_scaling=1.0, anisotropy_angle=0.0, drift_terms=None, point_drift=None,
                 external_drift=None, external_drift_x=None, external_drift_y=None, specified_drift=None,
                 functional_drift=None, verbose=False, enable_plotting=False, exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        if drift_terms is None:
            drift_terms = []
        if specified_drift is None:
            specified_drift = []
        if functional_drift is None:
            functional_drift = []
        # no drift term exists yet: the statistics the common body may compute (verbose=True) are those of the
        # ordinary-kriging system, as in the reference, where they precede the drift initialisation (uk.py:380-394)
        self.regional_linear_drift = self.external_Z_drift = self.point_log_drift = False
        self.specified_drift = self.functional_drift = False
        self._init_common_2d(x, y, z, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                             anisotropy_scaling, anisotropy_angle, verbose, enable_plotting, exact_values, pseudo_inv,
                             pseudo_inv_type, coordinates_type="euclidean", statistics="lazy")

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
            self.point_log_array[:, :2] = _adjust_for_anisotropy(
                np.vstack((point_log[:, 0], point_log[:, 1])).T,
                [self.XCENTER, self.YCENTER],
                [self.anisotropy_scaling],
                [self.anisotropy_angle],
            )
            if self.verbose:
                print("Implementing external point-logarithmic drift; number of points =",
                      self.point_log_array.shape[0], "\n")
        else:
            self.point_log_drift = False

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

        # functional drift: callables evaluated with the adjusted coordinates (uk.py:496-510)
        if "functional" in drift_terms:
            if type(functional_drift) is not list:
                raise TypeError("Callables for functional drift terms must be encapsulated in a list.")
            if len(functional_drift) == 0:
                raise ValueError("Must provide at least one callable object when using the 'functional' drift capability.")
            self.functional_drift = True
            self.functional_drift_terms = functional_drift
        else:
            self.functional_drift = False

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

    def _device_drift_signature(self):
        """point_log wells and the external-Z raster are evaluated at the prediction points by the solve
        kernels themselves (kb200_set_device_drift); their content is part of the problem key."""
        import hashlib
        hsh = hashlib.blake2b(digest_size=16)
        if self.point_log_drift:
            hsh.update(np.ascontiguousarray(self.point_log_array, dtype=np.float64).tobytes())
        if self.external_Z_drift:
            for a in (self.external_Z_array_x, self.external_Z_array_y, self.external_Z_array):
                hsh.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
        return (bool(self.point_log_drift), bool(self.external_Z_drift), hsh.hexdigest())

    def _configure_device_drift(self, h):
        wells = self.point_log_array if self.point_log_drift else None
        ext = ((self.external_Z_array_x, self.external_Z_array_y, self.external_Z_array)
               if self.external_Z_drift else None)
        h.set_device_drift(wells, ext)

    def execute(self, style, xpoints, ypoints, mask=None, backend="cuda", specified_drift_arrays=None,
                dtype="float64", n_gpus=None):
        """Calculates a kriged grid and the associated variance (uk.py:1090-1328); ``backend='cuda'``.
        point_log and external_Z drift terms are evaluated at the prediction points on the device
        (uk.py:955-971, bilinear sampler uk.py:512-628); 'specified' and 'functional' terms are host
        arrays / host callables by definition and are shipped as columns."""
        if self.verbose:
            print("Executing Universal Kriging...\n")
        axes, sizes, flat_mask = self._prepare_points(style, (xpoints, ypoints), mask)
        xpts, ypts = axes
        spec_drift_grids = self._specified_drift_grids(style, specified_drift_arrays, sizes, xpts.size,
                                                       "UniversalKriging")
        self._check_backend(backend, "2D universal kriging")
        if self.external_Z_drift and xpts.size and ypts.size:
            ax, ay = self.external_Z_array_x, self.external_Z_array_y      # domain check of uk.py:545-551
            if (np.amax(xpts) > np.amax(ax) or np.amin(xpts) < np.amin(ax)
                    or np.amax(ypts) > np.amax(ay) or np.amin(ypts) < np.amin(ay)):
                raise ValueError("External drift array does not cover specified kriging domain.")

        drift_at = None
        if self.specified_drift or self.functional_drift:
            def drift_at(pts, idx):
                cols = []
                if self.specified_drift:
                    for g in spec_drift_grids:
                        flat = np.asarray(g, dtype=float).flatten()
                        cols.append(flat if idx is None else flat[idx])
                if self.functional_drift:
                    xa, ya = _adjust_for_anisotropy(
                        np.vstack((pts[0], pts[1])).T, [self.XCENTER, self.YCENTER],
                        [self.anisotropy_scaling], [self.anisotropy_angle]).T
                    for func in self.functional_drift_terms:
                        cols.append(np.asarray(func(xa, ya), dtype=float) * np.ones(xa.shape))
                return np.ascontiguousarray(np.vstack(cols), dtype=np.float64)

        zvalues, sigmasq = self._run_cuda(style, axes, flat_mask, drift_at=drift_at, dtype=dtype, n_gpus=n_gpus)
        return self._shape_output(style, zvalues, sigmasq, sizes, flat_mask)
