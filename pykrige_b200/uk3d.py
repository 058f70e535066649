"""UniversalKriging3D with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/uk3d.py:215-1146): regional-linear drift (three
columns X, Y, Z built on the device), specified and functional drift (host-evaluated columns).
"""
import numpy as np

from ._base import KrigeBase
from .core import _adjust_for_anisotropy
from .ok3d import _Krige3DMixin


class UniversalKriging3D(_Krige3DMixin, KrigeBase):
    """Three-dimensional universal kriging; arguments as in the reference docstring (uk3d.py:37-213)."""
    _POINTS_MSG = dict(KrigeBase._POINTS_MSG)
    _POINTS_MSG[3] = KrigeBase._POINTS_MSG[2]      # uk3d.py:1019-1022 names only xpoints and ypoints

    UNBIAS = True  # uk3d.py:200

    def __init__(self, x, y, z, val, variogram_model="linear", variogram_parameters=None, variogram_function=None,
                 nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0, anisotropy_angle_x=0.0,
                 anisotropy_angle_y=0.0, anisotropy_angle_z=0.0, drift_terms=None, specified_drift=None,
                 functional_drift=None, verbose=False, enable_plotting=False, exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        if drift_terms is None:
            drift_terms = []
        if specified_drift is None:
            specified_drift = []
        if functional_drift is None:
            functional_drift = []
        # no drift term exists yet (see uk.py): constructor-time statistics describe the ordinary-kriging system
        self.regional_linear_drift = self.specified_drift = self.functional_drift = False
        self._init_common_3d(x, y, z, val, variogram_model, variogram_parameters, variogram_function, nlags,
                             weight, anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x,
                             anisotropy_angle_y, anisotropy_angle_z, verbose, enable_plotting, exact_values,
                             pseudo_inv, pseudo_inv_type)
        if self.verbose:
            print("Initializing drift terms...")
        self.regional_linear_drift = "regional_linear" in drift_terms
        if self.regional_linear_drift and self.verbose:
            print("Implementing regional linear drift.")
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
        if "functional" in drift_terms:
            if type(functional_drift) is not list:
                raise TypeError("Callables for functional drift terms must be encapsulated in a list.")
            if len(functional_drift) == 0:
                raise ValueError("Must provide at least one callable object when using the 'functional' drift capability.")
            self.functional_drift = True
            self.functional_drift_terms = functional_drift
        else:
            self.functional_drift = False

    def _drift_spec(self):
        """Host-evaluated drift columns at the data in the reference's order (uk3d.py:718-727)."""
        cols = []
        if self.specified_drift:
            for arr in self.specified_drift_data_arrays:
                cols.append(np.asarray(arr, dtype=float))
        if self.functional_drift:
            for func in self.functional_drift_terms:
                cols.append(np.asarray(func(self.X_ADJUSTED, self.Y_ADJUSTED, self.Z_ADJUSTED), dtype=float))
        return (3 if self.regional_linear_drift else 0), cols

    def execute(self, style, xpoints, ypoints, zpoints, mask=None, backend="cuda", specified_drift_arrays=None,
                dtype="float64", n_gpus=None):
        """Calculates a kriged 3-D grid and the associated variance (uk3d.py:877-1146); ``backend='cuda'``."""
        if self.verbose:
            print("Executing Universal Kriging...\n")
        axes, sizes, flat_mask = self._prepare_points(style, (xpoints, ypoints, zpoints), mask)
        spec_drift_grids = self._specified_drift_grids(style, specified_drift_arrays, sizes, axes[0].size,
                                                       "UniversalKriging3D")
        self._check_backend(backend, "3D Universal kriging")   # capital U as in uk3d.py:1132

        drift_at = None
        if self.specified_drift or self.functional_drift:
            def drift_at(pts, idx):
                cols = []
                if self.specified_drift:
                    for g in spec_drift_grids:
                        flat = np.asarray(g, dtype=float).flatten()
                        cols.append(flat if idx is None else flat[idx])
                if self.functional_drift:
                    xa, ya, za = _adjust_for_anisotropy(
                        np.vstack((pts[0], pts[1], pts[2])).T,
                        [self.XCENTER, self.YCENTER, self.ZCENTER],
                        [self.anisotropy_scaling_y, self.anisotropy_scaling_z],
                        [self.anisotropy_angle_x, self.anisotropy_angle_y, self.anisotropy_angle_z]).T
                    for func in self.functional_drift_terms:
                        cols.append(np.asarray(func(xa, ya, za), dtype=float) * np.ones(xa.shape))
                return np.ascontiguousarray(np.vstack(cols), dtype=np.float64)

        kvalues, sigmasq = self._run_cuda(style, axes, flat_mask, drift_at=drift_at, dtype=dtype, n_gpus=n_gpus)
        return self._shape_output(style, kvalues, sigmasq, sizes, flat_mask)
