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
                dtype="float64", n_gpus=None, values=None):
        """Calculates a kriged 3-D grid and the associated variance (uk3d.py:877-1146); ``backend='cuda'``.

        ``values`` (shape ``(N, V)``, row i for data point i of the constructor) kriges V value fields with this
        object's variogram, anisotropy, drift terms, ``exact_values`` and coordinate type through one factorisation;
        the constructor's values are neither used nor changed, and the variogram is never refitted to ``values``.
        ``kvalues`` then gets a leading field axis (``(V, ...)``; for 'masked' the mask is broadcast over it) and
        ``sigmasq`` keeps its shape, since it does not depend on the values. A 1-D ``values`` of shape ``(N,)``
        returns the usual shapes. float64 only, one GPU, not with ``pseudo_inv=True`` on the global path. Above
        ``KB200_MAX_FIELDS`` (64) fields the call runs in chunks of 64, each with its own factorisation.
        """
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

        fields, one = self._check_values(values, dtype, None, n_gpus)
        kvalues, sigmasq = self._run_cuda(style, axes, flat_mask, drift_at=drift_at, dtype=dtype, n_gpus=n_gpus,
                                          **self._fields_kw(fields))
        if one:
            kvalues = kvalues[0]
        return self._shape_output(style, kvalues, sigmasq, sizes, flat_mask)

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
        return self._leave_one_out(None, values, backend, "3D Universal kriging")
