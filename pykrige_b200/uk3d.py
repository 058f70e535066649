"""UniversalKriging3D with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/uk3d.py:215-1146): regional-linear drift (three
columns X, Y, Z built on the device), specified and functional drift (host-evaluated columns).
"""
import numpy as np

from ._base import KrigeBase, Krige3D


class UniversalKriging3D(Krige3D):
    """Three-dimensional universal kriging; arguments as in the reference docstring (uk3d.py:37-213)."""
    _POINTS_MSG = dict(KrigeBase._POINTS_MSG)
    _POINTS_MSG[3] = KrigeBase._POINTS_MSG[2]      # uk3d.py:1019-1022 names only xpoints and ypoints

    UNBIAS = True  # uk3d.py:200
    _KIND = "3D Universal kriging"      # capital U as in uk3d.py:1132
    _universal = True

    def __init__(self, x, y, z, val, variogram_model="linear", variogram_parameters=None, variogram_function=None,
                 nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0, anisotropy_angle_x=0.0,
                 anisotropy_angle_y=0.0, anisotropy_angle_z=0.0, drift_terms=None, specified_drift=None,
                 functional_drift=None, verbose=False, enable_plotting=False, exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        if drift_terms is None:
            drift_terms = []
        # no drift term exists yet (see uk.py): constructor-time statistics describe the ordinary-kriging system
        self.regional_linear_drift = self.specified_drift = self.functional_drift = False
        self._init_model((x, y, z), val, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                         (anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x, anisotropy_angle_y,
                          anisotropy_angle_z), verbose, enable_plotting, exact_values, pseudo_inv, pseudo_inv_type)
        if self.verbose:
            print("Initializing drift terms...")
        self.regional_linear_drift = "regional_linear" in drift_terms
        if self.regional_linear_drift and self.verbose:
            print("Implementing regional linear drift.")
        self._init_host_drift_terms(drift_terms, specified_drift, functional_drift)

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
        return self._execute(style, (xpoints, ypoints, zpoints), mask, backend,
                             specified_drift_arrays=specified_drift_arrays, dtype=dtype, n_gpus=n_gpus, values=values)

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
