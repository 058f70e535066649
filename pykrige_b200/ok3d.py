"""OrdinaryKriging3D with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/ok3d.py:198-932).
"""
from ._base import Krige3D, P_INV_TYPES  # noqa: F401


class OrdinaryKriging3D(Krige3D):
    """Three-dimensional ordinary kriging; arguments as in the reference docstring (ok3d.py:37-196)."""
    _KIND = "3D ordinary kriging"

    def __init__(self, x, y, z, val, variogram_model="linear", variogram_parameters=None, variogram_function=None,
                 nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0, anisotropy_angle_x=0.0,
                 anisotropy_angle_y=0.0, anisotropy_angle_z=0.0, verbose=False, enable_plotting=False,
                 exact_values=True, pseudo_inv=False, pseudo_inv_type="pinv"):
        self._init_model((x, y, z), val, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                         (anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x, anisotropy_angle_y,
                          anisotropy_angle_z), verbose, enable_plotting, exact_values, pseudo_inv, pseudo_inv_type)

    def execute(self, style, xpoints, ypoints, zpoints, mask=None, backend="cuda", n_closest_points=None,
                dtype="float64", n_gpus=None, values=None):
        """Calculates a kriged 3-D grid and the associated variance (ok3d.py:735-932); ``backend='cuda'``.
        Output shape (nz, ny, nx) for 'grid'/'masked', (n,) for 'points'.

        ``values`` (shape ``(N, V)``, row i for data point i of the constructor) kriges V value fields with this
        object's variogram, anisotropy, drift terms, ``exact_values`` and coordinate type through one factorisation;
        the constructor's values are neither used nor changed, and the variogram is never refitted to ``values``.
        ``kvalues`` then gets a leading field axis (``(V, ...)``; for 'masked' the mask is broadcast over it) and
        ``sigmasq`` keeps its shape, since it does not depend on the values. A 1-D ``values`` of shape ``(N,)``
        returns the usual shapes. float64 only, one GPU, not with ``pseudo_inv=True`` on the global path. Above
        ``KB200_MAX_FIELDS`` (64) fields the call runs in chunks of 64, each with its own factorisation.
        """
        return self._execute(style, (xpoints, ypoints, zpoints), mask, backend, n_closest_points=n_closest_points,
                             dtype=dtype, n_gpus=n_gpus, values=values)

    def leave_one_out(self, n_closest_points=None, values=None, backend="cuda"):
        """Leave-one-out cross-validation: every station kriged from the other N - 1 stations with this object's fixed
        variogram, anisotropy, coordinate type and ``exact_values`` (the variogram is not refitted per fold). Returns
        ``(zvalues, sigmasq)`` in station order: ``zvalues`` (N,), or (V, N) for a 2-D ``values``; ``sigmasq`` (N,).
        The residuals are ``values - zvalues`` and the standardised residuals divide them by ``sqrt(sigmasq)``.

        Without ``n_closest_points`` the global path reads the factorisation the last float64 execute() left on the
        device (or makes one, which a later execute() reuses): O(N^2) on top of it, not N factorisations.
        ``n_closest_points = k`` (2 <= k <= N - 1) runs the moving window with k neighbours from the other stations.
        ``values`` (shape (N,) or (N, V)) as in execute(values=...). ``pseudo_inv=True`` is refused on the global path
        (NotImplementedError) and ignored by the moving window, as in execute().
        """
        return self._cross_validate(None, n_closest_points, values, backend)

    def leave_group_out(self, groups, n_closest_points=None, values=None, backend="cuda"):
        """Leave-group-out cross-validation: every station kriged from the stations outside its group, with this
        object's fixed variogram, anisotropy, coordinate type and ``exact_values`` (the variogram is not refitted per
        fold). ``groups`` is one label per station (N labels of any type ``numpy.unique`` sorts: k random folds,
        spatial blocks, ...); stations of the same group are held out together. Returns ``(zvalues, sigmasq)`` in station order, shaped as
        leave_one_out(): ``zvalues`` (N,), or (V, N) for a 2-D ``values``; ``sigmasq`` (N,).

        Without ``n_closest_points`` the global path reads the factorisation the last float64 execute() left on the
        device (or makes one, which a later execute() reuses) and forms C^-1 once: O(N^3 / 3) plus one small solve per
        group, not one factorisation per group. ``n_closest_points = k`` runs the moving window with k neighbours from
        the other groups (2 <= k <= N - size of the largest group). ``values`` as in execute(values=...).
        ``pseudo_inv=True`` is refused on the global path (NotImplementedError) and ignored by the moving window.
        """
        return self._cross_validate(groups, n_closest_points, values, backend)
