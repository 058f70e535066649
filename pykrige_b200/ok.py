"""OrdinaryKriging (2-D) with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/ok.py:187-1020): same constructor
arguments, public attributes and ``execute`` signature; ``execute`` runs on the GPU
through libkrige_b200.so instead of scipy (no CPU fallback).
"""
import numpy as np  # noqa: F401  (re-exported for callers that reach for ok.np like with the reference module)

from ._base import Krige2D, P_INV_TYPES  # noqa: F401


class OrdinaryKriging(Krige2D):
    """Two-dimensional ordinary kriging; see the reference docstring (ok.py:42-175) for the
    meaning of every argument. Only ``execute(..., backend='cuda')`` differs."""
    _KIND = "2D ordinary kriging"
    _k_before_points = True
    _prints_coordinates_type = True

    def __init__(self, x, y, z, variogram_model="linear", variogram_parameters=None, variogram_function=None, nlags=6,
                 weight=False, anisotropy_scaling=1.0, anisotropy_angle=0.0, verbose=False, enable_plotting=False,
                 enable_statistics=False, coordinates_type="euclidean", exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        self._init_model((x, y), z, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                         (anisotropy_scaling, anisotropy_angle), verbose, enable_plotting, exact_values, pseudo_inv,
                         pseudo_inv_type, coordinates_type=coordinates_type,
                         statistics="eager" if enable_statistics else "off")

    def execute(self, style, xpoints, ypoints, mask=None, backend="cuda", n_closest_points=None, dtype="float64",
                n_gpus=None, values=None):
        """Calculates a kriged grid and the associated variance (ok.py:760-1020).

        ``backend='cuda'`` is the only backend of this package. ``style``, ``mask`` and
        ``n_closest_points`` behave as in the reference, including the exception types.
        ``n_gpus=G`` shards the prediction points over G GPUs of this box from this one host thread.
        Returns ``(zvalues, sigmasq)`` shaped ``(ny, nx)`` for 'grid'/'masked' (masked arrays
        for 'masked') or ``(n,)`` for 'points'.

        ``values`` (shape ``(N, V)``, row i for data point i of the constructor) kriges V value fields with this
        object's variogram, anisotropy, drift terms, ``exact_values`` and coordinate type through one factorisation;
        the constructor's values are neither used nor changed, and the variogram is never refitted to ``values``.
        ``zvalues`` then gets a leading field axis (``(V, ...)``; for 'masked' the mask is broadcast over it) and
        ``sigmasq`` keeps its shape, since it does not depend on the values. A 1-D ``values`` of shape ``(N,)``
        returns the usual shapes. float64 only, one GPU, not with ``pseudo_inv=True`` on the global path. Above
        ``KB200_MAX_FIELDS`` (64) fields the call runs in chunks of 64, each with its own factorisation.
        """
        return self._execute(style, (xpoints, ypoints), mask, backend, n_closest_points=n_closest_points, dtype=dtype,
                             n_gpus=n_gpus, values=values)

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
