"""OrdinaryKriging (2-D) with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/ok.py:187-1020): same constructor
arguments, public attributes and ``execute`` signature; ``execute`` runs on the GPU
through libkrige_b200.so instead of scipy (no CPU fallback).
"""
import numpy as np  # noqa: F401  (re-exported for callers that reach for ok.np like with the reference module)

from ._base import KrigeBase
from ._krige2d import Krige2DMixin, P_INV_TYPES  # noqa: F401


class OrdinaryKriging(Krige2DMixin, KrigeBase):
    """Two-dimensional ordinary kriging; see the reference docstring (ok.py:42-175) for the
    meaning of every argument. Only ``execute(..., backend='cuda')`` differs."""
    _prints_coordinates_type = True

    def __init__(self, x, y, z, variogram_model="linear", variogram_parameters=None, variogram_function=None, nlags=6,
                 weight=False, anisotropy_scaling=1.0, anisotropy_angle=0.0, verbose=False, enable_plotting=False,
                 enable_statistics=False, coordinates_type="euclidean", exact_values=True, pseudo_inv=False,
                 pseudo_inv_type="pinv"):
        self._init_common_2d(x, y, z, variogram_model, variogram_parameters, variogram_function, nlags, weight,
                             anisotropy_scaling, anisotropy_angle, verbose, enable_plotting, exact_values, pseudo_inv,
                             pseudo_inv_type, coordinates_type=coordinates_type,
                             statistics="eager" if enable_statistics else "off")

    def execute(self, style, xpoints, ypoints, mask=None, backend="cuda", n_closest_points=None, dtype="float64",
                n_gpus=None):
        """Calculates a kriged grid and the associated variance (ok.py:760-1020).

        ``backend='cuda'`` is the only backend of this package. ``style``, ``mask`` and
        ``n_closest_points`` behave as in the reference, including the exception types.
        ``n_gpus=G`` shards the prediction points over G GPUs of this box from this one host thread.
        Returns ``(zvalues, sigmasq)`` shaped ``(ny, nx)`` for 'grid'/'masked' (masked arrays
        for 'masked') or ``(n,)`` for 'points'.
        """
        if self.verbose:
            print("Executing Ordinary Kriging...\n")
        if style != "grid" and style != "masked" and style != "points":
            raise ValueError("style argument must be 'grid', 'points', or 'masked'")
        if n_closest_points is not None and n_closest_points <= 1:
            raise ValueError("n_closest_points has to be at least two!")
        axes, sizes, flat_mask = self._prepare_points(style, (xpoints, ypoints), mask)
        self._check_backend(backend, "2D ordinary kriging")
        zvalues, sigmasq = self._run_cuda(style, axes, flat_mask, n_closest_points=n_closest_points, dtype=dtype,
                                          n_gpus=n_gpus)
        return self._shape_output(style, zvalues, sigmasq, sizes, flat_mask)
