"""Variogram plug-in surface of the H100 backend.

Same call signature as the reference's plug-ins — ``f(m, d) -> gamma(d)`` with ``m`` the
*stored* parameter list (partial-sill form) — and the same function ``__name__`` strings,
because the native backends key their model tables on ``__name__``
(reference: src/pykrige/variogram_models.py:25-81, src/pykrige/lib/variogram_models.pyx:5-21).

These numpy versions are used on the host for variogram fitting/plotting only; the
``backend='cuda'`` hot path evaluates the device twins in ``csrc/common.cuh``.
"""
import numpy as np

__all__ = [
    "linear_variogram_model",
    "power_variogram_model",
    "gaussian_variogram_model",
    "exponential_variogram_model",
    "spherical_variogram_model",
    "hole_effect_variogram_model",
    "DEVICE_MODEL_IDS",
]


def linear_variogram_model(m, d):
    """gamma = slope*d + nugget ; m = [slope, nugget]  (variogram_models.py:25-29)"""
    slope, nugget = float(m[0]), float(m[1])
    return nugget + slope * np.asarray(d, dtype=float)


def power_variogram_model(m, d):
    """gamma = scale*d**exponent + nugget ; m = [scale, exponent, nugget]  (variogram_models.py:32-37)"""
    scale, exponent, nugget = float(m[0]), float(m[1]), float(m[2])
    return nugget + scale * np.power(np.asarray(d, dtype=float), exponent)


def gaussian_variogram_model(m, d):
    """gamma = psill*(1 - exp(-d^2/(4r/7)^2)) + nugget ; m = [psill, range, nugget]  (variogram_models.py:40-45)"""
    psill, rng, nugget = float(m[0]), float(m[1]), float(m[2])
    a = rng * 4.0 / 7.0
    d = np.asarray(d, dtype=float)
    return nugget + psill * (1.0 - np.exp(-(d * d) / (a * a)))


def exponential_variogram_model(m, d):
    """gamma = psill*(1 - exp(-d/(r/3))) + nugget ; m = [psill, range, nugget]  (variogram_models.py:48-53)"""
    psill, rng, nugget = float(m[0]), float(m[1]), float(m[2])
    return nugget + psill * (1.0 - np.exp(-np.asarray(d, dtype=float) / (rng / 3.0)))


def spherical_variogram_model(m, d):
    """gamma = psill*(1.5 d/r - 0.5 (d/r)^3) + nugget for d <= r, else psill + nugget  (variogram_models.py:56-70)"""
    psill, rng, nugget = float(m[0]), float(m[1]), float(m[2])
    d = np.asarray(d, dtype=float)
    # same operation order as the reference's expression, (3d)/(2r) - d^3/(2r^3): the soft-L1 fit of
    # core._calculate_variogram_model amplifies a last-ulp difference in this kinked model to ~5e-4 in the parameters
    inside = psill * ((3.0 * d) / (2.0 * rng) - (d**3.0) / (2.0 * rng**3.0)) + nugget
    return np.where(d <= rng, inside, psill + nugget)


def hole_effect_variogram_model(m, d):
    """gamma = psill*(1 - (1 - d/(r/3)) exp(-d/(r/3))) + nugget  (variogram_models.py:73-81)"""
    psill, rng, nugget = float(m[0]), float(m[1]), float(m[2])
    q = np.asarray(d, dtype=float) / (rng / 3.0)
    return nugget + psill * (1.0 - (1.0 - q) * np.exp(-q))


# __name__ -> device model id (include/krige_b200.h KB200_VG_*). Anything else (custom
# callables, GSTools models) has no device twin: NotImplementedError under backend='cuda',
# the same convention as the reference's Cython table (variogram_models.pyx:20-21).
DEVICE_MODEL_IDS = {
    "linear_variogram_model": 0,
    "power_variogram_model": 1,
    "gaussian_variogram_model": 2,
    "exponential_variogram_model": 3,
    "spherical_variogram_model": 4,
    "hole_effect_variogram_model": 5,
}
