"""scikit-learn estimator around the four kriging classes, routed to ``backend='cuda'``.

The caller side of the hot path in the reference (src/pykrige/compat.py:97-291): ``Krige.fit`` builds
the kriging object, ``Krige.predict`` calls ``execute(style='points', backend=..., n_closest_points=...)``.
The reference hard-codes ``backend='loop'`` (compat.py:283); here the default is ``'cuda'``. Works with
``GridSearchCV`` / ``RandomizedSearchCV`` like the original (tests/test_api.py:15-47).
"""
import numpy as np

from .ok import OrdinaryKriging
from .uk import UniversalKriging
from .ok3d import OrdinaryKriging3D
from .uk3d import UniversalKriging3D

try:
    from sklearn.base import BaseEstimator, ClassifierMixin, RegressorMixin

    SKLEARN_INSTALLED = True
except ImportError:  # pragma: no cover
    SKLEARN_INSTALLED = False

    class RegressorMixin:  # minimal stand-ins so the class can be defined
        pass

    class ClassifierMixin:
        pass

    class BaseEstimator:
        pass


krige_methods = {
    "ordinary": OrdinaryKriging,
    "universal": UniversalKriging,
    "ordinary3d": OrdinaryKriging3D,
    "universal3d": UniversalKriging3D,
}
threed_krige = ("ordinary3d", "universal3d")

# constructor keywords each method understands beyond the common ones (compat.py:41-74)
krige_methods_kws = {
    "ordinary": ["anisotropy_scaling", "anisotropy_angle", "enable_statistics", "coordinates_type"],
    "universal": ["anisotropy_scaling", "anisotropy_angle", "drift_terms", "point_drift", "external_drift",
                  "external_drift_x", "external_drift_y", "functional_drift"],
    "ordinary3d": ["anisotropy_scaling_y", "anisotropy_scaling_z", "anisotropy_angle_x", "anisotropy_angle_y",
                   "anisotropy_angle_z"],
    "universal3d": ["anisotropy_scaling_y", "anisotropy_scaling_z", "anisotropy_angle_x", "anisotropy_angle_y",
                    "anisotropy_angle_z", "drift_terms", "functional_drift"],
}


class SklearnException(Exception):
    """scikit-learn is needed but not installed."""


def validate_method(method):
    if method not in krige_methods:
        raise ValueError("Kriging method must be one of {}".format(krige_methods.keys()))


def validate_sklearn():
    """Raises SklearnException without scikit-learn (compat.py:89-94): rk.py and ck.py call it on import."""
    if not SKLEARN_INSTALLED:
        raise SklearnException("sklearn needs to be installed in order to use this module")


def check_sklearn_model(model, task="regression"):
    """RuntimeError unless `model` is a scikit-learn estimator of the given task, 'regression' or 'classification'
    (compat.py:294-307)."""
    mixin = {"regression": RegressorMixin, "classification": ClassifierMixin}.get(task)
    if mixin is not None and not (isinstance(model, BaseEstimator) and isinstance(model, mixin)):
        raise RuntimeError("Needs to supply an instance of a scikit-learn %s class." % task)


class Krige(RegressorMixin, BaseEstimator):
    """scikit-learn wrapper for ordinary / universal kriging in 2-D and 3-D (compat.py:97-180)."""

    def __init__(self, method="ordinary", variogram_model="linear", nlags=6, weight=False, n_closest_points=10,
                 verbose=False, exact_values=True, pseudo_inv=False, pseudo_inv_type="pinv",
                 variogram_parameters=None, variogram_function=None, anisotropy_scaling=(1.0, 1.0),
                 anisotropy_angle=(0.0, 0.0, 0.0), enable_statistics=False, coordinates_type="euclidean",
                 drift_terms=None, point_drift=None, ext_drift_grid=(None, None, None), functional_drift=None,
                 backend="cuda"):
        validate_method(method)
        self.method = method
        self.variogram_model = variogram_model
        self.nlags = nlags
        self.weight = weight
        self.n_closest_points = n_closest_points
        self.verbose = verbose
        self.exact_values = exact_values
        self.pseudo_inv = pseudo_inv
        self.pseudo_inv_type = pseudo_inv_type
        self.variogram_parameters = variogram_parameters
        self.variogram_function = variogram_function
        self.anisotropy_scaling = anisotropy_scaling
        self.anisotropy_angle = anisotropy_angle
        self.enable_statistics = enable_statistics
        self.coordinates_type = coordinates_type
        self.drift_terms = drift_terms
        self.point_drift = point_drift
        self.ext_drift_grid = ext_drift_grid
        self.functional_drift = functional_drift
        self.backend = backend
        self.model = None

    def fit(self, x, y, *args, **kwargs):
        """x: (N, 2) or (N, 3) points, y: (N,) targets (compat.py:181-233)."""
        x = np.asarray(x)
        val_kw = "val" if self.method in threed_krige else "z"
        setup = dict(variogram_model=self.variogram_model, variogram_parameters=self.variogram_parameters,
                     variogram_function=self.variogram_function, nlags=self.nlags, weight=self.weight,
                     verbose=self.verbose, exact_values=self.exact_values, pseudo_inv=self.pseudo_inv,
                     pseudo_inv_type=self.pseudo_inv_type)
        extra = dict(anisotropy_scaling=self.anisotropy_scaling[0], anisotropy_angle=self.anisotropy_angle[0],
                     enable_statistics=self.enable_statistics, coordinates_type=self.coordinates_type,
                     anisotropy_scaling_y=self.anisotropy_scaling[0], anisotropy_scaling_z=self.anisotropy_scaling[1],
                     anisotropy_angle_x=self.anisotropy_angle[0], anisotropy_angle_y=self.anisotropy_angle[1],
                     anisotropy_angle_z=self.anisotropy_angle[2], drift_terms=self.drift_terms,
                     point_drift=self.point_drift, external_drift=self.ext_drift_grid[0],
                     external_drift_x=self.ext_drift_grid[1], external_drift_y=self.ext_drift_grid[2],
                     functional_drift=self.functional_drift)
        for kw in krige_methods_kws[self.method]:
            setup[kw] = extra[kw]
        kw = self._dimensionality_check(x)
        kw.update(setup)
        kw[val_kw] = y
        self.model = krige_methods[self.method](**kw)
        return self

    def _dimensionality_check(self, x, ext=""):
        want = 3 if self.method in threed_krige else 2
        if x.shape[1] != want:
            raise ValueError("%dd krige can use only %dd points" % (want, want))
        names = ("x", "y", "z")[:want]
        return {nm + ext: x[:, i] for i, nm in enumerate(names)}

    def predict(self, x, *args, **kwargs):
        """Kriged values at the (N, 2|3) points x (compat.py:251-269)."""
        if not self.model:
            raise Exception("Not trained. Train first")
        points = self._dimensionality_check(np.asarray(x), ext="points")
        return self.execute(points, *args, **kwargs)[0]

    def execute(self, points, *args, **kwargs):
        """(prediction, variance) for a dict of xpoints/ypoints[/zpoints] (compat.py:271-291)."""
        call = dict(style="points", backend=self.backend)
        call.update(kwargs)
        points.update(call)
        if isinstance(self.model, (OrdinaryKriging, OrdinaryKriging3D)):
            points.update(dict(n_closest_points=self.n_closest_points))
        elif self.verbose:
            print("n_closest_points will be ignored for UniversalKriging")
        return self.model.execute(**points)
