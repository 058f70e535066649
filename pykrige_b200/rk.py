"""Regression kriging: a scikit-learn regressor on the covariates plus kriging of its residuals (reference:
src/pykrige/rk.py).

The regressor models the trend from covariates p, and a `compat.Krige` kriges the residuals y - f(p) at the station
coordinates x. A prediction is f(p) plus the kriged residual. The kriging runs on the device (`Krige`'s default
backend is 'cuda'): the moving window for 'ordinary' / 'ordinary3d' with `n_closest_points`, the global path otherwise.
"""
from .compat import Krige, check_sklearn_model, validate_sklearn

validate_sklearn()

from sklearn.metrics import r2_score  # noqa: E402
from sklearn.svm import SVR  # noqa: E402


class RegressionKriging:
    """Regression kriging (https://en.wikipedia.org/wiki/Regression-Kriging).

    Parameters
    ----------
    regression_model : scikit-learn regressor instance, fitted on the covariates
    method : 'ordinary', 'universal', 'ordinary3d' or 'universal3d'
    variogram_model, nlags, weight, verbose, exact_values, pseudo_inv, pseudo_inv_type, variogram_parameters,
    variogram_function, enable_statistics, coordinates_type, drift_terms, point_drift, functional_drift :
        as in the kriging classes
    n_closest_points : int
        neighbours of the moving window ('ordinary' / 'ordinary3d'; ignored by the universal methods)
    anisotropy_scaling : tuple
        one value in 2-D, two in 3-D
    anisotropy_angle : tuple
        one value in 2-D, three in 3-D
    ext_drift_grid : tuple
        (external_drift, external_drift_x, external_drift_y) of UniversalKriging
    """

    def __init__(self, regression_model=SVR(), method="ordinary", variogram_model="linear", n_closest_points=10,
                 nlags=6, weight=False, verbose=False, exact_values=True, pseudo_inv=False, pseudo_inv_type="pinv",
                 variogram_parameters=None, variogram_function=None, anisotropy_scaling=(1.0, 1.0),
                 anisotropy_angle=(0.0, 0.0, 0.0), enable_statistics=False, coordinates_type="euclidean",
                 drift_terms=None, point_drift=None, ext_drift_grid=(None, None, None), functional_drift=None):
        check_sklearn_model(regression_model)
        self.regression_model = regression_model
        self.n_closest_points = n_closest_points
        self.krige = Krige(method=method, variogram_model=variogram_model, nlags=nlags, weight=weight,
                           n_closest_points=n_closest_points, verbose=verbose, exact_values=exact_values,
                           pseudo_inv=pseudo_inv, pseudo_inv_type=pseudo_inv_type,
                           variogram_parameters=variogram_parameters, variogram_function=variogram_function,
                           anisotropy_scaling=anisotropy_scaling, anisotropy_angle=anisotropy_angle,
                           enable_statistics=enable_statistics, coordinates_type=coordinates_type,
                           drift_terms=drift_terms, point_drift=point_drift, ext_drift_grid=ext_drift_grid,
                           functional_drift=functional_drift)

    def fit(self, p, x, y):
        """Fits the regressor on (p, y), then the kriging of its residuals at the stations.

        p : (Ns, d) covariates; x : (Ns, 2) or (Ns, 3) station coordinates; y : (Ns,) targets
        """
        self.regression_model.fit(p, y)
        trend = self.regression_model.predict(p)
        print("Finished learning regression model")
        self.krige.fit(x=x, y=y - trend)
        print("Finished kriging residuals")

    def predict(self, p, x, **kwargs):
        """The regressor's prediction at covariates p plus the residual kriged at coordinates x, shape (Ns,).
        kwargs go to the kriging object's execute()."""
        return self.krige_residual(x, **kwargs) + self.regression_model.predict(p)

    def krige_residual(self, x, **kwargs):
        """The residual kriged at the (Ns, 2) or (Ns, 3) coordinates x."""
        return self.krige.predict(x, **kwargs)

    def score(self, p, x, y, sample_weight=None, **kwargs):
        """Coefficient of determination R^2 of predict(p, x) against y."""
        return r2_score(y_pred=self.predict(p, x, **kwargs), y_true=y, sample_weight=sample_weight)
