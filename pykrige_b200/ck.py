"""Classification kriging: a scikit-learn classifier plus kriging of its residuals in isometric log-ratio coordinates
(reference: src/pykrige/ck.py).

The class probabilities of the classifier and the one-hot targets are compositions of C parts. Their isometric
log-ratio (ilr) transforms are C - 1 real coordinates, and each coordinate of the residual (targets minus classifier)
is kriged at the station coordinates. A prediction adds the kriged residual to the classifier's ilr coordinates, maps
the sum back to probabilities and takes the most probable class.

The C - 1 kriging problems share the stations and all kriging options and differ only in their values. When the
variogram is fixed (`variogram_parameters` given) they also share the variogram, and `krige_residual` kriges the C - 1
residual columns as value fields of one problem, `execute(values=R)`: one factorisation or one moving-window pass
instead of C - 1. Each field's result is bit-identical to the single-field call with that column (DESIGN.md §5d), so
the result does not depend on which route ran.
"""
import numpy as np

from .compat import Krige, check_sklearn_model, validate_sklearn

validate_sklearn()

from scipy.linalg import helmert  # noqa: E402
from sklearn.metrics import accuracy_score  # noqa: E402
from sklearn.svm import SVC  # noqa: E402


class ClassificationKriging:
    """Classification kriging: simplicial indicator kriging of the ilr residuals of a classifier.

    Parameters
    ----------
    classification_model : scikit-learn classifier instance with predict_proba, fitted on the covariates
    method : 'ordinary', 'universal', 'ordinary3d' or 'universal3d'
    variogram_model, nlags, weight, verbose, exact_values, pseudo_inv, pseudo_inv_type, variogram_parameters,
    variogram_function, enable_statistics, coordinates_type, drift_terms, point_drift, functional_drift :
        as in the kriging classes; with `variogram_parameters` given every class uses that variogram, otherwise
        each class fits its own
    n_closest_points : int
        neighbours of the moving window ('ordinary' / 'ordinary3d'; ignored by the universal methods)
    anisotropy_scaling : tuple
        one value in 2-D, two in 3-D
    anisotropy_angle : tuple
        one value in 2-D, three in 3-D
    ext_drift_grid : tuple
        (external_drift, external_drift_x, external_drift_y) of UniversalKriging

    Attributes after fit: `classes_` (the classifier's classes) and `krige`, a list of C - 1 fitted `Krige`
    objects, one per ilr coordinate.
    """

    def __init__(self, classification_model=SVC(), method="ordinary", variogram_model="linear", n_closest_points=10,
                 nlags=6, weight=False, verbose=False, exact_values=True, pseudo_inv=False, pseudo_inv_type="pinv",
                 variogram_parameters=None, variogram_function=None, anisotropy_scaling=(1.0, 1.0),
                 anisotropy_angle=(0.0, 0.0, 0.0), enable_statistics=False, coordinates_type="euclidean",
                 drift_terms=None, point_drift=None, ext_drift_grid=(None, None, None), functional_drift=None):
        check_sklearn_model(classification_model, task="classification")
        self.classification_model = classification_model
        self.n_closest_points = n_closest_points
        self._kriging_kwargs = dict(
            method=method, variogram_model=variogram_model, nlags=nlags, weight=weight,
            n_closest_points=n_closest_points, verbose=verbose, exact_values=exact_values, pseudo_inv=pseudo_inv,
            pseudo_inv_type=pseudo_inv_type, variogram_parameters=variogram_parameters,
            variogram_function=variogram_function, anisotropy_scaling=anisotropy_scaling,
            anisotropy_angle=anisotropy_angle, enable_statistics=enable_statistics, coordinates_type=coordinates_type,
            drift_terms=drift_terms, point_drift=point_drift, ext_drift_grid=ext_drift_grid,
            functional_drift=functional_drift)

    def fit(self, p, x, y):
        """Fits the classifier on (p, y), then one kriging of the ilr residual per coordinate at the stations.

        p : (Ns, d) covariates; x : (Ns, 2) or (Ns, 3) station coordinates; y : (Ns, 1) class labels
        """
        self.classification_model.fit(p, np.ravel(y))
        print("Finished learning classification model")
        self.classes_ = self.classification_model.classes_
        self.krige = [Krige(**self._kriging_kwargs) for _ in range(len(self.classes_) - 1)]
        one_hot = (np.reshape(y, (-1, 1)) == np.reshape(self.classes_, (1, -1))).astype(np.float64)
        self._residuals = (ilr_transformation(one_hot)
                           - ilr_transformation(self.classification_model.predict_proba(p)))
        for i, k in enumerate(self.krige):
            k.fit(x=x, y=self._residuals[:, i])
        print("Finished kriging residuals")

    def predict(self, p, x, **kwargs):
        """Index (into `classes_`) of the most probable class at covariates p and coordinates x, shape (Ns,).
        kwargs go to the kriging objects' execute()."""
        ilr = self.krige_residual(x, **kwargs) + ilr_transformation(self.classification_model.predict_proba(p))
        return np.argmax(inverse_ilr_transformation(ilr), axis=1)

    def krige_residual(self, x, **kwargs):
        """The C - 1 ilr residual coordinates kriged at the (Ns, 2) or (Ns, 3) coordinates x, shape (Ns, C - 1)."""
        if self._shares_one_problem(kwargs):
            k = self.krige[0]
            z = k.execute(k._dimensionality_check(np.asarray(x), ext="points"), values=self._residuals, **kwargs)[0]
            return np.asarray(z).T
        return np.vstack([k.predict(x=x, **kwargs) for k in self.krige]).T

    def _shares_one_problem(self, kwargs):
        """Whether the residual columns can be kriged as value fields of one problem: the variogram is fixed (else
        each class fits its own), and neither pseudo_inv on the global path nor a dtype or n_gpus that value fields
        refuse (`_base.KrigeBase._check_values`) is in play."""
        kw = self._kriging_kwargs
        moving_window = kw["method"] in ("ordinary", "ordinary3d") and kw["n_closest_points"] is not None
        return (kw["variogram_parameters"] is not None
                and (moving_window or not kw["pseudo_inv"])
                and kwargs.get("dtype", "float64") == "float64"
                and kwargs.get("n_gpus") in (None, 1))

    def score(self, p, x, y, sample_weight=None, **kwargs):
        """Accuracy of predict(p, x) against the labels y."""
        return accuracy_score(y_pred=self.predict(p, x, **kwargs), y_true=y, sample_weight=sample_weight)


def closure(data, k=1.0):
    """Scales each row of data (n_samples, n_parts) to sum to k. Rows summing to zero give nan and inf."""
    return k * data / np.sum(data, axis=1, keepdims=True)


def ilr_transformation(data):
    """Isometric log-ratio coordinates (n_samples, D - 1) of compositions data (n_samples, D).

    Parts are clipped at machine epsilon, so zero probabilities are allowed. The basis is the negated, transposed
    Helmert matrix without its first row: coordinate j contrasts part j + 1 with the geometric mean of parts 0..j.
    (Pawlowsky-Glahn, Egozcue & Tolosana-Delgado, Modelling and Analysis of Compositional Data, 2015, p. 37.)
    """
    # einsum, not matmul: its summation order gives PyKrige's bits, and the automatic variogram fit of the residuals
    # turns a last-ulp difference here into a relative 1e-3 in near-zero fitted parameters
    basis = -helmert(np.shape(data)[1]).T
    return np.einsum("np,pc->nc", np.log(np.maximum(data, np.finfo(float).eps)), basis)


def inverse_ilr_transformation(data):
    """Closed compositions (n_samples, D + 1) of ilr coordinates data (n_samples, D): the inverse of
    ilr_transformation for compositions without parts below machine epsilon."""
    basis = -helmert(np.shape(data)[1] + 1)
    return closure(np.exp(np.einsum("nc,cp->np", data, basis)))
