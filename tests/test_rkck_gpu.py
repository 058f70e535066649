"""GPU tests of RegressionKriging and ClassificationKriging: the fixtures of the imported reference through the device
at the parity tolerance of tests/test_parity_gpu.py, the reference's own score thresholds, and the two routes of
ClassificationKriging.krige_residual (C - 1 single-field problems, or one problem with C - 1 value fields) bit for bit
on the moving window and on the global path."""
import warnings

import numpy as np
import pytest
from numpy.testing import assert_array_equal

import rkck_cases as rc
from test_rkck_host import check_against_fixture, fixture_data, ref, same_platform  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

R64 = 1e-5


@pytest.mark.parametrize("case", rc.CASES, ids=[c["name"] for c in rc.CASES])
def test_fixture_cases_on_the_device(case, ref, capsys):  # noqa: F811
    d = fixture_data(ref, case)
    model = rc.make("pykrige_b200", case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model.fit(d["p_train"], d["x_train"], d["y_train"])
        out = capsys.readouterr().out
        check_against_fixture(model, case, ref, d, R64, stdout=out, exact=same_platform(ref))
    if case["kind"] == "ck":
        shared = case["fixed"] and not case["pseudo_inv"]
        assert model.krige[0].model._kb_handle.n_fields == (len(model.classes_) - 1 if shared else 0)
        if case["pseudo_inv"]:                  # universal kriging with pseudo_inv: the per-class route on the device
            assert all(k.model._kb_handle.n_fields == 0 for k in model.krige)


@pytest.mark.parametrize("kind", ["rk", "ck"])
def test_reference_score_thresholds(kind, capsys):
    """tests/test_regression_krige.py / test_classification_krige.py of the reference, on its un-jittered lattice:
    score > 0.25 for each estimator with 'ordinary' (moving window, n_closest_points=2) and 'universal'."""
    from sklearn.ensemble import RandomForestClassifier, RandomForestRegressor
    from sklearn.linear_model import ElasticNet, Lasso, LinearRegression
    from sklearn.svm import SVC, SVR
    from pykrige_b200.ck import ClassificationKriging
    from pykrige_b200.rk import RegressionKriging
    if kind == "rk":
        d = rc.split(*rc.reference_data())
        ests = [lambda: SVR(C=0.01, gamma="auto"),
                lambda: RandomForestRegressor(min_samples_split=5, n_estimators=50, random_state=0),
                LinearRegression, Lasso, ElasticNet]
    else:
        d = rc.split(*rc.reference_data(n_classes=5))
        ests = [lambda: SVC(C=0.01, gamma="auto", probability=True, random_state=0),
                lambda: RandomForestClassifier(n_estimators=50, random_state=0)]
    for make in ests:
        for method in ("ordinary", "universal"):
            if kind == "rk":
                m = RegressionKriging(regression_model=make(), method=method, n_closest_points=2)
            else:
                m = ClassificationKriging(classification_model=make(), method=method, n_closest_points=2)
            m.fit(d["p_train"], d["x_train"], d["y_train"])
            assert m.score(d["p_test"], d["x_test"], d["y_test"]) > 0.25, (kind, method, make)


def _many_classes(n_classes, n=600, seed=3):
    """Stations with n_classes labels that depend on the covariates and on position."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 1000.0, size=(n, 2))
    p = np.column_stack([x / 1000.0 + rng.normal(scale=0.1, size=(n, 2)), rng.normal(size=(n, 2))])
    score = 3.0 * p[:, 0] + 2.0 * p[:, 1] + np.sin(x[:, 0] / 150.0) + 0.3 * rng.normal(size=n)
    edges = np.quantile(score, np.linspace(0.0, 1.0, n_classes + 1)[1:-1])
    return p, x, np.digitize(score, edges).astype(np.float64).reshape(-1, 1)


ROUTES = [(c, method, k) for c in (3, 5, 66) for method, k in (("ordinary", 10), ("ordinary", None), ("universal", 10))]


@pytest.mark.parametrize("n_classes,method,k", ROUTES, ids=["c%d_%s_k%s" % r for r in ROUTES])
def test_shared_route_is_the_per_class_route_bit_for_bit(n_classes, method, k, monkeypatch, capsys):
    """C - 1 = 2, 4 and 65 ilr coordinates (65 exceeds the 64 fields of one problem, so the shared route runs two
    chunks) on the moving window and the global path (ordinary without n_closest_points; universal)."""
    from sklearn.ensemble import RandomForestClassifier
    from pykrige_b200.ck import ClassificationKriging
    p, x, y = _many_classes(n_classes)
    model = ClassificationKriging(classification_model=RandomForestClassifier(n_estimators=20, random_state=0),
                                  method=method, n_closest_points=k, variogram_model="spherical",
                                  variogram_parameters=[1.0, 250.0, 0.05])
    model.fit(p[:500], x[:500], y[:500])
    assert len(model.classes_) == n_classes and model._shares_one_problem({})
    q = np.vstack([x[500:], x[:20]])                # new points and exact hits of stations
    shared = model.krige_residual(q)
    assert model.krige[0].model._kb_handle.n_fields > 0
    with monkeypatch.context() as m:
        m.setattr(ClassificationKriging, "_shares_one_problem", lambda self, kwargs: False)
        per_class = model.krige_residual(q)
        pred_per_class = model.predict(p[500:], x[500:])
    assert shared.shape == per_class.shape == (q.shape[0], n_classes - 1)
    assert_array_equal(shared, per_class)
    assert_array_equal(model.predict(p[500:], x[500:]), pred_per_class)


def test_drop_in_for_the_reference_examples(capsys):
    """examples/07_regression_kriging2d.py and 10_classification_kriging2d.py of the reference with their download
    replaced by synthetic data of the same shape: the estimators, the defaults (linear variogram fitted per problem,
    n_closest_points=10) and the calls of the examples."""
    from sklearn.ensemble import RandomForestClassifier, RandomForestRegressor
    from sklearn.linear_model import LinearRegression, LogisticRegression
    from sklearn.model_selection import train_test_split
    from sklearn.preprocessing import KBinsDiscretizer
    from sklearn.svm import SVC, SVR
    from pykrige_b200.ck import ClassificationKriging
    from pykrige_b200.rk import RegressionKriging
    rng = np.random.default_rng(8)
    n = 5000
    x = np.column_stack([rng.uniform(32.5, 42.0, n), rng.uniform(-124.3, -114.3, n)])      # lat / lon
    p = np.column_stack([rng.lognormal(1.0, 0.5, n), rng.uniform(1, 52, n), rng.lognormal(1.6, 0.3, n),
                         rng.lognormal(0.0, 0.2, n), rng.lognormal(7.0, 0.7, n), rng.lognormal(1.0, 0.3, n)])
    target = 0.4 * p[:, 0] + 0.01 * p[:, 1] + np.sin(x[:, 0]) + np.cos(x[:, 1] / 2.0) + 0.2 * rng.normal(size=n)
    p_train, p_test, x_train, x_test, t_train, t_test = train_test_split(p, x, target, test_size=0.3, random_state=42)
    for m in (SVR(C=0.1, gamma="auto"), RandomForestRegressor(n_estimators=100, random_state=0),
              LinearRegression(copy_X=True, fit_intercept=False)):
        m_rk = RegressionKriging(regression_model=m, n_closest_points=10)
        m_rk.fit(p_train, x_train, t_train)
        assert m_rk.score(p_test, x_test, t_test) > 0.5
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cls = KBinsDiscretizer(encode="ordinal").fit_transform(target.reshape(-1, 1))
    p_train, p_test, x_train, x_test, c_train, c_test = train_test_split(p, x, cls, test_size=0.3, random_state=42)
    for m in (SVC(C=0.1, gamma="auto", probability=True, random_state=0),
              RandomForestClassifier(n_estimators=100, random_state=0), LogisticRegression(max_iter=10000)):
        m_ck = ClassificationKriging(classification_model=m, n_closest_points=10)
        m_ck.fit(p_train, x_train, c_train)
        assert m_ck.score(p_test, x_test, c_test) > 0.25
