"""Cases of RegressionKriging / ClassificationKriging shared by tests/golden/make_golden_rkck.py (ref_rkck.npz, written
by the imported reference), tests/test_rkck_host.py and tests/test_rkck_gpu.py.

The data are the synthetic set-up of the reference's tests/test_regression_krige.py and test_classification_krige.py:
100 samples with five collinear covariates, a linear target with uniform noise, stations on a 10 x 10 lon/lat lattice,
a 70/30 split. The lattice has exact distance ties, which the moving window with n_closest_points=2 breaks by station
index here and by cKDTree's own order in the reference, so the fixture cases move every station by a seeded jitter of
up to 2 degrees. The 3-D methods add a seeded depth coordinate. Classes are quantile bins of the target."""
from itertools import product

import numpy as np

EXP = [1.0, 120.0, 0.1]                  # fixed variogram of the 'fixed' cases: exponential [sill, range, nugget]


def custom_variogram(m, d):
    """A 'custom' callable (an exponential variogram with a linear tail) for the fixed-parameter custom case."""
    return m[0] * (1.0 - np.exp(-d / m[1])) + m[2] * d


def reference_data(dim=2, n_classes=None, jitter=False):
    """(p, x, y) before the split: covariates (100, 5), station coordinates (100, dim), targets (100,) or, with
    n_classes, class labels (100, 1) as the reference's KBinsDiscretizer(encode='ordinal') gives them."""
    rs = np.random.RandomState(1)
    t = np.linspace(-1.0, 1.0, 100)
    p = np.tile(t, reps=(5, 1)).T
    y = 1 + 5 * p[:, 0] - 2 * p[:, 1] - 2 * p[:, 2] + 3 * p[:, 3] + 4 * p[:, 4] + 2 * (rs.rand(100) - 0.5)
    x = np.array(list(product(np.linspace(-180.0, 180.0, 10), np.linspace(-90.0, 90.0, 10))))
    aux = np.random.RandomState(7)
    if jitter:
        x = x + aux.uniform(-2.0, 2.0, size=x.shape)
    if dim == 3:
        x = np.column_stack([x, aux.uniform(0.0, 100.0, size=100)])
    if n_classes is not None:
        edges = np.quantile(y, np.linspace(0.0, 1.0, n_classes + 1)[1:-1])
        y = np.digitize(y, edges).astype(np.float64).reshape(-1, 1)
    return p, x, y


def split(p, x, y):
    """The reference tests' split: train_test_split(..., train_size=0.7, random_state=10)."""
    from sklearn.model_selection import train_test_split
    p_tr, p_te, y_tr, y_te, x_tr, x_te = train_test_split(p, y, x, train_size=0.7, random_state=10)
    return dict(p_train=p_tr, x_train=x_tr, y_train=y_tr, p_test=p_te, x_test=x_te, y_test=y_te)


def estimator(name):
    """A fresh, deterministic scikit-learn estimator."""
    from sklearn.ensemble import RandomForestClassifier, RandomForestRegressor
    from sklearn.linear_model import LinearRegression
    from sklearn.svm import SVC, SVR
    return {
        "linear": lambda: LinearRegression(),
        "svr": lambda: SVR(C=0.01, gamma="auto"),
        "rf_reg": lambda: RandomForestRegressor(min_samples_split=5, n_estimators=50, random_state=0),
        "svc": lambda: SVC(C=0.01, gamma="auto", probability=True, random_state=0),
        "rf_cls": lambda: RandomForestClassifier(n_estimators=50, random_state=0),
    }[name]()


def _cases():
    out = []
    rk_est = ["linear", "svr", "rf_reg"]
    ck_est = ["svc", "rf_cls"]
    i = 0
    for kind in ("rk", "ck"):
        for method in ("ordinary", "universal", "ordinary3d", "universal3d"):
            for fixed in (False, True):
                for k in ((2, 10) if method.startswith("ordinary") else (10,)):
                    est = (rk_est if kind == "rk" else ck_est)[i % (3 if kind == "rk" else 2)]
                    c = dict(kind=kind, method=method, k=k, fixed=fixed, est=est, n_classes=None, pseudo_inv=False,
                             custom=False, verbose=False)
                    if kind == "ck":
                        c["n_classes"] = 3 if i % 2 else 5
                    out.append(c)
                    i += 1
    out.append(dict(kind="ck", method="universal", k=10, fixed=True, est="svc", n_classes=3, pseudo_inv=True,
                    custom=False, verbose=False))
    out.append(dict(kind="ck", method="ordinary", k=10, fixed=True, est="rf_cls", n_classes=5, pseudo_inv=False,
                    custom=True, verbose=False))
    out.append(dict(kind="rk", method="ordinary", k=10, fixed=True, est="linear", n_classes=None, pseudo_inv=False,
                    custom=False, verbose=True))
    for c in out:
        c["dim"] = 3 if c["method"].endswith("3d") else 2
        c["name"] = "%s_%s_k%d_%s_%s%s%s%s%s" % (
            c["kind"], c["method"], c["k"], "fixed" if c["fixed"] else "auto", c["est"],
            "_c%d" % c["n_classes"] if c["n_classes"] else "", "_pinv" if c["pseudo_inv"] else "",
            "_custom" if c["custom"] else "", "_verbose" if c["verbose"] else "")
    return out


CASES = _cases()


def data_key(case):
    return "%dd_c%d" % (case["dim"], case["n_classes"] or 0)


def fixture_data(case):
    """The jittered, split data of a fixture case."""
    return split(*reference_data(case["dim"], case["n_classes"], jitter=True))


def make(module, case, estimator_name=None):
    """The case's RegressionKriging / ClassificationKriging from `module` (the reference's pykrige or pykrige_b200)."""
    import importlib
    kw = dict(method=case["method"], n_closest_points=case["k"], pseudo_inv=case["pseudo_inv"],
              verbose=case["verbose"])
    if case["custom"]:
        kw.update(variogram_model="custom", variogram_function=custom_variogram, variogram_parameters=[1.0, 120.0, 1e-3])
    elif case["fixed"]:
        kw.update(variogram_model="exponential", variogram_parameters=list(EXP))
    est = estimator(estimator_name or case["est"])
    if case["kind"] == "rk":
        return importlib.import_module(module + ".rk").RegressionKriging(regression_model=est, **kw)
    return importlib.import_module(module + ".ck").ClassificationKriging(classification_model=est, **kw)


def fitted_parameters(model):
    """Per-class fitted variogram parameters, (C - 1, n_params); RegressionKriging: (1, n_params)."""
    kr = model.krige if isinstance(model.krige, list) else [model.krige]
    return np.array([np.asarray(k.model.variogram_model_parameters, dtype=np.float64) for k in kr])
