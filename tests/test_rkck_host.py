"""CPU tests of RegressionKriging (pykrige_b200/rk.py) and ClassificationKriging (pykrige_b200/ck.py).

`_cabi.Handle` is replaced by tests/fields_emulator.py (tests/abi_emulator.py plus kb200_set_values), so whole fit /
predict / score calls run through the product code above the C ABI and are compared with the imported reference's
outputs (tests/golden/ref_rkck.npz, written by tests/golden/make_golden_rkck.py). The device itself is tests/test_rkck_gpu.py."""
import os

import numpy as np
import pytest
from numpy.testing import assert_array_equal

import cases
import rkck_cases as rc
from conftest import GOLDEN, assert_parity
from fields_emulator import FieldsEmulatedHandle

pytest.importorskip("sklearn")

R64 = 1e-5          # the tolerance of the other emulated host tests and of the GPU parity tests


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "ref_rkck.npz"))


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", FieldsEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    return pykrige_b200


def same_platform(ref):
    """Bit-for-bit comparisons of fitted parameters need the generator's numpy SIMD dispatch and scikit-learn."""
    import sklearn
    return str(ref["cpu_fingerprint"]) == cases.cpu_fingerprint() and str(ref["sklearn_version"]) == sklearn.__version__


def fixture_data(ref, case):
    return {f: ref["data/%s/%s" % (rc.data_key(case), f)] for f in
            ("p_train", "x_train", "y_train", "p_test", "x_test", "y_test")}


def check_against_fixture(model, case, ref, d, R, stdout=None, exact=True):
    """predict / krige_residual / score / fitted parameters / fit's stdout of a fitted model against the fixture."""
    n = case["name"]
    if stdout is not None:
        want = str(ref[n + "/stdout"])
        if exact:
            assert stdout == want
        else:                                   # the verbose lines carry the fitted numbers
            strip = [ln for ln in want.split("\n") if not any(ch.isdigit() for ch in ln)]
            assert [ln for ln in stdout.split("\n") if not any(ch.isdigit() for ch in ln)] == strip
    params = rc.fitted_parameters(model)
    if exact:
        assert_array_equal(params, ref[n + "/params"])
    else:
        np.testing.assert_allclose(params, ref[n + "/params"], rtol=1e-6, atol=1e-12)
    resid = model.krige_residual(d["x_test"])
    assert_parity(resid, ref[n + "/resid"], R, n + " krige_residual")
    pred = model.predict(d["p_test"], d["x_test"])
    score = model.score(d["p_test"], d["x_test"], d["y_test"])
    if case["kind"] == "rk":
        assert_parity(pred, ref[n + "/pred"], R, n + " predict")
        np.testing.assert_allclose(score, float(ref[n + "/score"]), rtol=10 * R)
        return
    proba = np.sort(ref[n + "/proba"], axis=1)
    clear = proba[:, -1] - proba[:, -2] > 1e-4 * proba[:, -1]       # no near-tie between the two most probable classes
    assert clear.sum() >= 0.9 * clear.size, n
    assert_array_equal(pred[clear], ref[n + "/pred"][clear])
    if clear.all():
        assert score == float(ref[n + "/score"])


@pytest.mark.parametrize("case", rc.CASES, ids=[c["name"] for c in rc.CASES])
def test_fit_predict_score_against_the_reference(pk, case, ref, capsys):
    """Every fixture case: fitted variogram parameters and stdout bit for bit, predictions and kriged residuals at the
    emulator tolerance, the route the residuals took."""
    import warnings
    d = fixture_data(ref, case)
    model = rc.make("pykrige_b200", case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model.fit(d["p_train"], d["x_train"], d["y_train"])
        out = capsys.readouterr().out
        check_against_fixture(model, case, ref, d, R64, stdout=out, exact=same_platform(ref))
    if case["kind"] == "ck":
        shared = case["fixed"] and not case["pseudo_inv"]
        assert model._shares_one_problem({}) == shared
        h0 = model.krige[0].model._kb_handle
        assert h0.n_fields == (len(model.classes_) - 1 if shared else 0)
        if shared:                              # one problem: the other Krige objects never reached the device
            assert all(getattr(k.model, "_kb_handle", None) is None for k in model.krige[1:])


def test_ilr_pair_and_closure_against_the_reference(ref):
    from pykrige_b200.ck import closure, ilr_transformation, inverse_ilr_transformation
    if same_platform(ref):      # the bits the automatic variogram fit of the residuals needs
        assert_array_equal(ilr_transformation(ref["ilr/in"]), ref["ilr/out"])
        assert_array_equal(inverse_ilr_transformation(ref["inv/in"]), ref["inv/out"])
    np.testing.assert_allclose(ilr_transformation(ref["ilr/in"]), ref["ilr/out"], rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(inverse_ilr_transformation(ref["inv/in"]), ref["inv/out"], rtol=1e-13, atol=1e-300)
    with np.errstate(all="ignore"):
        c, ck = closure(ref["closure/in"]), closure(ref["closure/in"], k=100.0)
    assert not np.isfinite(ref["closure/out"][-2:]).any()
    assert_array_equal(c, ref["closure/out"])           # nan and inf where the reference has them
    assert_array_equal(ck, ref["closure/out_k"])
    comp = ref["ilr/in"][5:]                              # no part below machine epsilon: the pair round-trips
    np.testing.assert_allclose(inverse_ilr_transformation(ilr_transformation(comp)), closure(comp), rtol=1e-12)
    assert ilr_transformation(comp).shape == (comp.shape[0], comp.shape[1] - 1)


def test_models_of_the_wrong_kind_are_refused(pk):
    from sklearn.svm import SVC, SVR
    from pykrige_b200.ck import ClassificationKriging
    from pykrige_b200.rk import RegressionKriging
    for bad in (SVC(), object(), "svr"):
        with pytest.raises(RuntimeError, match="^Needs to supply an instance of a scikit-learn regression class.$"):
            RegressionKriging(regression_model=bad)
    for bad in (SVR(), object()):
        with pytest.raises(RuntimeError, match="^Needs to supply an instance of a scikit-learn classification class.$"):
            ClassificationKriging(classification_model=bad)
    with pytest.raises(ValueError, match="Kriging method must be one of"):
        RegressionKriging(method="simple")


def test_missing_sklearn_is_reported(monkeypatch):
    from pykrige_b200 import compat
    monkeypatch.setattr(compat, "SKLEARN_INSTALLED", False)
    with pytest.raises(compat.SklearnException, match="sklearn needs to be installed"):
        compat.validate_sklearn()


def test_public_names(pk):
    from pykrige_b200.ck import ClassificationKriging
    from pykrige_b200.rk import RegressionKriging
    assert pk.RegressionKriging is RegressionKriging and pk.ClassificationKriging is ClassificationKriging
    with pytest.raises(AttributeError):
        pk.KrigingTools


def _routes(pk, monkeypatch, method, k, n_classes, **kw):
    """krige_residual of one fitted ClassificationKriging through both routes, and the model."""
    from pykrige_b200.ck import ClassificationKriging
    p, x, y = rc.reference_data(3 if method.endswith("3d") else 2, n_classes, jitter=True)
    model = ClassificationKriging(classification_model=rc.estimator("rf_cls"), method=method, n_closest_points=k,
                                  variogram_model="exponential", variogram_parameters=list(rc.EXP), **kw)
    model.fit(p, x, y)
    q = x[::3] + 7.0
    shared = model.krige_residual(q)
    with monkeypatch.context() as m:
        m.setattr(ClassificationKriging, "_shares_one_problem", lambda self, kwargs: False)
        per_class = model.krige_residual(q)
    return model, shared, per_class


@pytest.mark.parametrize("method,k", [("ordinary", 10), ("ordinary", None), ("universal", 10), ("ordinary3d", 5),
                                      ("universal3d", 10)])
def test_shared_route_equals_the_per_class_route(pk, monkeypatch, capsys, method, k):
    """Under the emulator the two routes of krige_residual agree bit for bit (the emulator kriges each field as its own
    problem, so this checks the host plumbing: column order, transposition, the Krige object's own arguments)."""
    model, shared, per_class = _routes(pk, monkeypatch, method, k, 5)
    assert shared.shape == per_class.shape == (34, 4)
    assert_array_equal(shared, per_class)
    assert model.krige[0].model._kb_handle.n_fields == 0          # the per-class call re-described krige[0] alone


def test_shared_route_chunks_above_the_field_limit(pk, monkeypatch, capsys):
    from pykrige_b200 import _cabi
    monkeypatch.setattr(_cabi, "MAX_FIELDS", 3)
    model, shared, per_class = _routes(pk, monkeypatch, "ordinary", 10, 5)
    assert model.krige[0].model._kb_handle.calls.count("set_problem_knn") >= 2
    assert_array_equal(shared, per_class)


def test_refused_value_fields_take_the_per_class_route(pk, monkeypatch, capsys):
    """pseudo_inv on the global path, a dtype other than float64 and n_gpus > 1 are refused by execute(values=...):
    those calls krige class by class, as the reference does."""
    from pykrige_b200.ck import ClassificationKriging
    model, _, _ = _routes(pk, monkeypatch, "universal", 10, 3, pseudo_inv=True)
    assert not model._shares_one_problem({})
    z = model.krige_residual(rc.reference_data(2, 3, jitter=True)[1][:5])
    assert z.shape == (5, 2) and all(k.model._kb_handle.n_fields == 0 for k in model.krige)
    mw = ClassificationKriging(classification_model=rc.estimator("rf_cls"), variogram_model="exponential",
                               variogram_parameters=list(rc.EXP), pseudo_inv=True)   # the moving window ignores it
    assert mw._shares_one_problem({})
    assert not mw._shares_one_problem({"dtype": "float32"})
    assert not mw._shares_one_problem({"n_gpus": 2})
    auto = ClassificationKriging(classification_model=rc.estimator("rf_cls"))
    assert not auto._shares_one_problem({})
