"""Generate tests/golden/ref_rkck.npz by running the UNMODIFIED reference's RegressionKriging / ClassificationKriging
(rk.py, ck.py), imported the way make_golden.py imports it (only available in the build container, never on the GPU box).

    python tests/golden/make_golden_rkck.py

For every case of tests/rkck_cases.py: the split data, predict() and krige_residual() at the test stations, the
per-class fitted variogram parameters, score() and the stdout of fit(); ClassificationKriging also the class
probabilities. Then the reference's ilr / inverse ilr / closure on fixed compositions, including zero parts and rows
that sum to zero. Used by tests/test_rkck_host.py and tests/test_rkck_gpu.py.
"""
import contextlib
import io
import os
import warnings

import numpy as np

import make_golden  # noqa: F401  (puts the reference and tests/ on sys.path, patches out the O(N^4) statistics)
import cases
import rkck_cases as rc

HERE = os.path.dirname(os.path.abspath(__file__))


def ref_rkck():
    import sklearn
    from pykrige import ck as rck
    out = {"cpu_fingerprint": np.array(cases.cpu_fingerprint()), "sklearn_version": np.array(sklearn.__version__)}
    for case in rc.CASES:
        d = rc.fixture_data(case)
        for f, a in d.items():
            out["data/%s/%s" % (rc.data_key(case), f)] = a
        model = rc.make("pykrige", case)
        buf = io.StringIO()
        with warnings.catch_warnings(), contextlib.redirect_stdout(buf):
            warnings.simplefilter("ignore")
            model.fit(d["p_train"], d["x_train"], d["y_train"])
        with warnings.catch_warnings(), contextlib.redirect_stdout(io.StringIO()):
            warnings.simplefilter("ignore")
            resid = model.krige_residual(d["x_test"])
            pred = model.predict(d["p_test"], d["x_test"])
            score = model.score(d["p_test"], d["x_test"], d["y_test"])
        n = case["name"]
        out[n + "/stdout"] = np.array(buf.getvalue())
        out[n + "/resid"] = np.asarray(resid, dtype=np.float64)
        out[n + "/pred"] = np.asarray(pred)
        out[n + "/score"] = np.array(score)
        out[n + "/params"] = rc.fitted_parameters(model)
        if case["kind"] == "ck":
            ilr = resid + rck.ilr_transformation(model.classification_model.predict_proba(d["p_test"]))
            out[n + "/proba"] = rck.inverse_ilr_transformation(ilr)
        print("%-48s score=%.4f params[0]=%s" % (n, score, out[n + "/params"][0]))
    rng = np.random.default_rng(5)
    comp = rng.dirichlet(np.ones(4), size=12)
    comp[0, 1] = comp[1, :3] = comp[2, 0] = 0.0                # zero probabilities, clipped at eps
    comp[3] = [1.0, 0.0, 0.0, 0.0]                             # a one-hot row
    comp[4] = [1e-20, 1e-17, 0.5, 0.5]                         # parts below eps
    out["ilr/in"] = comp
    out["ilr/out"] = rck.ilr_transformation(comp)
    coords = np.vstack([rng.normal(scale=3.0, size=(10, 3)), out["ilr/out"][:2], [[-40.0, 30.0, 20.0]]])
    out["inv/in"] = coords
    out["inv/out"] = rck.inverse_ilr_transformation(coords)
    parts = np.vstack([rng.uniform(0.0, 2.0, size=(6, 5)), np.zeros((1, 5)), [[1.0, -1.0, 0.0, 0.0, 0.0]]])
    out["closure/in"] = parts                                  # the last two rows sum to zero: nan / inf
    with np.errstate(all="ignore"):
        out["closure/out"] = rck.closure(parts)
        out["closure/out_k"] = rck.closure(parts, k=100.0)
    np.savez_compressed(os.path.join(HERE, "ref_rkck.npz"), **out)


if __name__ == "__main__":
    ref_rkck()
