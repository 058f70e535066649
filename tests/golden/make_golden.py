"""Generate the committed golden fixtures by running the UNMODIFIED reference (imported from
/root/reference/src — only available in the build container, never on the GPU box).

    python tests/golden/make_golden.py

Writes
  tests/golden/reference_goldens.npz : the reference's own test vectors (tests/test_core.py:28-42,
      490-507, 707-725, 1957-1989): 15 data points, KT3D_H2O OK/UK answers on the 100x100 grid,
      KT3D 3-D data + (z, sigma^2) answers.
  tests/golden/ref_cases.npz : (z, sigmasq) of reference.execute(backend='vectorized'|'loop') for every
      seeded case of tests/cases.py.
  tests/golden/ref_pinv.npz : (z, sigmasq) of the reference with pseudo_inv=True (redundant data points).
  tests/golden/ref_scenarios.npz : fitted parameters, lags, (z, sigmasq) and statistics of the reference for the
      whole-chain scenarios (no variogram parameters given) on the reference's own small fixtures.
  tests/golden/ref_custom.npz : (z, sigmasq) of the reference for variogram_model='custom' callables.
  tests/golden/ref_vgfit.npz : gamma(d) of the six built-in variogram functions on fixed distance vectors (bit patterns)
      and the parameters the reference's constructor fits (variogram_parameters=None) on seeded random scatter.
  tests/golden/ref_api.npz : what the reference's four classes do BEFORE any kriging arithmetic for tests/cases.py
      API_CASES: public attributes, stdout, warnings, exception types and messages of the constructors,
      update_variogram_model and the argument validation of execute().
  tests/golden/ref_fuzz.npz : (z, sigmasq) or the exception type of the reference for the randomised whole-execute()
      configurations of tests/cases.py fuzz_config (backend='vectorized'; 'loop' for the moving window).
  tests/golden/ref_ctor.npz : lags/semivariance of core._initialize_variogram_model and delta/sigma/epsilon
      of core._find_statistics for the constructor-side cases of tests/cases.py.
  tests/golden/ref_twins.npz : (z, sigmasq) of the reference's compiled backend='C' loops (oracle/_ref) on the
      inputs of the twin tests.
The O(N^4) constructor statistics of OK3D/UK/UK3D are patched out (SURVEY F5); nothing else of the
reference is touched.
"""
import os
import sys
import time
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, "/root/reference/src")
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pykrige  # noqa: E402  (the reference)
import pykrige.ok3d, pykrige.uk, pykrige.uk3d  # noqa: E402,E401
import pykrige.kriging_tools as kt  # noqa: E402
import cases  # noqa: E402

assert pykrige.__file__.startswith("/root/reference"), pykrige.__file__


def _no_stats(*a, **k):
    return np.zeros(2), np.ones(2), np.zeros(2)


for mod in (pykrige.ok3d, pykrige.uk, pykrige.uk3d):
    mod._find_statistics = _no_stats


def reference_goldens():
    td = "/root/reference/tests/test_data"
    data = np.genfromtxt(os.path.join(td, "test_data.txt"))
    ok_ans, ok_gx, ok_gy, _, _ = kt.read_asc_grid(os.path.join(td, "test1_answer.asc"), footer=2)
    uk_ans, uk_gx, uk_gy, _, _ = kt.read_asc_grid(os.path.join(td, "test2_answer.asc"), footer=2)
    d3 = np.genfromtxt(os.path.join(td, "test3d_data.txt"), skip_header=1)
    a3 = np.genfromtxt(os.path.join(td, "test3d_answer.txt"))
    ext_ans, ext_gx, ext_gy, _, _ = kt.read_asc_grid(os.path.join(td, "test3_answer.asc"))
    dem, dem_x, dem_y, _, _ = kt.read_asc_grid(os.path.join(td, "test3_dem.asc"))
    np.savez_compressed(
        os.path.join(HERE, "reference_goldens.npz"),
        data=data, ok_answer=np.asarray(ok_ans), ok_gridx=ok_gx, ok_gridy=ok_gy,
        uk_answer=np.asarray(uk_ans), uk_gridx=uk_gx, uk_gridy=uk_gy,
        data3d=d3, answer3d=a3,
        ext_answer=np.asarray(ext_ans), ext_gridx=ext_gx, ext_gridy=ext_gy,
        dem=np.asarray(dem), dem_x=dem_x, dem_y=dem_y,
    )


def ref_cases():
    out = {}
    for case in cases.CASES:
        t0 = time.time()
        inp = cases.build_inputs(case)
        model = cases.make_model(pykrige, case, inp, reference=True)
        z, ss = cases.run_model(model, case, inp, case["ref_backend"])
        out[case["name"] + "/z"] = np.asarray(np.ma.getdata(z), dtype=np.float64)
        out[case["name"] + "/ss"] = np.asarray(np.ma.getdata(ss), dtype=np.float64)
        # a cheap fingerprint of the inputs so a drifting RNG is detected by the tests
        out[case["name"] + "/fp"] = np.array([inp["data"].sum(), inp["values"].sum()])
        print("%-28s %6.2fs  z[%s] mean=%.6f" % (case["name"], time.time() - t0, z.shape, float(np.mean(z))))
    np.savez_compressed(os.path.join(HERE, "ref_cases.npz"), **out)


def ref_pinv():
    """(z, sigmasq) of the reference with pseudo_inv=True for tests/cases.py PINV_CASES -> ref_pinv.npz."""
    out = {}
    for case in cases.PINV_CASES:
        inp = cases.build_inputs(case)
        model = cases.make_model(pykrige, case, inp, reference=True)
        z, ss = cases.run_model(model, case, inp, case["ref_backend"])
        out[case["name"] + "/z"] = np.asarray(np.ma.getdata(z), dtype=np.float64)
        out[case["name"] + "/ss"] = np.asarray(np.ma.getdata(ss), dtype=np.float64)
        out[case["name"] + "/fp"] = np.array([inp["data"].sum(), inp["values"].sum()])
        print("%-30s z[%s] mean=%.6f ss mean=%.6f" % (case["name"], z.shape, float(np.mean(z)), float(np.mean(ss))))
    np.savez_compressed(os.path.join(HERE, "ref_pinv.npz"), **out)


def ref_custom():
    """(z, sigmasq) of the reference for variogram_model='custom' callables (tests/cases.py CUSTOM_CASES)."""
    out = {}
    for case in cases.CUSTOM_CASES:
        inp = cases.build_inputs(case)
        model = cases.make_model(pykrige, case, inp, reference=True)
        z, ss = cases.run_model(model, case, inp, case["ref_backend"])
        out[case["name"] + "/z"] = np.asarray(np.ma.getdata(z), dtype=np.float64)
        out[case["name"] + "/ss"] = np.asarray(np.ma.getdata(ss), dtype=np.float64)
        out[case["name"] + "/fp"] = np.array([inp["data"].sum(), inp["values"].sum()])
        print("%-36s z[%s] mean=%.6f ss mean=%.6f" % (case["name"], z.shape, float(np.mean(z)), float(np.mean(ss))))
    np.savez_compressed(os.path.join(HERE, "ref_custom.npz"), **out)


def ref_scenarios():
    """Whole-chain scenarios (fitted variograms) of tests/cases.py SCENARIOS -> ref_scenarios.npz."""
    gold = np.load(os.path.join(HERE, "reference_goldens.npz"))
    out = {}
    for sc in cases.SCENARIOS:
        data, args, kw = cases.scenario_inputs(sc, gold["data"])
        import importlib
        if sc.get("stats") and sc["cls"] != "OK":           # un-patch the statistics for this scenario
            from pykrige import core as rcore
            for mod in (pykrige.ok3d, pykrige.uk, pykrige.uk3d):
                mod._find_statistics = rcore._find_statistics
        model = cases.scenario_model(pykrige, sc, data)
        z, ss = model.execute(sc["style"], *args, backend="vectorized", **kw)
        out[sc["name"] + "/params"] = np.asarray(model.variogram_model_parameters, dtype=np.float64)
        out[sc["name"] + "/lags"] = np.asarray(model.lags, dtype=np.float64)
        out[sc["name"] + "/semi"] = np.asarray(model.semivariance, dtype=np.float64)
        out[sc["name"] + "/z"] = np.asarray(np.ma.getdata(z), dtype=np.float64)
        out[sc["name"] + "/ss"] = np.asarray(np.ma.getdata(ss), dtype=np.float64)
        if sc.get("stats"):
            out[sc["name"] + "/Q"] = np.array([model.Q1, model.Q2, model.cR], dtype=np.float64)
            out[sc["name"] + "/epsilon"] = np.asarray(model.epsilon, dtype=np.float64)
        print("%-36s params=%s" % (sc["name"], np.array2string(out[sc["name"] + "/params"], precision=5)))
        for mod in (pykrige.ok3d, pykrige.uk, pykrige.uk3d):
            mod._find_statistics = _no_stats
    np.savez_compressed(os.path.join(HERE, "ref_scenarios.npz"), **out)


def ref_ctor():
    """Outputs of the reference's constructor-side routines (core._initialize_variogram_model,
    core._find_statistics) for tests/cases.py VARIOGRAM_CASES / STATS_CASES -> ref_ctor.npz."""
    from pykrige import core as rcore
    from pykrige import variogram_models as rvm
    fn = {"linear": rvm.linear_variogram_model, "power": rvm.power_variogram_model,
          "gaussian": rvm.gaussian_variogram_model, "exponential": rvm.exponential_variogram_model,
          "spherical": rvm.spherical_variogram_model, "hole-effect": rvm.hole_effect_variogram_model}
    out = {}
    for case in cases.VARIOGRAM_CASES:
        X, y = cases.build_ctor_inputs(case)
        lags, semi, _ = rcore._initialize_variogram_model(
            X, y, "linear", [1.0, 0.0], fn["linear"], case["nlags"], False, case["coordinates_type"])
        out[case["name"] + "/lags"] = np.asarray(lags, dtype=np.float64)
        out[case["name"] + "/semi"] = np.asarray(semi, dtype=np.float64)
        out[case["name"] + "/fp"] = np.array([X.sum(), y.sum()])
        print("%-22s lags=%d" % (case["name"], len(lags)))
    for case in cases.STATS_CASES:
        t0 = time.time()
        X, y = cases.build_ctor_inputs(case)
        delta, sigma, epsilon = rcore._find_statistics(
            X, y, fn[case["model"]], case["params"], case["coordinates_type"])
        out[case["name"] + "/delta"] = np.asarray(delta, dtype=np.float64)
        out[case["name"] + "/sigma"] = np.asarray(sigma, dtype=np.float64)
        out[case["name"] + "/epsilon"] = np.asarray(epsilon, dtype=np.float64)
        out[case["name"] + "/fp"] = np.array([X.sum(), y.sum()])
        print("%-22s %5.2fs kept=%d of %d" % (case["name"], time.time() - t0, len(delta), len(y)))
    np.savez_compressed(os.path.join(HERE, "ref_ctor.npz"), **out)


def ref_vgfit():
    """gamma(d) of the reference's six variogram functions (exact bit patterns) and the constructor's automatic fit
    (ok.py:326-346 -> core.py:582-651, soft-L1 TRF) for seeded scatter -> ref_vgfit.npz."""
    from pykrige import variogram_models as rvm
    out = {}
    d = cases.vgfit_distances()
    for m in cases.VGFIT_MODELS:
        f = getattr(rvm, m.replace("-", "_") + "_variogram_model")
        out["gamma/" + m] = np.asarray(f(cases.VGFIT_PARAMS[m], d.copy()), dtype=np.float64)
    for n in (60, 300):
        x, y, z = cases.vgfit_inputs(n)
        for m in cases.VGFIT_MODELS:
            for w in (False, True):
                ok = pykrige.OrdinaryKriging(x, y, z, variogram_model=m, weight=w, nlags=8)
                out["fit/%d/%s/%d" % (n, m, int(w))] = np.asarray(ok.variogram_model_parameters, dtype=np.float64)
                print("fit N=%-4d %-12s weight=%d -> %s" % (n, m, w, out["fit/%d/%s/%d" % (n, m, int(w))]))
    out["cpu_fingerprint"] = np.array(cases.cpu_fingerprint())
    np.savez_compressed(os.path.join(HERE, "ref_vgfit.npz"), **out)


def ref_api():
    """Host-mirror API cases (tests/cases.py API_CASES) through the UNPATCHED reference -> ref_api.npz."""
    import json
    saved = [(mod, mod._find_statistics) for mod in (pykrige.ok3d, pykrige.uk, pykrige.uk3d)]
    from pykrige import core as rcore
    for mod, _ in saved:                       # N = 40: the real cross-validation loop is affordable
        mod._find_statistics = rcore._find_statistics
    named = cases.api_inputs()
    meta, arrays = {}, {}
    try:
        for case in cases.API_CASES:
            rec = cases.api_run(pykrige, case, named, backend="vectorized")
            attrs = {}
            for k, v in rec["attrs"].items():
                if isinstance(v, np.ndarray):
                    arrays[case["name"] + "/" + k] = v
                    attrs[k] = "@array"
                else:
                    attrs[k] = v
            if rec["ret"] is not None:
                arrays[case["name"] + "/@ret"] = rec["ret"]
            meta[case["name"]] = dict(kind=rec["kind"], exc=rec["exc"], msg=rec["msg"], stdout=rec["stdout"],
                                      warnings=rec["warnings"], attrs=attrs)
            print("%-40s %s %s" % (case["name"], rec["kind"], rec["exc"]))
    finally:
        for mod, f in saved:
            mod._find_statistics = f
    arrays["@meta"] = np.array(json.dumps(meta, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, "ref_api.npz"), **arrays)


def ref_fuzz():
    import warnings
    out = {}
    n_ok = n_exc = 0
    for t in range(cases.N_FUZZ):
        c = cases.fuzz_config(t)
        if c is None:
            continue
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                model = getattr(pykrige, c["cls"])(*c["data"], **c["kw"])
                z, ss = model.execute(c["style"], *c["pts"], backend="loop" if c["knn"] else "vectorized", **c["ekw"])
            out["%d/z" % t] = np.ma.getdata(z)
            out["%d/ss" % t] = np.ma.getdata(ss)
            out["%d/mask" % t] = np.ma.getmaskarray(z) if np.ma.isMaskedArray(z) else np.zeros(0, bool)
            # 2-norm condition number of the reference's own kriging matrix (ok.py:626-648 / uk.py:861-920): how many
            # digits the reference's scipy.linalg.inv itself can be trusted to
            try:
                a = model._get_kriging_matrix(len(c["data"][0]))
            except TypeError:                      # uk.py / uk3d.py: _get_kriging_matrix(n, n_withdrifts)
                n_rows = len(c["data"][0])
                drift = c["kw"].get("drift_terms", [])
                nd = ((2 if c["cls"].endswith("Kriging") else 3) * ("regional_linear" in drift) + 2 * ("point_log" in drift)
                      + sum(q in drift for q in ("external_Z", "specified", "functional")))
                a = model._get_kriging_matrix(n_rows, n_rows + nd)
            out["%d/cond" % t] = np.array(np.linalg.cond(a))
            n_ok += 1
        except Exception as e:  # noqa: BLE001
            out["%d/exc" % t] = np.array(type(e).__name__)
            n_exc += 1
    print("fuzz: %d results, %d exceptions" % (n_ok, n_exc))
    n_ok = n_exc = 0
    for t in range(cases.N_KIND):                   # geographic / pseudo_inv / duplicates / custom callables
        c = cases.kind_config(t)
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                model = getattr(pykrige, c["cls"])(*c["data"], **c["kw"])
                z, ss = model.execute(c["style"], *c["pts"], backend="loop" if c["knn"] else "vectorized", **c["ekw"])
            out["kind%d/z" % t] = np.ma.getdata(z)
            out["kind%d/ss" % t] = np.ma.getdata(ss)
            n_ok += 1
        except Exception as e:  # noqa: BLE001
            out["kind%d/exc" % t] = np.array(type(e).__name__)
            n_exc += 1
    print("kinds: %d results, %d exceptions" % (n_ok, n_exc))
    for t in range(cases.N_SEQ):                    # stateful sequences on one object
        c = cases.seq_config(t)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for k, (z, ss) in enumerate(cases.seq_run(pykrige, c, "vectorized")):
                out["seq%d/%d/z" % (t, k)] = z
                out["seq%d/%d/ss" % (t, k)] = ss
    np.savez_compressed(os.path.join(HERE, "ref_fuzz.npz"), **out)


def ref_twins():
    """(z, sigmasq) of the reference's compiled `_c_exec_loop` / `_c_exec_loop_moving_window` (lib/cok.pyx, built into
    oracle/_ref by oracle/build_ref.py) on the seeded inputs of the twin tests in tests/test_oracle.py and
    tests/test_parity_gpu.py, so that those tests compare with the reference without needing it."""
    sys.path.insert(0, ROOT)
    from oracle import krige_oracle as ko, ref_native as rn
    # the twins live in a package also named `pykrige`: set the imported reference aside while they load
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "pykrige" or k.startswith("pykrige.")}
    try:
        out = _twin_outputs(ko, rn)
    finally:
        for k in [k for k in sys.modules if k == "pykrige" or k.startswith("pykrige.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    np.savez_compressed(os.path.join(HERE, "ref_twins.npz"), **out)


def _twin_outputs(ko, rn):
    assert rn.available(), "oracle/_ref is not built"
    out = {}
    xyz, val = cases.synth_data(11, 300, 2)
    pts = cases.synth_points(11, 200, 2, xyz)
    out["oracle/fp"] = np.array([xyz.sum(), val.sum(), pts.sum()])
    for model in ("linear", "power", "gaussian", "exponential", "spherical"):
        stored = ko.stored_parameters(model, cases.MODELS[model])
        for exact in (True, False):
            z, ss = rn.exec_loop(xyz, pts, val, model, stored, exact_values=exact)
            out["oracle/%s/%d/z" % (model, exact)], out["oracle/%s/%d/ss" % (model, exact)] = z, ss
    for dim, k in ((2, 8), (3, 12)):
        xyz, val = cases.synth_data(12 + dim, 400, dim)
        pts = cases.synth_points(12 + dim, 150, dim, xyz)
        out["oracle_mw/%d/fp" % dim] = np.array([xyz.sum(), val.sum(), pts.sum()])
        z, ss = rn.exec_loop_moving_window(xyz, pts, val, "exponential", ko.stored_parameters("exponential", [1.0, 150.0, 0.05]), k)
        out["oracle_mw/%d/z" % dim], out["oracle_mw/%d/ss" % dim] = z, ss
    xyz, val = cases.synth_data(2024, 1500, 2)
    pts = cases.synth_points(2024, 2000, 2, xyz)
    out["cuda/fp"] = np.array([xyz.sum(), val.sum(), pts.sum()])
    for model in ("exponential", "spherical", "linear"):
        z, ss = rn.exec_loop(xyz, pts, val, model, ko.stored_parameters(model, cases.MODELS[model]))
        out["cuda/%s/z" % model], out["cuda/%s/ss" % model] = z, ss
    z, ss = rn.exec_loop_moving_window(xyz, pts, val, "exponential", ko.stored_parameters("exponential", [1.0, 150.0, 0.05]), 16)
    out["cuda/knn/z"], out["cuda/knn/ss"] = z, ss
    return out


if __name__ == "__main__":
    which = sys.argv[1:] or ["goldens", "cases", "ctor", "pinv", "scenarios", "custom", "vgfit", "api", "fuzz", "twins"]
    if "twins" in which:
        ref_twins()
    if "fuzz" in which:
        ref_fuzz()
    if "api" in which:
        ref_api()
    if "vgfit" in which:
        ref_vgfit()
    if "goldens" in which:
        reference_goldens()
    if "cases" in which:
        ref_cases()
    if "ctor" in which:
        ref_ctor()
    if "pinv" in which:
        ref_pinv()
    if "scenarios" in which:
        ref_scenarios()
    if "custom" in which:
        ref_custom()
