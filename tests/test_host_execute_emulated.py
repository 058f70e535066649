"""CPU tests of the HOST side of execute(..., backend='cuda'), end to end, on a box without a GPU.

`_cabi.Handle` is replaced by tests/abi_emulator.py (the documented semantics of include/krige_b200.h on top of the CPU
oracle); everything above the C ABI is the product code: point planning, mask compaction and scatter, the order and
frame of the drift columns, device-drift configuration, the custom-variogram table, output shaping. Whole execute()
calls are compared with the SAME fixtures the GPU tests use (tests/golden/*.npz: outputs of the unmodified imported
reference and the reference's own KT3D / MEUK answers). A host regression therefore shows up here, in the CPU suite,
and not only on the GPU box. The CUDA path itself is NOT exercised by this file — that is tests/test_parity_gpu.py."""
import numpy as np
import pytest
from numpy.testing import assert_allclose

import cases
from abi_emulator import EmulatedHandle
from conftest import assert_parity

R64 = 1e-5          # the same tolerance as the GPU tests (SURVEY.md §8d); the emulator itself agrees to ~1e-9


@pytest.fixture()
def pk(monkeypatch):
    import pykrige_b200
    from pykrige_b200 import _cabi

    def no_device():
        raise _cabi.KrigeB200Error("emulated box: no CUDA device for the constructor-side helpers")

    monkeypatch.setattr(_cabi, "Handle", EmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)     # experimental variogram / statistics take the host route
    return pykrige_b200


def _run(pk, case):
    inp = cases.build_inputs(case)
    model = cases.make_model(pk, case, inp)
    z, ss = cases.run_model(model, case, inp, "cuda")
    return inp, model, z, ss


def _compare(case, inp, z, ss, zr, sr, R=R64):
    assert z.shape == zr.shape and ss.shape == sr.shape
    if case["style"] == "masked":
        assert np.ma.is_masked(z) and np.ma.is_masked(ss)
        assert np.array_equal(np.ma.getmaskarray(z), inp["mask"])
        keep = ~inp["mask"]
        z, ss, zr, sr = np.ma.getdata(z)[keep], np.ma.getdata(ss)[keep], zr[keep], sr[keep]
    assert_parity(np.ravel(z), np.ravel(zr), R, case["name"] + " z")
    assert_parity(np.ravel(ss), np.ravel(sr), R, case["name"] + " ss")


ALL_CASES = [c for c in cases.CASES if c["name"] != "ok2d_hole_effect_small"]


@pytest.mark.parametrize("case", ALL_CASES, ids=[c["name"] for c in ALL_CASES])
def test_seeded_cases_through_the_host_wrappers(pk, case, ref_cases):
    """Every seeded case of tests/cases.py (OK / UK / 3-D, all drift kinds, anisotropy, grid / masked / points,
    non-exact, geographic, moving window) — the cases of test_parity_gpu.py::test_global_cases_match_reference and
    ::test_moving_window_cases_match_reference."""
    inp, model, z, ss = _run(pk, case)
    _compare(case, inp, z, ss, ref_cases[case["name"] + "/z"], ref_cases[case["name"] + "/ss"])
    h = model._kb_handle
    assert ("set_problem_knn" if case["k"] is not None else "set_problem") in h.calls


@pytest.mark.parametrize("case", cases.PINV_CASES, ids=[c["name"] for c in cases.PINV_CASES])
def test_pseudo_inverse_cases_through_the_host_wrappers(pk, case, ref_pinv):
    inp, model, z, ss = _run(pk, case)
    _compare(case, inp, z, ss, ref_pinv[case["name"] + "/z"], ref_pinv[case["name"] + "/ss"])
    assert model._kb_handle.problem["pinv"]


@pytest.mark.parametrize("case", cases.CUSTOM_CASES, ids=[c["name"] for c in cases.CUSTOM_CASES])
def test_custom_variogram_cases_through_the_host_wrappers(pk, case, ref_custom):
    """variogram_model='custom': the host tabulates the callable over [0, dmax] (kb200_set_variogram_table); the
    emulator refuses any distance beyond the tabulated range, so _table_dmax is checked as well."""
    inp, model, z, ss = _run(pk, case)
    _compare(case, inp, z, ss, ref_custom[case["name"] + "/z"], ref_custom[case["name"] + "/ss"])
    assert model._kb_handle.table is not None


@pytest.mark.parametrize("sc", cases.SCENARIOS, ids=[s["name"] for s in cases.SCENARIOS])
def test_whole_chain_scenarios_through_the_host_wrappers(pk, sc, ref_scenarios, ref_goldens):
    """Constructor with a fitted variogram -> execute -> statistics on the reference's own small data sets."""
    data, args, kw = cases.scenario_inputs(sc, ref_goldens["data"])
    m = cases.scenario_model(pk, sc, data)
    z, ss = m.execute(sc["style"], *args, backend="cuda", **kw)
    zr, sr = ref_scenarios[sc["name"] + "/z"], ref_scenarios[sc["name"] + "/ss"]
    assert z.shape == zr.shape and ss.shape == sr.shape
    if sc["style"] == "masked":
        assert np.ma.is_masked(z)
        keep = ~np.ma.getmaskarray(z)
        z, ss, zr, sr = np.ma.getdata(z)[keep], np.ma.getdata(ss)[keep], zr[keep], sr[keep]
    if sc.get("three_drifts"):      # exactly determined by its drift terms (rcond 2e-33 in the reference): shape only
        assert np.all(np.isfinite(z)) and np.all(np.isfinite(ss))
        return
    assert_parity(np.ravel(z), np.ravel(zr), R64, sc["name"] + " z")
    assert_parity(np.ravel(ss), np.ravel(sr), R64, sc["name"] + " ss")
    if sc.get("stats"):
        assert_allclose([m.Q1, m.Q2, m.cR], ref_scenarios[sc["name"] + "/Q"], rtol=1e-9)
        assert_allclose(m.epsilon, ref_scenarios[sc["name"] + "/epsilon"], rtol=1e-9, atol=1e-12)


def test_reference_golden_grids_through_the_host_wrappers(pk, ref_goldens):
    """The reference's own answers (tests/test_core.py:490-507, 707-725, 1479-1507, 1957-1989): KT3D_H2O ordinary and
    universal kriging, the MEUK external-drift grid, the KT3D 3-D answers."""
    g = ref_goldens
    d = g["data"]
    ok = pk.OrdinaryKriging(d[:, 0], d[:, 1], d[:, 2], variogram_model="exponential", variogram_parameters=[500.0, 3000.0, 0.0])
    z, ss = ok.execute("grid", g["ok_gridx"], g["ok_gridy"], backend="cuda")
    assert_allclose(z, g["ok_answer"], rtol=1e-6)
    uk = pk.UniversalKriging(d[:, 0], d[:, 1], d[:, 2], variogram_model="exponential", variogram_parameters=[500.0, 3000.0, 0.0],
                             drift_terms=["regional_linear"])
    z, ss = uk.execute("grid", g["uk_gridx"], g["uk_gridy"], backend="cuda")
    assert_allclose(z, g["uk_answer"], rtol=1e-6)
    ext = pk.UniversalKriging(d[:, 0], d[:, 1], d[:, 2], variogram_model="spherical", variogram_parameters=[500.0, 3000.0, 0.0],
                              drift_terms=["external_Z"], external_drift=g["dem"], external_drift_x=g["dem_x"],
                              external_drift_y=g["dem_y"])
    z, ss = ext.execute("grid", g["ext_gridx"], g["ext_gridy"], backend="cuda")
    assert_allclose(z, g["ext_answer"], rtol=1e-5, atol=1e-8)
    with pytest.raises(ValueError):
        ext.execute("grid", g["ext_gridx"] + 1.0e6, g["ext_gridy"], backend="cuda")
    d3 = g["data3d"]
    ax = np.arange(10.0)
    k3 = pk.OrdinaryKriging3D(d3[:, 0], d3[:, 1], d3[:, 2], d3[:, 3], variogram_model="linear", variogram_parameters=[1.0, 0.1])
    k, ss = k3.execute("grid", ax, ax, ax, backend="cuda")
    assert_allclose(k, g["answer3d"][:, 0].reshape(10, 10, 10), rtol=1e-3, atol=1e-8)
    assert_allclose(ss, g["answer3d"][:, 1].reshape(10, 10, 10), rtol=1e-3, atol=1e-8)


def test_problem_cache_follows_the_data(pk):
    """execute() twice: the second call reuses the described problem; editing the data in place, changing the
    variogram or switching the moving window on describes it again (_problem_signature / _content_digest)."""
    xyz, val = cases.synth_data(321, 80, 2)
    m = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
    gx = gy = np.linspace(0.0, 1000.0, 9)
    z0, _ = m.execute("grid", gx, gy, backend="cuda")
    h = m._kb_handle
    assert h.calls.count("set_problem") == 1
    z1, _ = m.execute("grid", gx, gy, backend="cuda")
    assert h.calls.count("set_problem") == 1 and np.array_equal(z0, z1)
    m.Z[3] += 5.0                                            # in-place edit of the values
    z2, _ = m.execute("grid", gx, gy, backend="cuda")
    assert h.calls.count("set_problem") == 2 and not np.array_equal(z0, z2)
    m.update_variogram_model("spherical", [1.0, 400.0, 0.05])
    m.execute("grid", gx, gy, backend="cuda")
    assert h.calls.count("set_problem") == 3
    m.execute("grid", gx, gy, backend="cuda", n_closest_points=6)
    assert h.calls.count("set_problem_knn") == 1
    m.execute("grid", gx, gy, backend="cuda")              # back to the global path: described again
    assert h.calls.count("set_problem") == 4


def test_sklearn_wrapper_through_the_host_wrappers(pk):
    """compat.Krige.fit / predict (compat.py:181-291) route to execute(style='points', backend='cuda')."""
    from pykrige_b200.compat import Krige
    from oracle import krige_oracle as ko
    xyz, val = cases.synth_data(11, 90, 2)
    pts = cases.synth_points(11, 40, 2, xyz)
    est = Krige(method="ordinary", variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05], n_closest_points=7)
    est.fit(xyz, val)
    zo, _ = ko.krige(xyz, val, "exponential", ko.stored_parameters("exponential", [1.0, 300.0, 0.05]), pts, n_closest_points=7)
    assert_parity(est.predict(pts), zo, R64, "Krige.predict")
    assert "execute_knn_points" in est.model._kb_handle.calls
    uni = Krige(method="universal", variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05],
                drift_terms=["regional_linear"])
    uni.fit(xyz, val)
    zo, _ = ko.krige(xyz, val, "exponential", ko.stored_parameters("exponential", [1.0, 300.0, 0.05]), pts, regional_linear=True)
    assert_parity(uni.predict(pts), zo, R64, "Krige(universal).predict")


@pytest.fixture(scope="module")
def ref_fuzz():
    import os
    from conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))


@pytest.mark.parametrize("t", range(cases.N_FUZZ))
def test_randomised_configurations_through_the_host_wrappers(pk, t, ref_fuzz):
    """tests/cases.py fuzz_config(t): classes x styles x drift kinds x anisotropy x exact_values x moving window, masks and
    specified-drift arrays also transposed, rasters with a descending axis — against the imported reference
    (tests/golden/ref_fuzz.npz)."""
    import warnings
    c = cases.fuzz_config(t)
    if c is None:
        pytest.skip("over-determined draw")
    if "%d/exc" % t in ref_fuzz.files:
        with pytest.raises(Exception) as ei:
            getattr(pk, c["cls"])(*c["data"], **c["kw"]).execute(c["style"], *c["pts"], backend="cuda", **c["ekw"])
        assert type(ei.value).__name__ == str(ref_fuzz["%d/exc" % t]), c["text"]
        return
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        z, ss = getattr(pk, c["cls"])(*c["data"], **c["kw"]).execute(c["style"], *c["pts"], backend="cuda", **c["ekw"])
    zr, sr, mr = ref_fuzz["%d/z" % t], ref_fuzz["%d/ss" % t], ref_fuzz["%d/mask" % t]
    assert z.shape == zr.shape and ss.shape == sr.shape, c["text"]
    if c["style"] == "masked":
        assert np.array_equal(np.ma.getmaskarray(z), mr) and np.array_equal(np.ma.getmaskarray(ss), mr), c["text"]
        keep = ~mr
        z, ss, zr, sr = np.ma.getdata(z)[keep], np.ma.getdata(ss)[keep], zr[keep], sr[keep]
    if zr.size:
        assert_parity(np.ravel(z), np.ravel(zr), 1e-6, c["text"] + " z")
        assert_parity(np.ravel(ss), np.ravel(sr), 1e-6, c["text"] + " ss")


def test_emulator_keeps_the_signatures_of_the_real_handle():
    """The emulator stands in for _cabi.Handle: every method it offers exists on the real class with the same parameter
    names in the same order (so a change of the C-ABI binding cannot silently leave the emulated tests behind)."""
    import inspect
    from pykrige_b200 import _cabi
    for name, fn in inspect.getmembers(EmulatedHandle, predicate=inspect.isfunction):
        if name.startswith("_"):
            continue
        real = getattr(_cabi.Handle, name, None)
        assert real is not None, "Handle has no method %s" % name
        mine = list(inspect.signature(fn).parameters)
        theirs = list(inspect.signature(real).parameters)
        assert [p.replace("stream", "cuda_stream") if name == "set_stream" else p for p in mine] == theirs, (name, mine, theirs)


def test_verbose_constructors_with_a_device_present(monkeypatch, capsys):
    """verbose=True makes the UK / 3-D constructors compute the cross-validation statistics where the reference does
    (uk.py:380-394: BEFORE the drift terms are initialised). With a device present that goes through _ensure_problem,
    which must then describe the ordinary-kriging system — not trip over drift attributes that do not exist yet
    (seen with a device present: AttributeError 'point_log_drift')."""
    import pykrige_b200 as pk
    from pykrige_b200 import _cabi
    monkeypatch.setattr(_cabi, "Handle", EmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", lambda: EmulatedHandle())      # device_available() -> True
    named = cases.api_inputs()
    x, y, zc, v = named["x"], named["y"], named["zc"], named["v"]
    uk = pk.UniversalKriging(x, y, v, variogram_model="linear", variogram_parameters=[0.01, 0.1], verbose=True,
                             drift_terms=["regional_linear", "point_log", "external_Z", "specified", "functional"],
                             point_drift=named["wells"], external_drift=named["dem"], external_drift_x=named["demx"],
                             external_drift_y=named["demy"], specified_drift=[named["sx"] * named["sy"]], functional_drift=[named["f_sin"]])
    out = capsys.readouterr().out
    assert out.index("Calculating statistics") < out.index("Q1 =") < out.index("Initializing drift terms...")
    assert uk.point_log_drift and uk.external_Z_drift and uk.specified_drift and uk.functional_drift
    assert "set_problem" in uk._kb_handle.calls and uk._kb_handle.problem["n_rl"] == 0 and not uk._kb_handle.problem["hd"]
    z, ss = uk.execute("points", named["gx5"], named["gy"], backend="cuda", specified_drift_arrays=[named["z5"]])
    assert uk._kb_handle.problem["n_rl"] == 2 and len(uk._kb_handle.problem["hd"]) == 5      # described again, with the drift
    u3 = pk.UniversalKriging3D(x, y, zc, v, variogram_model="linear", variogram_parameters=[0.01, 0.1], verbose=True,
                               drift_terms=["regional_linear", "specified", "functional"], specified_drift=[named["sx"] * named["sy"]],
                               functional_drift=[named["f_xyz"]])
    assert u3.specified_drift and u3.functional_drift and u3.Q1 is not None
    u3.update_variogram_model("gaussian", [2.0, 30.0, 0.1])
    k3 = pk.OrdinaryKriging3D(x, y, zc, v, variogram_model="linear", variogram_parameters=[0.01, 0.1], verbose=True)
    assert k3.Q1 is not None


@pytest.mark.parametrize("case", cases.API_CASES, ids=[c["name"] for c in cases.API_CASES])
def test_host_api_cases_with_a_device_present(case, monkeypatch):
    """The API cases of tests/test_host.py once more with a (emulated) device visible to the constructors: every place
    that may touch the device before the object is complete (constructor-time statistics under verbose=True,
    update_variogram_model) must behave as on a CPU-only box — same outcome, same exception, same stdout apart from the
    last digits of the statistics."""
    import json
    import os
    from conftest import GOLDEN
    import pykrige_b200 as pk
    from pykrige_b200 import _cabi
    monkeypatch.setattr(_cabi, "Handle", EmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", lambda: EmulatedHandle())
    d = np.load(os.path.join(GOLDEN, "ref_api.npz"))
    want = json.loads(str(d["@meta"]))[case["name"]]
    got = cases.api_run(pk, case, cases.api_inputs(), backend="cuda")
    if case["name"].endswith("_execute_masked_1d"):          # tests/test_host.py: API_KNOWN_DIFFERENCES
        assert got["exc"] == "ValueError"
        return
    assert (got["kind"], got["exc"], got["msg"]) == (want["kind"], want["exc"], want["msg"])

    def strip_stats(text):
        return "\n".join(ln for ln in text.split("\n") if not ln.startswith(("Q1 =", "Q2 =", "cR =")))
    assert strip_stats(got["stdout"]) == strip_stats(want["stdout"])
    assert got["warnings"] == want["warnings"]


@pytest.mark.parametrize("t", range(cases.N_SEQ))
def test_stateful_sequences_through_the_host_wrappers(pk, t, ref_fuzz):
    """execute / update_variogram_model (also with a new anisotropy) / execute on one object (tests/cases.py seq_config):
    the cached device problem follows the variogram and the re-adjusted data; point_log wells keep their original
    frame, functional drift sees the new one — as the imported reference (ref_fuzz.npz 'seq*')."""
    import warnings
    c = cases.seq_config(t)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        outs = cases.seq_run(pk, c, "cuda")
    assert outs
    for k, (z, ss) in enumerate(outs):
        assert_parity(np.ravel(z), np.ravel(ref_fuzz["seq%d/%d/z" % (t, k)]), 1e-6, c["text"] + " z step %d" % k)
        assert_parity(np.ravel(ss), np.ravel(ref_fuzz["seq%d/%d/ss" % (t, k)]), 1e-6, c["text"] + " ss step %d" % k)


@pytest.mark.parametrize("t", range(cases.N_KIND))
def test_randomised_special_kinds_through_the_host_wrappers(pk, t, ref_fuzz):
    """tests/cases.py kind_config(t): geographic coordinates, pseudo_inv with redundant points, exact duplicates without
    it (LinAlgError, as scipy.linalg.inv in the reference), custom variogram callables (also UK / anisotropy), each with
    and without the moving window — against the imported reference (ref_fuzz.npz 'kind*')."""
    import warnings
    c = cases.kind_config(t)

    def run():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return getattr(pk, c["cls"])(*c["data"], **c["kw"]).execute(c["style"], *c["pts"], backend="cuda", **c["ekw"])
    if "kind%d/exc" % t in ref_fuzz.files:
        with pytest.raises(Exception) as ei:
            run()
        assert type(ei.value).__name__ == str(ref_fuzz["kind%d/exc" % t]), c["text"]
        return
    z, ss = run()
    zr, sr = ref_fuzz["kind%d/z" % t], ref_fuzz["kind%d/ss" % t]
    assert z.shape == zr.shape, c["text"]
    keep = ~np.ma.getmaskarray(z) if c["style"] == "masked" else np.ones(zr.shape, bool)
    if keep.any():
        R = 2e-5 if c["kind"] == "pinv" else 1e-6          # scipy's pinv / pinvh differ from each other at 1e-6 on these
        assert_parity(np.ma.getdata(z)[keep], zr[keep], R, c["text"] + " z")
        assert_parity(np.ma.getdata(ss)[keep], sr[keep], R, c["text"] + " ss")
