"""CPU tests of the host side: reference-facing API behaviour (the error checks of ok.py:834-874,
uk.py:1169-1274, ok3d.py:833-876), parameter normalisation (core.py:196-376), anisotropy
(core.py:120-193), and the C-ABI library (loads, exports every symbol of include/krige_b200.h,
fails loudly without a GPU)."""
import ctypes
import os
import re
import numpy as np
import pytest
from numpy.testing import assert_allclose

import pykrige_b200 as pk
from pykrige_b200 import core, _cabi, multigpu, variogram_models as vm
from oracle import krige_oracle as ko
import cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "krige_b200.h")).read()
    declared = set(re.findall(r"\b(kb200_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_cabi.EXPORTS), declared ^ set(_cabi.EXPORTS)
    lib = _cabi.load_library()
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.kb200_version() >= 1000


def test_group_offers_only_what_a_group_can_serve():
    """_cabi.Group shares the error mapping, the problem marshalling and the host execute calls with _cabi.Handle, but
    not the handle-only calls: those would hand the group's pointer to kb200_* functions that expect a handle."""
    for name in ("set_stream", "set_values", "blob_commit", "execute_grid_dev", "execute_points_dev",
                 "execute_knn_grid_dev", "experimental_variogram", "loo", "knn_loo", "debug_fetch"):
        assert hasattr(_cabi.Handle, name), name
        assert not hasattr(_cabi.Group, name), name
    for name in ("set_problem", "set_problem_knn", "execute_points", "execute_grid", "execute_knn_points",
                 "execute_knn_grid", "set_coordinates", "set_pseudo_inverse", "set_variogram_table",
                 "set_device_drift", "reset_counters", "timings", "statistics", "blob"):
        assert hasattr(_cabi.Group, name), name


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_cabi.KrigeB200Error):
        _cabi.Handle()
    ok = pk.OrdinaryKriging([0, 1, 2.0], [0, 1, 0.5], [1, 2, 3.0], variogram_parameters=[1.0, 0.1])
    with pytest.raises(_cabi.KrigeB200Error):
        ok.execute("points", [0.5], [0.5], backend="cuda")


def test_variogram_models_match_oracle():
    d = np.linspace(0.0, 900.0, 301)
    for name, plist in cases.MODELS.items():
        stored = ko.stored_parameters(name, plist)
        f = pk.OrdinaryKriging.variogram_dict[name]
        assert_allclose(f(stored, d), ko.variogram(name, stored, d), rtol=1e-14, atol=1e-15)
        assert f.__name__ in vm.DEVICE_MODEL_IDS


def test_parameter_list_normalisation():
    """tests/test_core.py:114-181: list form is FULL sill -> psill; dict may give sill or psill."""
    assert core._make_variogram_parameter_list("linear", [1.5, 0.2]) == [1.5, 0.2]
    assert core._make_variogram_parameter_list("power", [1.5, 1.2, 0.2]) == [1.5, 1.2, 0.2]
    for m in ("gaussian", "spherical", "exponential", "hole-effect"):
        assert core._make_variogram_parameter_list(m, [2.0, 10.0, 0.5]) == [1.5, 10.0, 0.5]
        assert core._make_variogram_parameter_list(m, {"sill": 2.0, "range": 10.0, "nugget": 0.5}) == [1.5, 10.0, 0.5]
        assert core._make_variogram_parameter_list(m, {"psill": 1.5, "range": 10.0, "nugget": 0.5}) == [1.5, 10.0, 0.5]
        with pytest.raises(KeyError):
            core._make_variogram_parameter_list(m, {"range": 10.0, "nugget": 0.5})
    assert core._make_variogram_parameter_list("linear", {"slope": 1.0, "nugget": 0.1}) == [1.0, 0.1]
    with pytest.raises(ValueError):
        core._make_variogram_parameter_list("linear", [1.0])
    with pytest.raises(TypeError):
        core._make_variogram_parameter_list("linear", (1.0, 0.1))
    with pytest.raises(TypeError):
        core._make_variogram_parameter_list("custom", {"a": 1})
    assert core._make_variogram_parameter_list("exponential", None) is None


def test_anisotropy_matches_oracle():
    rng = np.random.default_rng(0)
    X2 = rng.normal(size=(50, 2)) * 100
    X3 = rng.normal(size=(50, 3)) * 100
    assert_allclose(core._adjust_for_anisotropy(X2, [3.0, -2.0], [1.7], [33.0]),
                    ko.adjust_for_anisotropy(X2, [3.0, -2.0], [1.7], [33.0]), rtol=1e-13, atol=1e-11)
    assert_allclose(core._adjust_for_anisotropy(X3, [3.0, -2.0, 5.0], [1.4, 3.0], [10.0, -25.0, 40.0]),
                    ko.adjust_for_anisotropy(X3, [3.0, -2.0, 5.0], [1.4, 3.0], [10.0, -25.0, 40.0]),
                    rtol=1e-13, atol=1e-11)
    # tests/test_core.py:83-111 known rotation
    x = np.array([[1.0, 0.0], [0.0, 1.0]])
    out = core._adjust_for_anisotropy(x, [0.0, 0.0], [2.0], [90.0])
    assert_allclose(out, [[0.0, -2.0], [1.0, 0.0]], atol=1e-12)


def test_fitted_variogram_is_reasonable():
    xyz, val = cases.synth_data(5, 150, 2)
    ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="spherical", nlags=8)
    p = ok.variogram_model_parameters
    assert len(p) == 3 and p[0] >= 0 and p[1] > 0 and p[2] >= 0
    assert ok.lags.size == ok.semivariance.size <= 8
    lags, g = ok.get_variogram_points()
    assert_allclose(g, vm.spherical_variogram_model(p, lags))


def test_variogram_functions_and_automatic_fit_reproduce_the_reference():
    """variogram_parameters=None (ok.py:326-346 -> core.py:582-651): the soft-L1 least-squares fit amplifies a last-ulp
    difference of the model function (spherical: ~5e-4 in the fitted parameters), so the six host functions follow the
    reference's operation order bit for bit (tests/golden/ref_vgfit.npz, generated from the imported reference by
    make_golden.py vgfit) and the fitted parameters agree to 1e-9."""
    ref = np.load(os.path.join(ROOT, "tests", "golden", "ref_vgfit.npz"))
    same_cpu = str(ref["cpu_fingerprint"]) == cases.cpu_fingerprint()
    d = cases.vgfit_distances()
    for m in cases.VGFIT_MODELS:
        g = pk.OrdinaryKriging.variogram_dict[m](cases.VGFIT_PARAMS[m], d.copy())
        if same_cpu:      # same numpy + SIMD dispatch as the generator: identical bit patterns
            assert np.array_equal(g, ref["gamma/" + m]), (m, np.max(np.abs(g - ref["gamma/" + m])))
        else:
            np.testing.assert_array_max_ulp(g, ref["gamma/" + m], maxulp=4)
    for n in (60, 300):
        x, y, z = cases.vgfit_inputs(n)
        for m in cases.VGFIT_MODELS:
            for w in (False, True):
                ok = pk.OrdinaryKriging(x, y, z, variogram_model=m, weight=w, nlags=8)
                pr = ref["fit/%d/%s/%d" % (n, m, int(w))]
                tol = 1e-9 if same_cpu else 2e-3
                assert_allclose(ok.variogram_model_parameters, pr, rtol=tol, atol=tol * np.abs(pr).max(),
                                err_msg="%s N=%d weight=%s" % (m, n, w))


# ---- host mirror vs the imported reference: everything the four classes do before the device call -----------------
@pytest.fixture(scope="module")
def ref_api():
    import json
    d = np.load(os.path.join(ROOT, "tests", "golden", "ref_api.npz"))
    return json.loads(str(d["@meta"])), d


# places where this package deliberately differs from the reference (each one a crash in the reference)
API_KNOWN_DIFFERENCES = {
    # a 1-D mask on a 2-D grid: IndexError in mask.shape[1] in the reference; here the ValueError of ok.py:855
    "ok_execute_masked_1d": ("ValueError", "Mask is not two-dimensional."),
    "uk_execute_masked_1d": ("ValueError", "Mask is not two-dimensional."),
}


@pytest.mark.parametrize("case", cases.API_CASES, ids=[c["name"] for c in cases.API_CASES])
def test_host_api_matches_reference(case, ref_api):
    """Constructors, update_variogram_model and the argument validation of execute() (tests/cases.py API_CASES)
    against tests/golden/ref_api.npz (the UNMODIFIED imported reference, make_golden.py api): same public attributes
    (bit for bit on the generating CPU), same stdout under verbose=True, same warnings, same exception types and
    messages."""
    meta, arrays = ref_api
    want = meta[case["name"]]
    got = cases.api_run(pk, case, cases.api_inputs(), backend="cuda")
    if case["name"] in API_KNOWN_DIFFERENCES:
        assert (got["exc"], got["msg"]) == API_KNOWN_DIFFERENCES[case["name"]]
        return
    device = _cabi.device_available()       # with a device the statistics come from kb200_statistics (1e-6 parity)
    exact = (not device) and str(np.load(os.path.join(ROOT, "tests", "golden", "ref_vgfit.npz"))["cpu_fingerprint"]) \
        == cases.cpu_fingerprint()

    def strip_stats(text):
        return "\n".join(ln for ln in text.split("\n") if not ln.startswith(("Q1 =", "Q2 =", "cR =")))

    assert got["kind"] == want["kind"], (got["exc"], got["msg"], want["exc"], want["msg"])
    if want["kind"] == "exc":
        assert (got["exc"], got["msg"]) == (want["exc"], want["msg"])
        assert (got["stdout"] == want["stdout"]) if exact else (strip_stats(got["stdout"]) == strip_stats(want["stdout"]))
        return
    if exact:
        assert got["stdout"] == want["stdout"]
    else:
        assert strip_stats(got["stdout"]) == strip_stats(want["stdout"])
    assert got["warnings"] == want["warnings"]
    for k, v in want["attrs"].items():
        assert k in got["attrs"], "attribute %s missing" % k
        g = got["attrs"][k]
        if v == "@array":
            r = arrays[case["name"] + "/" + k]
            assert np.shape(g) == r.shape, k
            if exact:
                assert np.array_equal(g, r, equal_nan=True), (k, np.max(np.abs(g - r)))
            else:
                tol = 1e-6 if k in cases.API_STAT_ATTRS else (2e-3 if k in ("variogram_model_parameters",) else 1e-9)
                assert_allclose(g, r, rtol=tol, atol=tol * (np.abs(r).max() if r.size else 0.0), err_msg=k)
        else:
            assert g == v, (k, g, v)
    if case["name"] + "/@ret" in arrays.files:
        assert_allclose(got["ret"], arrays[case["name"] + "/@ret"], rtol=0 if exact else 1e-6)


def test_constructor_and_execute_argument_errors():
    xyz, val = cases.synth_data(1, 20, 2)
    with pytest.raises(ValueError):
        pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="blurg")
    with pytest.raises(ValueError):
        pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, exact_values="blurg")
    with pytest.raises(ValueError):
        pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="custom")
    with pytest.raises(ValueError):
        pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, pseudo_inv_type="nope")
    ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_parameters=[1.0, 0.1])
    gx, gy = np.arange(4.0), np.arange(3.0)
    with pytest.raises(ValueError):
        ok.execute("blurg", gx, gy)
    with pytest.raises(IOError):
        ok.execute("masked", gx, gy)
    with pytest.raises(ValueError):
        ok.execute("masked", gx, gy, mask=np.zeros((5, 5), bool))
    with pytest.raises(ValueError):
        ok.execute("points", np.arange(3.0), np.arange(4.0))
    with pytest.raises(ValueError):
        ok.execute("grid", gx, gy, n_closest_points=1)
    with pytest.raises(ValueError):
        ok.execute("grid", gx, gy, backend="vectorized")   # CPU backends live in the reference
    uk = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, variogram_parameters=[1.0, 0.1], drift_terms=["specified"],
                             specified_drift=[val])
    with pytest.raises(ValueError):
        uk.execute("grid", gx, gy)                          # specified drift arrays missing
    with pytest.raises(TypeError):
        pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, drift_terms=["functional"], functional_drift=lambda x, y: x,
                            variogram_parameters=[1.0, 0.1])
    with pytest.raises(ValueError):
        pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, drift_terms=["external_Z"], variogram_parameters=[1.0, 0.1])
    x3, v3 = cases.synth_data(2, 20, 3)
    k3 = pk.OrdinaryKriging3D(x3[:, 0], x3[:, 1], x3[:, 2], v3, variogram_parameters=[1.0, 0.1])
    with pytest.raises(ValueError):
        k3.execute("masked", gx, gy, gx, mask=np.zeros((2, 2), bool))
    with pytest.raises(IOError):
        k3.execute("masked", gx, gy, gx)
    assert k3._stats_state == "lazy"                        # O(N^4) statistics deferred (SURVEY F5)
    assert k3.Q1 is not None and k3._stats_state == "done"
    assert ok.Q1 is None                                    # enable_statistics=False (ok.py:360-377)


def test_external_z_sampler_matches_bilinear():
    xyz, val = cases.synth_data(4, 30, 2)
    case = cases.CASE_BY_NAME["uk2d_externalz"]
    inp = cases.build_inputs(case)
    uk = cases.make_model(pk, case, inp)
    from scipy.interpolate import RegularGridInterpolator
    f = RegularGridInterpolator((inp["ext_y"], inp["ext_x"]), inp["ext_z"])
    P = inp["points"]
    assert_allclose(uk._calculate_data_point_zscalars(P[:, 0], P[:, 1]), f(np.column_stack((P[:, 1], P[:, 0]))),
                    rtol=1e-12)
    # exactly on a node / on a grid line (degenerate branches of uk.py:560-595)
    xs = np.array([inp["ext_x"][3], inp["ext_x"][3], 0.5 * (inp["ext_x"][3] + inp["ext_x"][4])])
    ys = np.array([inp["ext_y"][5], 0.5 * (inp["ext_y"][5] + inp["ext_y"][6]), inp["ext_y"][5]])
    assert_allclose(uk._calculate_data_point_zscalars(xs, ys), f(np.column_stack((ys, xs))), rtol=1e-12)
    with pytest.raises(ValueError):
        uk._calculate_data_point_zscalars(np.array([1e6]), np.array([0.0]))


def test_shard_ranges_cover_exactly():
    for count in (0, 1, 7, 1000, 10**6 + 3):
        for world in (1, 2, 3, 4, 8):
            spans = [multigpu.shard_range(count, r, world) for r in range(world)]
            assert spans[0][0] == 0
            for (f0, c0), (f1, c1) in zip(spans, spans[1:]):
                assert f0 + c0 == f1
            assert spans[-1][0] + spans[-1][1] == count
            sizes = [c for _, c in spans]
            assert max(sizes) - min(sizes) <= 1


# ---- constructor side: host mirror of the experimental variogram / statistics ------------------
@pytest.mark.parametrize("case", cases.VARIOGRAM_CASES[:4] + cases.VARIOGRAM_CASES[6:10],
                         ids=lambda c: c["name"])
def test_host_experimental_variogram_matches_reference(case, ref_ctor):
    from pykrige_b200 import core
    X, y = cases.build_ctor_inputs(case)
    for block in (2048, 97):             # the row-blocked accumulation must not depend on the block size
        lags, semi = core._experimental_variogram(X, y, case["nlags"], block=block,
                                                  coordinates_type=case["coordinates_type"], device=False)
        assert_allclose(lags, ref_ctor[case["name"] + "/lags"], rtol=1e-10)
        assert_allclose(semi, ref_ctor[case["name"] + "/semi"], rtol=1e-10)


def test_host_statistics_match_reference(ref_ctor):
    from pykrige_b200 import core, variogram_models as vm
    case = cases.STATS_CASES[0]
    X, y = cases.build_ctor_inputs(case)
    d, s, e = core._find_statistics(X, y, vm.exponential_variogram_model, case["params"], "euclidean")
    assert_allclose(d, ref_ctor[case["name"] + "/delta"], rtol=1e-8, atol=1e-10)
    assert_allclose(s, ref_ctor[case["name"] + "/sigma"], rtol=1e-8)
    assert_allclose(e, ref_ctor[case["name"] + "/epsilon"], rtol=1e-8, atol=1e-10)


# ---- whole-chain scenarios: constructor (binning + least-squares fit) vs the imported reference ----
@pytest.mark.parametrize("sc", cases.SCENARIOS, ids=[s["name"] for s in cases.SCENARIOS])
def test_fitted_variogram_matches_reference(sc, ref_scenarios, ref_goldens):
    """No variogram parameters given: lags, semivariances and the soft-L1 fit must reproduce the
    reference's constructor (ok.py:326-346 -> core.py:379-651). Runs the host binning on a CPU-only
    box and the device binning where a GPU is present; both must land on the same fit."""
    data, _, _ = cases.scenario_inputs(sc, ref_goldens["data"])
    m = cases.scenario_model(pk, sc, data)
    assert_allclose(m.lags, ref_scenarios[sc["name"] + "/lags"], rtol=1e-10)
    assert_allclose(m.semivariance, ref_scenarios[sc["name"] + "/semi"], rtol=1e-10)
    pr = ref_scenarios[sc["name"] + "/params"]
    assert_allclose(m.variogram_model_parameters, pr, rtol=1e-6, atol=1e-7 * np.abs(pr).max())


# ---- 'custom' callables: host-side tabulation helpers (the device interpolation is in the GPU tests) ----
def test_custom_variogram_table_helpers():
    xyz, val = cases.synth_data(3, 60, 2)
    fn = lambda m, d: m[0] * np.log10(d + m[1]) + m[2]
    ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="custom", variogram_parameters=[1.0, 1.0, 1.0],
                            variogram_function=fn, anisotropy_scaling=2.0, anisotropy_angle=30.0)
    mid, vp = ok._device_model()
    assert mid == ok.TABLE_MODEL_ID == 6 and vp == []
    d0 = ok._table_dmax()
    # covers every data-data distance in the ADJUSTED frame with head-room
    A = np.column_stack((ok.X_ADJUSTED, ok.Y_ADJUSTED))
    span = np.sqrt(((A[:, None, :] - A[None, :, :]) ** 2).sum(-1)).max()
    assert d0 >= 2.0 * span
    assert ok._table_dmax() == d0                                   # stable
    d1 = ok._table_dmax([-5000.0, -5000.0], [9000.0, 9000.0])       # far prediction window: grows
    assert d1 > d0 and ok._table_dmax([0.0, 0.0], [10.0, 10.0]) == d1   # and never shrinks
    g = ok._variogram_table(d1)
    n = ok.TABLE_NODES
    assert g.shape == (n,) and g[0] == fn([1.0, 1.0, 1.0], 0.0)
    assert_allclose(g[-1], fn([1.0, 1.0, 1.0], d1), rtol=1e-14)
    i = n // 3
    assert_allclose(g[i], fn([1.0, 1.0, 1.0], d1 * (i / (n - 1)) ** 2), rtol=1e-14)   # sqrt-spaced nodes
    assert ok._variogram_table(d1) is g                              # cached per (callable, parameters, dmax)
    bad = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="custom", variogram_parameters=[1.0],
                             variogram_function=lambda m, d: m[0] * np.log(d))
    with pytest.raises(ValueError):
        bad._variogram_table(100.0)
    # built-in models keep their closed forms
    lin = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="linear", variogram_parameters=[0.01, 0.1])
    assert lin._device_model() == (0, [0.01, 0.1])


def test_ctypes_signatures_match_the_header():
    """Every prototype of include/krige_b200.h has a ctypes binding with the same number of parameters and
    compatible kinds (pointer / integer / double) — ABI drift between the header and pykrige_b200/_cabi.py
    would otherwise only show up as memory corruption on the GPU box."""
    lib = _cabi.load_library()
    text = open(os.path.join(ROOT, "include", "krige_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = re.findall(r"\n\s*(?:int64_t|int|void\s*\*|const char\s*\*|void|kb200_handle)\s*\*?\s*(kb200_\w+)\s*\(([^;]*?)\)\s*;", text)
    assert len(protos) >= 37
    assert sorted(n for n, _ in protos) == sorted(_cabi.EXPORTS)
    for name, params in protos:
        fn = getattr(lib, name)
        plist = [p.strip() for p in params.replace("\n", " ").split(",") if p.strip() and p.strip() != "void"]
        if fn.argtypes is None:
            assert name in ("kb200_version",), name
            continue
        assert len(fn.argtypes) == len(plist), (name, len(fn.argtypes), plist)
        for ct, decl in zip(fn.argtypes, plist):
            is_ptr = "*" in decl or "kb200_handle" in decl or "kb200_group" in decl
            if is_ptr:
                assert ct in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(ct, ctypes._Pointer), (name, decl, ct)
            elif decl.startswith("double"):
                assert ct is ctypes.c_double, (name, decl, ct)
            else:
                assert ct in (ctypes.c_int, ctypes.c_int64), (name, decl, ct)


def test_gstools_route_on_the_host():
    """ok.py:224-239 / ok3d.py:248-262 with a stand-in gstools package (tests/gstools_stub.py): a CovModel becomes a
    'custom' model whose callable is model.pykrige_vario, the anisotropy comes from the model, the dimension and
    version checks of compat_gstools.py:21-37 raise as in the reference."""
    import gstools_stub
    from pykrige_b200.compat_gstools import GSToolsException
    xyz, val = cases.synth_data(5, 40, 2)
    try:
        gstools_stub.install("1.5.2")
        m = gstools_stub.CovModel(dim=2, var=2.0, len_scale=150.0, nugget=0.1, anis=0.5, angle=20.0)
        ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, m)
        assert ok.variogram_model == "custom" and ok.model is m
        assert ok.variogram_model_parameters == []
        assert ok.anisotropy_scaling == m.pykrige_anis and ok.anisotropy_angle == m.pykrige_angle
        d = np.linspace(0.0, 500.0, 7)
        assert_allclose(ok.variogram_function(ok.variogram_model_parameters, d), m.variogram(d), rtol=0, atol=0)
        assert ok._device_model() == (ok.TABLE_MODEL_ID, [])           # tabulated on the device
        uk = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, m, drift_terms=["regional_linear"])
        assert uk.variogram_model == "custom"
        with pytest.raises(ValueError):                                 # 3-D model on a 2-D class
            pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, gstools_stub.CovModel(dim=3))
        with pytest.raises(ValueError):                                 # latlon model needs geographic coordinates
            pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, gstools_stub.CovModel(dim=2, latlon=True))
        x3, v3 = cases.synth_data(6, 30, 3)
        with pytest.raises(ValueError):                                 # 2-D model on a 3-D class
            pk.OrdinaryKriging3D(x3[:, 0], x3[:, 1], x3[:, 2], v3, gstools_stub.CovModel(dim=2))
        k3 = pk.OrdinaryKriging3D(x3[:, 0], x3[:, 1], x3[:, 2], v3, gstools_stub.CovModel(dim=3, anis=0.5))
        assert k3.anisotropy_scaling_y == 2.0 and k3.variogram_model == "custom"
        gstools_stub.install("1.2.0")
        with pytest.raises(GSToolsException):
            pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, m)
        gstools_stub.install("1.3.0")
        with pytest.raises(GSToolsException):                           # latlon needs >= 1.4
            pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, gstools_stub.CovModel(dim=2, latlon=True),
                               coordinates_type="geographic")
    finally:
        gstools_stub.uninstall()
    with pytest.raises(GSToolsException):                               # gstools absent
        pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, m)


def _blocked_gauss_jordan(A, nb):
    """The algebra csrc/factor.cu's general path runs (gj_panel_kernel / gj_swap_copy_kernel / gj_gemm_kernel), in numpy:
    nb pivoted scalar steps restricted to the column panel, the recorded row swaps and ONE rank-nb update of all other
    columns, column swaps in reverse at the end."""
    A = A.copy()
    n = A.shape[0]
    piv = np.arange(n)
    for k0 in range(0, n, nb):
        P = A[:, k0:k0 + nb].copy()
        for j in range(nb):
            kk = k0 + j
            p = kk + int(np.argmax(np.abs(P[kk:, j])))
            piv[kk] = p
            P[[kk, p]] = P[[p, kk]]
            inv = 1.0 / P[kk, j]
            rv = P[kk] * inv
            rv[j] = inv
            col = P[:, j].copy()
            P -= np.outer(col, rv)
            P[:, j] = -col * inv
            P[kk] = rv
        other = np.r_[0:k0, k0 + nb:n]
        R = A[:, other]
        for j in range(nb):
            kk, p = k0 + j, piv[k0 + j]
            R[[kk, p]] = R[[p, kk]]
        T = R[k0:k0 + nb].copy()
        R[k0:k0 + nb] = 0.0
        A[:, other] = R + P @ T
        A[:, k0:k0 + nb] = P
    for k in range(n - 1, -1, -1):
        A[:, [k, piv[k]]] = A[:, [piv[k], k]]
    return A


def test_blocked_gauss_jordan_algebra():
    """64 scalar Gauss-Jordan steps compose into the block exchange of the pivot block against the rest, with the row
    swaps deferred to the other columns: pins the algebra of the device's general (indefinite) path against
    numpy.linalg.inv on a symmetric indefinite matrix padded with an identity block, as the device pads it."""
    rng = np.random.default_rng(5)
    n, n_pad = 150, 192
    M = rng.standard_normal((n, n))
    M = M + M.T
    assert np.linalg.eigvalsh(M).min() < 0 < np.linalg.eigvalsh(M).max()
    A = np.eye(n_pad)
    A[:n, :n] = M
    G = _blocked_gauss_jordan(A, 64)
    assert_allclose(G[:n, :n], np.linalg.inv(M), rtol=0, atol=1e-10 * np.abs(np.linalg.inv(M)).max())
    assert_allclose(G[n:, n:], np.eye(n_pad - n), atol=0)
    assert np.all(G[:n, n:] == 0.0) and np.all(G[n:, :n] == 0.0)
    assert_allclose(_blocked_gauss_jordan(A, 1), G, atol=1e-10 * np.abs(G).max())      # the column-at-a-time form
