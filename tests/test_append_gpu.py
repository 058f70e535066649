"""add_data() on the H100 (run with -m gpu): kb200_append_data extends the held factorisation by a block row
(DESIGN.md §5g), and every result afterwards equals that of a new object built on the old stations followed by the new
ones with the current variogram fixed: execute() at max|d| / max|ref| <= 1e-9 in float64 and the solve tolerances of
tests/test_solve_boundaries_gpu.py in float32 / float64x, leave_one_out(), leave_group_out() and the statistics at
1e-9, across the 64-row tile boundaries, an n_pad reallocation and a chain of appends; the stored reference goldens
split into a first and an appended part; and the cases that fall back."""
import numpy as np
import pytest

import cases
from conftest import assert_parity

pytestmark = pytest.mark.gpu
NAMES = {"linear": ("slope", "nugget"), "power": ("scale", "exponent", "nugget")}
PARAMS = {"exponential": [1.0, 300.0, 0.05], "spherical": [2.0, 450.0, 0.1], "gaussian": [1.5, 500.0, 0.2],
          "linear": [0.01, 0.05], "power": [0.2, 1.4, 0.05], "hole-effect": [1.0, 900.0, 0.05]}
TOL = {"float64": 1e-9, "float32": 5e-4, "float64x": 1e-8}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


def fixed(model):
    p = list(model.variogram_model_parameters)
    return dict(zip(NAMES.get(model.variogram_model, ("psill", "range", "nugget")), p))


def make(pk, kind, xyz, val, model="exponential", params=None, **kw):
    params = kw.pop("variogram_parameters", params)
    kw = dict(variogram_model=model, variogram_parameters=PARAMS[model] if params is None else params, **kw)
    if kind == "ok":
        return pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, **kw)
    if kind == "uk":
        return pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, **kw)
    if kind == "ok3d":
        return pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], val, **kw)
    return pk.UniversalKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], val, **kw)


def add(model, xyz, val, spec=None):
    args = [xyz[:, c] for c in range(xyz.shape[1])] + [val]
    model.add_data(*args, specified_drift=spec)


def points(dim, seed=11, m=700):
    rng = np.random.default_rng(seed)
    box = (1000.0, 1000.0, 250.0)
    return [rng.uniform(-20.0, box[c] + 20.0, m) for c in range(dim)]


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


def compare(model, ref, pts, tol, **kw):
    z, s = model.execute("points", *pts, **kw)
    zr, sr = ref.execute("points", *pts, **kw)
    assert rel(z, zr) <= tol, rel(z, zr)
    assert rel(s, sr) <= tol, rel(s, sr)
    return z, s


def uk_drift(n_all, seed=5):
    """UK with regional_linear + point_log + external_Z + specified + functional (no anisotropy: the functional term
    sees the adjusted coordinates). Returns (constructor kwargs without the specified arrays, specified data, a function
    giving the specified drift at points)."""
    rng = np.random.default_rng(seed)
    ex, ey = np.linspace(-100.0, 1100.0, 41), np.linspace(-100.0, 1100.0, 37)
    gx, gy = np.meshgrid(ex, ey)
    kw = dict(drift_terms=["regional_linear", "point_log", "external_Z", "specified", "functional"],
              point_drift=[[480.0, 520.0, 0.7], [100.0, 900.0, 0.3]], external_drift=20.0 + 0.01 * gx + np.sin(gy / 170.0),
              external_drift_x=ex, external_drift_y=ey, functional_drift=[lambda x, y: np.sin(x / 300.0) * y / 1000.0])
    spec = rng.normal(size=n_all)
    return kw, spec, (lambda pts: [np.cos(pts[0] / 200.0)])


SIZES = [(63, 1), (64, 63), (64, 64), (65, 65), (255, 1), (256, 300), (257, 64), (4000, 64)]


@pytest.mark.parametrize("n,m", SIZES)
def test_ok_sizes_float64(pk, n, m):
    """OK with anisotropy across the tile edges: n_pad unchanged (in place) and grown (reallocated)."""
    xyz, val = cases.synth_data(n + m, n + m, 2)
    kw = dict(anisotropy_scaling=1.7, anisotropy_angle=35.0)
    model = make(pk, "ok", xyz[:n], val[:n], **kw)
    pts = points(2)
    model.execute("points", *pts)
    h = model._kb_handle
    h.reset_counters()
    add(model, xyz[n:], val[n:])
    model.execute("points", *pts)
    appended = h.timings()["launches"]
    ref = make(pk, "ok", xyz, val, variogram_parameters=fixed(model), **kw)
    compare(model, ref, pts, TOL["float64"])
    assert model._kb_handle is h
    if n >= 4000:                       # no full factorisation: far fewer launches than a new object's first execute
        fresh = make(pk, "ok", xyz, val, variogram_parameters=fixed(model), **kw)
        fresh.execute("points", *pts)
        assert appended < 0.5 * fresh._kb_handle.timings()["launches"], (appended, fresh._kb_handle.timings())


@pytest.mark.parametrize("model_name", ["spherical", "gaussian", "linear", "power"])
@pytest.mark.parametrize("n,m", [(255, 65), (1000, 300)])
def test_models(pk, model_name, n, m):
    xyz, val = cases.synth_data(7 + n, n + m, 2)
    xyz[n:, 0] += 150.0                                    # the bounding box (and for linear / power c0) grows
    model = make(pk, "ok", xyz[:n], val[:n], model_name)
    pts = points(2)
    model.execute("points", *pts)
    add(model, xyz[n:], val[n:])
    ref = make(pk, "ok", xyz, val, model_name, params=fixed(model))
    compare(model, ref, pts, TOL["float64"])


@pytest.mark.parametrize("dtype", ["float32", "float64x"])
def test_dtypes(pk, dtype):
    n, m = 1000, 65
    xyz, val = cases.synth_data(3, n + m, 2)
    model = make(pk, "ok", xyz[:n], val[:n])
    pts = points(2)
    model.execute("points", *pts, dtype=dtype)
    add(model, xyz[n:], val[n:])
    ref = make(pk, "ok", xyz, val, variogram_parameters=fixed(model))
    z, s = model.execute("points", *pts, dtype=dtype)
    zr, sr = ref.execute("points", *pts)                   # float64 of the new object: the dtype's accuracy class
    assert rel(z, zr) <= TOL[dtype] and rel(s, sr) <= TOL[dtype] * 10, (rel(z, zr), rel(s, sr))


@pytest.mark.parametrize("kind", ["uk", "ok3d", "uk3d"])
def test_kinds_and_cross_validation(pk, kind):
    """UK with every drift kind, OK3D and UK3D with anisotropy: execute(), leave_one_out(), leave_group_out() and the
    statistics after add_data equal the new object's; exact hits on appended stations give sigma^2 = 0."""
    n, m = 300, 70
    dim = 3 if kind.endswith("3d") else 2
    xyz, val = cases.synth_data(21, n + m, dim)
    spec_new = None
    kw, pkw = {}, {}
    if kind == "uk":
        kw, spec, spec_at = uk_drift(n + m)
        model = make(pk, kind, xyz[:n], val[:n], specified_drift=[spec[:n]], **kw)
        spec_new, kw = [spec[n:]], dict(kw, specified_drift=[spec])
        pts = points(dim)
        pkw = dict(specified_drift_arrays=spec_at(pts))
    else:
        kw = dict(anisotropy_scaling_y=1.5, anisotropy_angle_z=25.0)
        if kind == "uk3d":
            kw["drift_terms"] = ["regional_linear"]
        model = make(pk, kind, xyz[:n], val[:n], **kw)
        pts = points(dim)
    model.execute("points", *pts, **pkw)
    add(model, xyz[n:], val[n:], spec=spec_new)
    ref = make(pk, kind, xyz, val, variogram_parameters=fixed(model), **kw)
    compare(model, ref, pts, TOL["float64"], **pkw)
    for a, b in zip(model.leave_one_out(), ref.leave_one_out()):
        assert rel(a, b) <= TOL["float64"]
    groups = np.arange(n + m) % 7
    for a, b in zip(model.leave_group_out(groups), ref.leave_group_out(groups)):
        assert rel(a, b) <= TOL["float64"]
    for name in ("delta", "sigma"):
        assert rel(getattr(model, name), getattr(ref, name)) <= TOL["float64"]
    hit = [xyz[n:, c] for c in range(dim)]
    hkw = dict(specified_drift_arrays=[spec[n:]]) if kind == "uk" else {}
    z, s = model.execute("points", *hit, **hkw)
    assert np.abs(s).max() <= 1e-9 * max(np.abs(model.variogram_model_parameters).max(), 1.0)
    assert np.abs(z - val[n:]).max() <= 1e-8 * np.abs(val).max()


def test_chain_of_ten_appends_is_exact_and_repeatable(pk):
    sizes = [500, 1, 13, 64, 65, 2, 100, 37, 63, 1, 120]
    xyz, val = cases.synth_data(99, sum(sizes), 2)
    pts = points(2)

    def run():
        model = make(pk, "uk", xyz[:sizes[0]], val[:sizes[0]], drift_terms=["regional_linear"])
        model.execute("points", *pts)
        n = sizes[0]
        for m in sizes[1:]:
            add(model, xyz[n:n + m], val[n:n + m])
            n += m
        return model, model.execute("points", *pts)
    model, (z1, s1) = run()
    _, (z2, s2) = run()
    assert np.array_equal(z1, z2) and np.array_equal(s1, s2)
    ref = make(pk, "uk", xyz, val, variogram_parameters=fixed(model), drift_terms=["regional_linear"])
    zr, sr = ref.execute("points", *pts)
    assert rel(z1, zr) <= TOL["float64"] and rel(s1, sr) <= TOL["float64"]


def test_duplicate_station_with_zero_nugget_raises_as_a_new_object(pk):
    xyz, val = cases.synth_data(4, 200, 2)
    model = make(pk, "ok", xyz, val, "spherical", params=[2.0, 450.0, 0.0])
    pts = points(2)
    model.execute("points", *pts)
    add(model, xyz[5:6], val[5:6] + 1.0)
    ref = make(pk, "ok", np.vstack([xyz, xyz[5:6]]), np.concatenate([val, val[5:6] + 1.0]), "spherical",
               params=[2.0, 450.0, 0.0])
    with pytest.raises(np.linalg.LinAlgError):
        ref.execute("points", *pts)
    with pytest.raises(np.linalg.LinAlgError):
        model.execute("points", *pts)


@pytest.mark.parametrize("case", ["pseudo_inv", "hole_effect", "moving_window", "custom_beyond_dmax"])
def test_fallbacks_equal_a_new_object(pk, case):
    n, m = 150, 40
    xyz, val = cases.synth_data(8, n + m, 2)
    xyz[n:, 0] += 5000.0 if case == "custom_beyond_dmax" else 300.0   # past the custom table's range
    kw, ekw, model_name = {}, {}, "exponential"
    if case == "pseudo_inv":
        kw = dict(pseudo_inv=True)
    elif case == "hole_effect":
        model_name = "hole-effect"
    elif case == "moving_window":
        ekw = dict(n_closest_points=12)
    else:
        model_name = "custom"
        kw = dict(variogram_function=lambda p, d: p[0] * (1.0 - np.exp(-d / p[1])) + p[2])
    params = [1.0, 300.0, 0.05] if model_name == "custom" else None
    model = make(pk, "ok", xyz[:n], val[:n], model_name, params=params, **kw)
    pts = points(2)
    model.execute("points", *pts, **ekw)
    add(model, xyz[n:], val[n:])
    ref = make(pk, "ok", xyz, val, model_name,
               params=list(model.variogram_model_parameters) if model_name == "custom" else fixed(model), **kw)
    compare(model, ref, pts, TOL["float64"], **ekw)


GOLDEN_CASES = [c for c in cases.CASES if c["k"] is None and c["name"] != "ok2d_hole_effect_small"]


@pytest.mark.parametrize("case", GOLDEN_CASES, ids=[c["name"] for c in GOLDEN_CASES])
def test_reference_goldens_split_into_first_and_appended_part(pk, case, ref_cases):
    """The stored outputs of the imported reference, from an object built on the first 80 % of the stations, executed
    once, and given the rest through add_data."""
    inp = cases.build_inputs(case)
    n = case["n"]
    k = n - max(1, n // 5)
    first = dict(inp, data=inp["data"][:k], values=inp["values"][:k])
    spec_new = None
    if case["n_specified"]:
        first["spec_data"] = [a[:k] for a in inp["spec_data"]]
        spec_new = [a[k:] for a in inp["spec_data"]]
    model = cases.make_model(pk, case, first)
    cases.run_model(model, case, first, "cuda")
    add(model, inp["data"][k:], inp["values"][k:], spec=spec_new)
    z, ss = cases.run_model(model, case, inp, "cuda")
    zr, sr = ref_cases[case["name"] + "/z"], ref_cases[case["name"] + "/ss"]
    if case["style"] == "masked":
        keep = ~inp["mask"]
        z, ss, zr, sr = np.ma.getdata(z)[keep], np.ma.getdata(ss)[keep], zr[keep], sr[keep]
    assert_parity(z, zr, 1e-5, case["name"] + " z")
    assert_parity(ss, sr, 1e-5, case["name"] + " ss")
