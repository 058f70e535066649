"""GPU tests of leave_one_out(): every station kriged from the other N - 1 (kb200_loo, kb200_knn_loo).

The global path is compared, station by station, with brute-force reduced solves in extended precision
(tests/loo_emulator.py: brute_force_loo, fp64 LU with iterative refinement in np.longdouble) on problems of about 256 and 512
stations, which cross the 256-row chunks of the column-norm kernel, for the four classes, every drift kind, anisotropy,
geographic coordinates, a custom callable, both exact_values, coincident stations with a nugget and the Gauss-Jordan
fallback; and at full size (config 2, N = 5000) on eight stations. The moving window is compared with the oracle's
moving window on each reduced data set. The bit invariants (field v against a single-field call, sigma^2 for any V,
run to run) and the device refusals are pinned. Bounds: max|out - ref| / max|ref| <= LOO_TOL (fp64)."""
import numpy as np
import pytest

import cases
from cv_emulator import _refined_solve, brute_force_loo
from oracle import krige_oracle as ko

pytestmark = pytest.mark.gpu

LOO_TOL = 1e-8          # global path, z and sigma^2; the worst measured error is in DESIGN.md §5e
KNN_TOL = 1e-8          # moving window against the oracle's scipy solves
WORST = {}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


def _reference_inputs(obj):
    """Adjusted stations, drift columns at the stations, the oracle's model and parameters, exact, geographic."""
    x, y, z, v, center, Mt = obj._data_arrays()
    X = np.column_stack([x, y] + ([z] if z is not None else []))
    geo = getattr(obj, "coordinates_type", "euclidean") == "geographic"
    P = X if geo else (X - np.asarray(center)) @ np.asarray(Mt).reshape(X.shape[1], X.shape[1]).T + np.asarray(center)
    n_rl, hcols = obj._drift_spec()
    cols = ([P[:, c] for c in range(X.shape[1])] if n_rl else []) + [np.asarray(c, float) for c in hcols]
    fn = obj.variogram_function if obj.variogram_model == "custom" else obj.variogram_model
    return P, cols, fn, list(obj.variogram_model_parameters), bool(obj.exact_values), geo


def _judge(label, out, ref, tol):
    err = max(np.abs(out[0] - ref[0]).max() / np.abs(ref[0]).max(), np.abs(out[1] - ref[1]).max() / np.abs(ref[1]).max())
    WORST[label] = err
    print("loo %s: max rel err %.3e" % (label, err))
    assert err <= tol, (label, err)


def _stations(seed, n, dim, dups=False):
    X, val = cases.synth_data(seed, n, dim)
    if dups:                                # a coincident triple and a pair 1e-9 apart (inside eps after adjustment)
        X[7] = X[3]
        X[21] = X[3]
        X[30] = X[12]
        X[30, 0] += 1e-11
    return X, val


def _obj(pk, cls, X, val, **kw):
    cols = [X[:, c] for c in range(X.shape[1])]
    return getattr(pk, cls)(*cols, val, **kw)


EXP = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
GLOBAL = {
    "ok2d_n256": ("OrdinaryKriging", 256, 2, dict(EXP)),
    "ok2d_n512_sph_aniso_nonexact": ("OrdinaryKriging", 512, 2, dict(variogram_model="spherical",
                                     variogram_parameters=[1.5, 400.0, 0.1], anisotropy_scaling=2.0,
                                     anisotropy_angle=30.0, exact_values=False)),
    "ok2d_n257_linear": ("OrdinaryKriging", 257, 2, dict(variogram_model="linear", variogram_parameters=[0.002, 0.1])),
    "uk2d_n300_rl_spec_func": ("UniversalKriging", 300, 2, dict(EXP, drift_terms=["regional_linear", "specified",
                               "functional"], functional_drift=[lambda x, y: np.sin(x / 200.0) * y / 500.0])),
    "uk2d_n257_pointlog_extz": ("UniversalKriging", 257, 2, dict(EXP, drift_terms=["point_log", "external_Z"],
                                point_drift=np.array([[200.0, 300.0, 1.0], [700.0, 650.0, -0.5]]))),
    "ok3d_n256_gauss_aniso": ("OrdinaryKriging3D", 256, 3, dict(variogram_model="gaussian",
                              variogram_parameters=[1.0, 300.0, 0.05], anisotropy_scaling_y=1.5,
                              anisotropy_angle_z=20.0)),
    "uk3d_n300_rl": ("UniversalKriging3D", 300, 3, dict(EXP, drift_terms=["regional_linear"])),
    "geo_ok_n256": ("OrdinaryKriging", 256, "geo", dict(variogram_model="exponential",
                    variogram_parameters=[1.0, 40.0, 0.05], coordinates_type="geographic")),
    "custom_ok_n256": ("OrdinaryKriging", 256, 2, dict(variogram_model="custom", variogram_parameters=[0.5, 1.0, 0.1],
                       variogram_function=lambda m, d: m[0] * np.log10(d + m[1]) + m[2])),
    "dups_ok_n256": ("OrdinaryKriging", 256, 2, dict(EXP)),
    "dups_uk_n512": ("UniversalKriging", 512, 2, dict(EXP, drift_terms=["regional_linear"])),
    "dups_ok_n256_nonexact": ("OrdinaryKriging", 256, 2, dict(EXP, exact_values=False)),
}


def _build(pk, name):
    cls, n, dim, kw = GLOBAL[name]
    kw = dict(kw)
    if dim == "geo":
        rng = np.random.default_rng(17)
        X = np.column_stack([rng.uniform(-60, 60, n), rng.uniform(-45, 45, n)])
        val = 5 + np.sin(X[:, 0] / 20) + rng.normal(size=n) * 0.3
    else:
        X, val = _stations(31 + n, n, dim, dups=name.startswith("dups"))
    if "specified" in kw.get("drift_terms", ()):
        kw["specified_drift"] = [1e-3 * X[:, 0] * X[:, 1]]
    if "external_Z" in kw.get("drift_terms", ()):
        ex, ey = np.linspace(-10, 1010, 9), np.linspace(-10, 1010, 7)
        kw.update(external_drift=np.random.default_rng(4).uniform(0, 5, (ey.size, ex.size)), external_drift_x=ex,
                  external_drift_y=ey)
    return _obj(pk, cls, X, val, **kw), val


@pytest.mark.parametrize("name", list(GLOBAL))
def test_global_against_brute_force(pk, name):
    obj, val = _build(pk, name)
    z, ss = obj.leave_one_out()
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    ref = brute_force_loo(P, val, fn, m, exact, cols, geo=geo, refined=not geo)
    _judge(name, (z, ss), ref, LOO_TOL)


def test_gauss_jordan_path(pk):
    """Hole-effect on dense scatter: C is indefinite, the factorisation falls back to Gauss-Jordan (gform 1)."""
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 25, (300, 2))
    val = rng.normal(size=300)
    obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, variogram_model="hole-effect", variogram_parameters=[1.0, 3.0, 0.0])
    z, ss = obj.leave_one_out()
    with pytest.raises(NotImplementedError):                   # statistics refuse the indefinite fallback: gform 1
        obj._kb_handle.statistics(300)
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    _judge("gform1_hole_effect_n300", (z, ss), brute_force_loo(P, val, fn, m, exact, cols, refined=True), LOO_TOL)


def test_full_size_config2(pk):
    """Config 2 (N = 5000, exponential [1, 300, 0.05]) after a float64 execute() on the same object: eight stations
    against brute-force solves of the 4999-station problems."""
    X, val = cases.synth_data(1002, 5000, 2)
    obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **EXP)
    obj.execute("points", X[:3, 0] + 0.5, X[:3, 1])
    h = obj._kb_handle
    h.reset_counters()
    z, ss = obj.leave_one_out()
    assert h.timings()["cholesky_ms"] == 0.0                  # no new factorisation
    idx = np.array([0, 1, 255, 256, 2047, 4095, 4998, 4999])
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    zr, sr = np.zeros(idx.size), np.zeros(idx.size)
    for t, i in enumerate(idx):
        keep = np.arange(5000) != i
        a = ko.kriging_matrix(P[keep], fn, m)
        zr[t], sr[t] = _refined_solve(a, P[keep], P[i:i + 1], val[keep], fn, m, exact, ())
    _judge("cfg2_n5000_8_stations", (z[idx], ss[idx]), (zr, sr), LOO_TOL)


KNN = [("2d", 2), ("2d", 10), ("2d", 64), ("2d", 129), ("3d", 10), ("3d", 64), ("geo", 10), ("geo", 64),
       ("dups", 10), ("dups", 129)]


@pytest.mark.parametrize("kind,k", KNN, ids=["%s_k%d" % c for c in KNN])
def test_moving_window_against_oracle(pk, kind, k):
    n = 300
    if kind == "geo":
        rng = np.random.default_rng(23)
        X = np.column_stack([rng.uniform(-60, 60, n), rng.uniform(-45, 45, n)])
        val = 5 + np.sin(X[:, 0] / 20) + rng.normal(size=n) * 0.3
        obj = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, variogram_model="exponential",
                                 variogram_parameters=[1.0, 40.0, 0.05], coordinates_type="geographic")
    else:
        X, val = _stations(41, n, 3 if kind == "3d" else 2, dups=kind == "dups")
        obj = _obj(pk, "OrdinaryKriging3D" if kind == "3d" else "OrdinaryKriging", X, val, **EXP)
    z, ss = obj.leave_one_out(n_closest_points=k)
    P, cols, fn, m, exact, geo = _reference_inputs(obj)
    ref = brute_force_loo(P, val, fn, m, exact, k=k, geo=geo, index_ties=kind == "dups")
    _judge("knn_%s_k%d" % (kind, k), (z, ss), ref, KNN_TOL)


def test_bit_invariants(pk):
    """Field v is bit-identical to a single-field leave_one_out() of an object with z = values[:, v] and does not
    depend on V or its position; sigma^2 is the same bits for every V; a repeat gives the same bits."""
    X, val = _stations(5, 700, 2, dups=True)
    F = 40.0 + 10.0 * np.random.default_rng(8).standard_normal((700, 64))
    for kw in ({}, dict(n_closest_points=20)):
        uk = not kw
        mk = (lambda z: pk.UniversalKriging(X[:, 0], X[:, 1], z, drift_terms=["regional_linear"], **EXP)) if uk \
            else (lambda z: pk.OrdinaryKriging(X[:, 0], X[:, 1], z, **EXP))
        obj = mk(val)
        z64, s64 = obj.leave_one_out(values=F, **kw)
        z3, s3 = obj.leave_one_out(values=F[:, [5, 0, 63]], **kw)
        z1, s1 = obj.leave_one_out(values=F[:, 63], **kw)
        np.testing.assert_array_equal(z3, z64[[5, 0, 63]])
        np.testing.assert_array_equal(z1, z64[63])
        for s in (s3, s1):
            np.testing.assert_array_equal(s, s64)
        for v in (0, 63):
            zs, ss = mk(F[:, v]).leave_one_out(**kw)
            np.testing.assert_array_equal(zs, z64[v])
            np.testing.assert_array_equal(ss, s64)
        z64b, s64b = obj.leave_one_out(values=F, **kw)
        np.testing.assert_array_equal(z64b, z64)
        np.testing.assert_array_equal(s64b, s64)


def test_refusals_on_the_device(pk):
    from pykrige_b200 import _cabi
    X, val = _stations(9, 60, 2)
    with pytest.raises(NotImplementedError):
        pk.OrdinaryKriging(X[:, 0], X[:, 1], val, pseudo_inv=True, **EXP).leave_one_out()
    ok = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **EXP)
    for k in (1, 60):
        with pytest.raises(ValueError):
            ok.leave_one_out(n_closest_points=k)
    T = np.array([[0.0, 0.0], [10.0, 1.0], [3.0, 9.0]])
    uk3 = pk.UniversalKriging(T[:, 0], T[:, 1], np.array([1.0, 2.0, 0.5]), variogram_model="exponential",
                              variogram_parameters=[1.0, 20.0, 0.1], drift_terms=["regional_linear"])
    with pytest.raises(np.linalg.LinAlgError, match="station 0"):
        uk3.leave_one_out()
    # a problem received through kb200_blob_commit has no factor on the handle: the C ABI refuses it
    h = _cabi.Handle()
    args = (2, 0, X[:, 0], X[:, 1], None, val, [500.0, 500.0], np.eye(2), 3, [0.95, 300.0, 0.05], True, 1e-10)
    h.set_problem(*args)
    z, ss = h.loo(60)
    assert z.shape == (60,) and np.all(ss > 0)
    h.describe_problem(*args)
    h.blob_commit()                                     # the blob still holds the factored problem
    with pytest.raises(_cabi.KrigeB200Error, match="blob_commit"):
        h.loo(60)
    h.close()
