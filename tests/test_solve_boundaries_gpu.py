"""GPU boundary sweep of the global solve kernels against the extended-precision reference
(oracle.krige_oracle.exec_vector_refined: the exact solution of the reference's own fp64 gamma-form system).

The fp64 kernel (solve.cu) works on 16-row m-tiles and 16-wide k tiles inside 256-row blocks; of the wgmma kernels
(solve_wgmma.cu), float32 splits each 256-row block 128/128 over two warpgroups and the float64x ones use row
blocks of 48 / 64 / 64 rows with k = 32, and the Cholesky panels are 64 and 256 wide. The K + 2 dense dual rows sit
right after row n. The data sizes below put n and n + na on both sides of each of those boundaries, for ordinary
kriging (na = 2), universal kriging with a regional-linear drift (na = 4) and with the full 15 drift columns the C ABI
allows (na = 17), and every result is compared with the refined reference at a tolerance per arithmetic that is close
to what the kernel actually achieves: a mis-indexed fragment, a wrong k-tile bound or a lost dual row in one row block
shows up here even when it stays inside the 1e-5 of the reference-parity tests.

The fp64 kernel runs with 16-, 32- and 64-point tiles (KB200_TILE forces one width per call); a second test runs
enough points that every CTA processes several tiles, which is where shared-memory sums and the scratch ring are
re-used. The general paths (indefinite variogram: Gauss-Jordan inverse + quadratic form; pseudo_inv=True) read the
scratch ring back in their own epilogue and are swept at the same sizes.

Worst errors and condition numbers per arm are printed at the end of the module (pytest -s)."""
import numpy as np
import pytest

import cases
from conftest import assert_parity
from oracle import krige_oracle as ko

pytestmark = pytest.mark.gpu

# assert_parity tolerance R (rtol = R, atol = R * max|ref|) of each arithmetic, for z and for sigma^2. Set within a few
# times the worst error over this file on one H100 80GB HBM3 at a 400 W power limit (max|out - ref| / max|ref|):
# fp64 3.8e-11, float64x 3.5e-9, float64x5 2.7e-7, float64x4 2.8e-5, float32 3.3e-4 (a single point, where that is
# twice the R it needs), gform 1 1.2e-12, gform 2 4.5e-11. The fp64 worst is n = 64, na = 17 with the linear model,
# where the reference's own matrix has kappa = 3e9 (kappa * eps = 3e-7) and all three tile widths give the same bits.
TOL = {"float64": 1e-10, "float64x": 1e-8, "float64x5": 1e-6, "float64x4": 1e-4, "float32": 5e-4}
TOL_GJ = 5e-12          # gform = 1: Gauss-Jordan inverse of the indefinite matrix
TOL_PINV = 2e-10        # gform = 2: Jacobi-SVD pseudo-inverse vs scipy.linalg.pinv (both fp64)

ARMS = [("float64", 16), ("float64", 32), ("float64", 64), ("float32", None), ("float64x", None),
        ("float64x5", None), ("float64x4", None)]
FP64_ARMS = ARMS[:3]

NS = [1, 3, 15, 16, 17, 47, 48, 49, 63, 64, 65, 127, 128, 129, 143, 144, 239, 240, 241, 254, 255, 256, 257,
      383, 384, 511, 512, 513, 767]
MODELS = {"exponential": [1.0, 300.0, 0.05], "spherical": [1.0, 400.0, 0.05], "linear": [0.004, 0.05]}
_MODEL_CYCLE = ("exponential", "spherical", "linear")
ANISO_NS = (17, 129, 257, 513)                  # these sizes also carry a geometric anisotropy
NONEXACT = (241, 2)                             # and this problem exact_values=False


def _u(c):
    return (c - 500.0) / 500.0


# 13 smooth functional drift terms: the monomials of degree 2..4 in the centred, scaled adjusted coordinates, and one
# more; with the two regional-linear columns the 15 drift columns of KB200_MAX_DRIFT (na = 17)
_MONO = [(a, d - a) for d in (2, 3, 4) for a in range(d + 1)]
DRIFT13 = [(lambda x, y, a=a, b=b: _u(x) ** a * _u(y) ** b) for a, b in _MONO] + [lambda x, y: np.cos(_u(x) + _u(y))]
assert len(DRIFT13) == 13


def _sweep():
    out = []
    for i, n in enumerate(NS):
        for na in (2, 4, 17):
            if (na == 4 and n < 15) or (na == 17 and n < 63):
                continue
            out.append((n, na, "2d", _MODEL_CYCLE[(i + na) % 3]))
    out.append((255, 2, "3d", "spherical"))
    out.append((255, 2, "geo", "exponential"))
    return out


SWEEP = _sweep()
for _need in ((254, 2), (239, 17), (255, 2), (240, 17), (256, 17)):     # dual rows filling / crossing a block
    assert any(s[:2] == _need and s[2] == "2d" for s in SWEEP)

WORST = {}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst max|out - ref| / max|ref| against the refined reference, per arm (and the least passing R):")
        for arm in sorted(WORST):
            err, what, kappa, rmin = WORST[arm]
            print("  %-18s %.3e  at %s  (kappa %.2e)  R %.3e" % (arm, err, what, kappa, rmin))


class Problem:
    """One kriging problem: the pykrige_b200 model, its prediction points and the refined reference outputs."""

    def __init__(self, pk, n, na, kind="2d", model="exponential", m_scatter=100, params=None, exact=None, dups=0,
                 pseudo_inv=False, seed=None):
        self.n, self.na, self.kind = n, na, kind
        seed = 10000 + 10 * n + na if seed is None else seed
        dim = 3 if kind == "3d" else 2
        params = list(MODELS[model] if params is None else params)
        exact = ((n, na) != NONEXACT) if exact is None else exact
        aniso = kind == "2d" and n in ANISO_NS
        box = (60.0, 45.0, 1.0) if kind == "geo" else (1000.0, 1000.0, 250.0)
        xyz, val = cases.synth_data(seed, n, dim, box)
        for q in range(dups):                           # redundant data points: same place, different value
            xyz[n - 1 - 2 * q] = xyz[3 * q]
        pts = cases.synth_points(seed, m_scatter, dim, xyz, box)
        if kind == "geo":
            shift = np.array([-20.0, 30.0])
            xyz, pts = xyz + shift, pts + shift
        self.data, self.values, self.pts = xyz, val, pts
        kw = dict(variogram_model=model, variogram_parameters=params, exact_values=exact)
        if pseudo_inv:
            kw["pseudo_inv"] = True
        scaling, angle = [1.0] * (dim - 1), [0.0] * (2 * dim - 3)
        if aniso:
            kw.update(anisotropy_scaling=1.6, anisotropy_angle=35.0)
            scaling, angle = [1.6], [35.0]
        if kind == "geo":
            kw["coordinates_type"] = "geographic"
        if na > 2:
            kw["drift_terms"] = ["regional_linear"] + (["functional"] if na == 17 else [])
            if na == 17:
                kw["functional_drift"] = DRIFT13
            assert na in (4, 17)
        cls = {("2d", 2): pk.OrdinaryKriging, ("geo", 2): pk.OrdinaryKriging, ("3d", 2): pk.OrdinaryKriging3D,
               ("2d", 4): pk.UniversalKriging, ("2d", 17): pk.UniversalKriging}[(kind, na)]
        self.model = cls(*[xyz[:, c] for c in range(dim)], val, **kw)
        self.what = "n=%d na=%d %s %s%s%s" % (n, na, kind, model, " aniso" if aniso else "", "" if exact else " nonexact")

        m = ko.stored_parameters(model, params)
        self.mname, self.m, self.exact = model, m, exact
        if kind == "geo":
            gc = lambda A, B: ko.great_circle_distance(A[:, 0][:, None], A[:, 1][:, None], B[:, 0][None, :],
                                                       B[:, 1][None, :])
            self.P, self.Q = xyz, pts
            a = np.zeros((n + 1, n + 1))
            a[:n, :n] = -ko.variogram(model, m, gc(xyz, xyz))
            np.fill_diagonal(a, 0.0)
            a[n, :n] = a[:n, n] = 1.0
            self.a, self._bd, self._dcols = a, gc, None
            return
        center = (xyz.max(axis=0) + xyz.min(axis=0)) / 2.0
        self.center, self.scaling, self.angle = center, scaling, angle
        self.P = ko.adjust_for_anisotropy(xyz, center, scaling, angle)
        self.Q = ko.adjust_for_anisotropy(pts, center, scaling, angle)
        self._bd = None
        self._dcols = lambda X: ([X[:, 0], X[:, 1]] if na > 2 else []) + ([f(X[:, 0], X[:, 1]) for f in DRIFT13]
                                                                          if na == 17 else [])
        self.a = ko.kriging_matrix(self.P, model, m, self._dcols(self.P))

    def reference(self, idx=None, pseudo_inv=None):
        """(z, sigma^2, kappa) of the prediction points pts[idx] (all when idx is None)."""
        Q = self.Q if idx is None else self.Q[idx]
        if pseudo_inv:
            z, ss = ko.exec_vector(self.a, self.P, Q, self.values, self.mname, self.m, self.exact,
                                   self._dcols(Q) if self._dcols else (), pseudo_inv=pseudo_inv)
            return z, ss, float("nan")
        bd = self._bd(Q, self.P) if self._bd else None
        return ko.exec_vector_refined(self.a, self.P, Q, self.values, self.mname, self.m, self.exact,
                                      self._dcols(Q) if self._dcols else (), bd=bd)

    def run(self, dtype, idx=None):
        p = self.pts if idx is None else self.pts[idx]
        z, ss = self.model.execute("points", *[p[:, c] for c in range(p.shape[1])], backend="cuda", dtype=dtype)
        return np.asarray(z), np.asarray(ss)


def _set_tile(monkeypatch, tile):
    if tile:
        monkeypatch.setenv("KB200_TILE", str(tile))
    else:
        monkeypatch.delenv("KB200_TILE", raising=False)


def _judge(label, tol, what, kappa, out, ref, failures):
    """Record the worst relative error of this arm, and the failure if it is outside tol."""
    for o, r, q in ((out[0], ref[0], "z"), (out[1], ref[1], "ss")):
        d, scale = np.abs(o - r), np.max(np.abs(r))
        err = float(np.max(d) / scale)
        rmin = float(np.max(d / (scale + np.abs(r))))     # the least R for which assert_parity passes
        if not np.isfinite(err):
            err = rmin = float("inf")
        if err > WORST.get(label, (-1.0,))[0]:
            WORST[label] = (err, "%s %s" % (what, q), kappa, rmin)
        try:
            assert_parity(o, r, tol, "%s %s %s (kappa %.2e)" % (label, what, q, kappa))
        except AssertionError as e:
            failures.append(str(e))


def _arm_label(dtype, tile):
    return "%s/t%d" % (dtype, tile) if tile else dtype


def _sweep_arms(monkeypatch, prob, arms, tol, ref, idx=None, label_prefix="", pseudo=False):
    """Every arm against the same reference; all arms run before the failures are reported."""
    failures = []
    kappa = ref[2]
    for dtype, tile in arms:
        _set_tile(monkeypatch, tile)
        label = label_prefix + _arm_label(dtype, tile)
        t = tol[dtype] if isinstance(tol, dict) else tol
        z, ss = prob.run(dtype)
        if idx is not None:
            z, ss = z[idx], ss[idx]
        _judge(label, t, prob.what, kappa, (z, ss), ref[:2], failures)
        if idx is None:
            z1, s1 = prob.run(dtype, idx=[0])          # M = 1
            _judge(label, t, prob.what + " M=1", kappa, (z1, s1), (ref[0][:1], ref[1][:1]), failures)
    _set_tile(monkeypatch, None)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("n,na,kind,model", SWEEP, ids=["n%d_na%d_%s" % s[:3] for s in SWEEP])
def test_solve_boundary_sweep(pk, monkeypatch, n, na, kind, model):
    """n and n + na on both sides of every tile / block / panel boundary, M = 100 scattered points + up to 16 exact
    hits (never a multiple of a tile width) and M = 1, every arithmetic, against the refined reference."""
    prob = Problem(pk, n, na, kind, model)
    ref = prob.reference()
    _sweep_arms(monkeypatch, prob, ARMS, TOL, ref)


MULTI = [(129, 4), (240, 17), (255, 2), (256, 17)]


@pytest.mark.parametrize("n,na", MULTI, ids=["n%d_na%d" % s for s in MULTI])
def test_later_tiles_of_each_cta(pk, monkeypatch, n, na):
    """At least two tiles per CTA at every tile width (M >= 2 x SMs x 64): the second and later tiles of a persistent
    CTA re-use its shared-memory sums, its dual-row staging and its scratch ring. A subsample of 512 points that
    includes the last tile of the call is compared with the refined reference."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 2 * sms * 64 + 37
    prob = Problem(pk, n, na, "2d", _MODEL_CYCLE[n % 3], m_scatter=M - 16, seed=20000 + n)
    assert prob.pts.shape[0] == M
    rng = np.random.default_rng(n)
    idx = np.union1d(rng.choice(M - 64, 448, replace=False), np.arange(M - 64, M))
    ref = prob.reference(idx)
    _sweep_arms(monkeypatch, prob, ARMS, TOL, ref, idx=idx, label_prefix="multi ")


GJ = [(127, 2), (128, 4), (255, 2), (256, 4), (257, 2), (383, 4)]


@pytest.mark.parametrize("n,na", GJ, ids=["n%d_na%d" % s for s in GJ])
def test_general_inverse_path_at_boundaries(pk, monkeypatch, n, na):
    """gform = 1: hole-effect on dense scatter is not a valid covariance in 2-D, so the Cholesky of the covariance form
    fails and the Gauss-Jordan inverse + quadratic-form read-back runs instead (that it ran is seen from float32, which
    has no such fallback and refuses the same problem). All three tile widths against the refined reference."""
    prob = Problem(pk, n, na, "2d", "hole-effect", params=[1.0, 300.0, 0.02])
    ref = prob.reference()
    _sweep_arms(monkeypatch, prob, FP64_ARMS, TOL_GJ, ref, label_prefix="gform1 ")
    with pytest.raises(NotImplementedError):
        prob.run("float32", idx=[0])


PINV = [(127, 2), (255, 2), (256, 4), (257, 2)]


@pytest.mark.parametrize("n,na", PINV, ids=["n%d_na%d" % s for s in PINV])
def test_pseudo_inverse_path_at_boundaries(pk, monkeypatch, n, na):
    """gform = 2: pseudo_inv=True with three redundant data points and no nugget (an exactly singular matrix). The
    reference is scipy.linalg.pinv of the same matrix (exec_vector); all three tile widths."""
    prob = Problem(pk, n, na, "2d", "exponential", params=[1.0, 300.0, 0.0], dups=3, pseudo_inv=True)
    ref = prob.reference(pseudo_inv="pinv")
    _sweep_arms(monkeypatch, prob, FP64_ARMS, TOL_PINV, ref, label_prefix="gform2 ")


def test_sixteen_drift_columns_are_refused(pk):
    """KB200_MAX_DRIFT = 15 drift columns (regional-linear + host supplied). One more is an error from backend='cuda',
    not numbers; 15 are accepted (the na = 17 problems of the sweep)."""
    xyz, val = cases.synth_data(31, 200, 2)
    kw = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05], drift_terms=["regional_linear",
                                                                                                  "functional"])
    extra = [lambda x, y: np.sin(_u(x) * 2.0)]
    uk = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, functional_drift=DRIFT13 + extra, **kw)
    pts = cases.synth_points(31, 10, 2, xyz)
    for dtype in ("float64", "float32", "float64x"):
        with pytest.raises(ValueError, match="drift"):
            uk.execute("points", pts[:, 0], pts[:, 1], backend="cuda", dtype=dtype)
    ok15 = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, functional_drift=DRIFT13, **kw)
    z, ss = ok15.execute("points", pts[:, 0], pts[:, 1], backend="cuda")
    assert np.all(np.isfinite(z)) and np.all(np.isfinite(ss))
