"""GPU boundary sweep of the moving-window kernel (csrc/knn.cu, execute(n_closest_points=k)) against an exact neighbour
search and an extended-precision local solve (tests/knn_reference.py).

The kernel grows a block of cells until k candidates lie inside the distance to the nearest unvisited face, compacts its
candidate buffer past 480 entries, selects the k nearest through a 256-bucket histogram with an exact (d^2, index)
ranking of the boundary bucket (a full sort when that bucket holds more than 32), and solves the local system by a tiled
Cholesky on the fp64 tensor pipe (k <= 128: identity padding to a multiple of 8, augmented rows [c ; 1 ; Z_0 ..]) or by
LU (k > 128, and every k after a block that is not positive definite). Each arm here puts one of those on an edge: k
on both sides of every tile boundary up to the shared-memory ceiling of 156, the number of points around a multiple of
the points per CTA, value-field counts that step the augmented tile rows, lattices and coincident stations (exact ties,
crowded boundary buckets), near-duplicates at the pivot floor, a dense cluster, degenerate cell grids, large
coordinate offsets, anisotropy, queries on cell faces and far outside the data, geographic data over the poles and the
date line, the shifted models, and leave-one-out / leave-group-out.

A weight probe observes the kernel directly: with one-hot value fields E[:, c] = e_j, z of field c is the weight the
kernel gave station j, and exactly 0.0 when j is not among its neighbours (a non-neighbour's value never enters the
augmented rows). So every probed point is checked for
- support: the weight of every probed station outside the expected neighbour set is exactly 0.0 (with cross-validation
  also that of the held-out station and its group); this has no tolerance;
- weights: max |lambda - lambda_ref| within the tolerance of the solver path;
- outputs: sum lambda = 1, and z and sigma^2 of the single-field call against the refined reference.

Tolerances, one per solver path, as max |out - ref| / max |ref| (z, sigma^2) and max |lambda - lambda_ref| (weights),
set within a few times the worst error over this file on one H100 80GB HBM3 at a 700 W power limit: Cholesky 2.0e-14
(collinear data, z, kappa 5e2), LU 5.4e-14 (hole-effect weights at k = 140, kappa 2e4), shifted models 5.5e-13 (power
weights at k = 140, where the reference's own local system has kappa = 1e7). The near-duplicate and gaussian arms are
held to 0.5 kappa eps where that is larger; near-duplicates 1e-7 of the extent apart reach 8.2e-10 at kappa = 2e8
(0.02 kappa eps) and 1.9e-10 at kappa = 9e6 (0.1 kappa eps).
Worst errors and kappa_2 of the local system per arm are printed at the end of the module (pytest -s)."""
import numpy as np
import pytest

import cases
import knn_reference as kr
from oracle import krige_oracle as ko

pytestmark = pytest.mark.gpu

TOL = {"chol": 1e-13, "lu": 2e-13, "shift": 2e-12}
ILL_C = 0.5                     # ill-conditioned arms: kappa_2 * eps * ILL_C when that is larger than the path's tolerance
EPS64 = float(np.finfo(np.float64).eps)

K_SWEEP = [2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 155, 156]
EXP = [1.0, 300.0, 0.05]
SHIFTED = ("linear", "power", "custom")

WORST = {}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst error against the refined reference per arm (z, sigma^2: / max|ref|; weights: absolute):")
        for arm in sorted(WORST):
            err, what, kappa = WORST[arm]
            print("  %-34s %.3e  at %s  (kappa %.2e)" % (arm, err, what, kappa))


def path_of(k, model):
    """The tolerance class of a run: the shifted covariance form of the unbounded models (either solver), else the
    solver the kernel runs: LU above k = 128 and for the hole-effect model (not positive definite), else Cholesky."""
    if model in SHIFTED:
        return "shift"
    return "lu" if k > kr.CHOL_K_MAX or model == "hole-effect" else "chol"


def _linear_fn(m, d):
    return m[0] * d + m[1]


class Window:
    """One moving-window problem: the pykrige_b200 model and the reference frame of its data."""

    def __init__(self, pk, data, values, model="exponential", params=EXP, aniso=None, exact=True, geo=False):
        data = np.asarray(data, dtype=np.float64)
        self.dim, self.n, self.geo, self.exact = data.shape[1], data.shape[0], geo, exact
        self.values = np.asarray(values, dtype=np.float64)
        self.mname = model
        kw = dict(variogram_model=model, variogram_parameters=list(params), exact_values=exact)
        if model == "custom":
            kw["variogram_function"] = _linear_fn
            self.fn, self.m = _linear_fn, list(params)
        else:
            self.fn, self.m = model, ko.stored_parameters(model, params)
        scaling, angle = [1.0] * (self.dim - 1), [0.0] * (2 * self.dim - 3)
        if aniso is not None:
            scaling, angle = aniso
            if self.dim == 2:
                kw.update(anisotropy_scaling=scaling[0], anisotropy_angle=angle[0])
            else:
                kw.update(anisotropy_scaling_y=scaling[0], anisotropy_scaling_z=scaling[1], anisotropy_angle_x=angle[0],
                          anisotropy_angle_y=angle[1], anisotropy_angle_z=angle[2])
        if geo:
            kw["coordinates_type"] = "geographic"
        cls = pk.OrdinaryKriging3D if self.dim == 3 else pk.OrdinaryKriging
        self.model = cls(*[data[:, c] for c in range(self.dim)], self.values, **kw)
        from pykrige_b200.core import anisotropy_matrix
        self.center = (data.max(axis=0) + data.min(axis=0)) / 2.0
        self.M = anisotropy_matrix(self.dim, scaling, angle)
        self.raw = data
        self.P = data if geo else kr.device_frame(data, self.center, self.M)
        self.S = kr.search_coords(self.P, geo)

    def frame(self, Q):
        return np.asarray(Q, dtype=np.float64) if self.geo else kr.device_frame(Q, self.center, self.M)

    def execute(self, k, Q, values=None):
        Q = np.asarray(Q, dtype=np.float64)
        z, ss = self.model.execute("points", *[Q[:, c] for c in range(self.dim)], backend="cuda",
                                   n_closest_points=k, values=values)
        return np.asarray(z), np.asarray(ss)

    def probe(self, k, Q, stations):
        """W[c, p]: the weight the kernel gave station stations[c] at point p. The one-hot fields go in chunks of
        _cabi.MAX_FIELDS, the chunks execute() would cut anyway, so no N x len(stations) matrix is ever built."""
        from pykrige_b200 import _cabi
        out = []
        for c0 in range(0, len(stations), _cabi.MAX_FIELDS):
            chunk = np.asarray(stations[c0:c0 + _cabi.MAX_FIELDS])
            E = np.zeros((self.n, chunk.size))
            E[chunk, np.arange(chunk.size)] = 1.0
            out.append(np.atleast_2d(self.execute(k, Q, E)[0]))
        return np.concatenate(out)

    def cross_validate(self, k, groups=None, values=None):
        if groups is None:
            z, ss = self.model.leave_one_out(n_closest_points=k, values=values)
        else:
            z, ss = self.model.leave_group_out(groups, n_closest_points=k, values=values)
        return np.asarray(z), np.asarray(ss)

    def probe_stations(self, k, Q, limit=400):
        """Every station when there are few, else the union of each point's 2k brute-force nearest."""
        if self.n <= limit:
            return np.arange(self.n)
        SQ = kr.search_coords(self.frame(Q), self.geo)
        out = []
        for i in range(SQ.shape[0]):
            d2 = np.sum((self.S - SQ[i]) ** 2, axis=1)
            out.append(np.argsort(d2, kind="stable")[:min(self.n, 2 * k + 8)])
        return np.unique(np.concatenate(out))


class Judge:
    """Collects the errors of one arm against the reference; failures are reported after the whole arm ran."""

    def __init__(self, label, tol, ill=False):
        self.label, self.tol, self.ill = label, tol, ill
        self.failures = []
        self.z, self.zr, self.ss, self.ssr, self.kappa = [], [], [], [], []

    def _tol(self, kappa):
        return max(self.tol, ILL_C * kappa * EPS64) if self.ill else self.tol

    def point(self, win, k, q_adj, s_q, i, what, z=None, ss=None, W=None, stations=None, exclude=None, fields=None,
              zf=None):
        """Point i (adjusted q_adj, search coordinates s_q) of a call: z / ss its outputs, W[:, i] the probed weights of
        `stations`, zf[:, i] the outputs of value fields `fields` [N, V]."""
        nb = kr.neighbours(win.S, s_q, k, exclude=exclude)
        sel = nb.sel
        if nb.flagged and W is None:
            # a near-tie at the k-th distance that rounding may order either way, and no probe to show which of the
            # acceptable sets the kernel took: nothing to judge this point against
            return float("nan")
        if W is not None:
            w = W[:, i]
            allowed = nb.allowed() if nb.flagged else nb.sel
            outside = ~np.isin(stations, allowed)
            bad = outside & (w != 0.0)
            if exclude is not None:
                held = np.isin(stations, exclude)
                bad |= held & (w != 0.0)
            if bad.any():
                self.failures.append("%s %s point %d: nonzero weight on non-neighbours %s (expected %s)"
                                     % (self.label, what, i, stations[bad][:8].tolist(), sel[:8].tolist()))
            if nb.flagged:
                cand = np.union1d(nb.must, stations[np.isin(stations, nb.band) & (w != 0.0)])
                if nb.accepts(cand):
                    sel = cand
        lam, zr, ssr, kappa = kr.local_solution(win.P[sel], q_adj, win.values[sel], win.fn, win.m, win.exact, win.geo)
        tol = self._tol(kappa)
        if W is not None:
            pos = {s: c for c, s in enumerate(stations)}
            have = np.array([s in pos for s in sel])
            wdev = np.array([W[pos[s], i] for s in sel[have]])
            if wdev.size:
                e = float(np.max(np.abs(wdev - lam[have])))
                self._worst("weights", e, "%s point %d" % (what, i), kappa)
                if e > tol:
                    self.failures.append("%s %s point %d: max|lambda - ref| = %.3e > %.1e (kappa %.2e)"
                                         % (self.label, what, i, e, tol, kappa))
            if have.all():
                e = abs(float(np.sum(wdev)) - 1.0)
                if e > max(tol, 1e-12):
                    self.failures.append("%s %s point %d: sum lambda - 1 = %.3e" % (self.label, what, i, e))
        if z is not None:
            self.z.append(z[i]); self.zr.append(zr); self.ss.append(ss[i]); self.ssr.append(ssr)
            self.kappa.append(kappa)
        if fields is not None:
            zfr = fields[sel].T @ lam.astype(np.longdouble)
            e = float(np.max(np.abs(zf[:, i] - zfr.astype(np.float64))) / max(1.0, np.max(np.abs(fields))))
            self._worst("fields", e, "%s point %d" % (what, i), kappa)
            if e > tol:
                self.failures.append("%s %s point %d: value fields off by %.3e > %.1e" % (self.label, what, i, e, tol))
        return kappa

    def _worst(self, kind, err, what, kappa):
        key = "%s %s" % (self.label, kind)
        if not np.isfinite(err):
            err = float("inf")
        if err > WORST.get(key, (-1.0,))[0]:
            WORST[key] = (err, what, kappa)

    def finish(self, what=""):
        if self.z:
            kap = np.asarray(self.kappa)
            for name, o, r in (("z", self.z, self.zr), ("ss", self.ss, self.ssr)):
                o, r = np.asarray(o), np.asarray(r)
                d = np.abs(o - r) / max(float(np.max(np.abs(r))), 1e-300)
                j = int(np.argmax(np.where(np.isfinite(d), d, np.inf)))
                err = float(d[j]) if np.isfinite(d[j]) else float("inf")
                self._worst(name, err, "%s point %d" % (what, j), float(kap[j]))
                lim = np.array([self._tol(c) for c in kap])
                if not np.all(d <= lim):
                    bad = np.flatnonzero(~(d <= lim))
                    self.failures.append("%s %s %s: %d points off, worst %.3e at point %d (kappa %.2e)"
                                         % (self.label, what, name, bad.size, err, j, kap[j]))
        assert not self.failures, "\n".join(self.failures[:20])


def check_call(judge, win, k, Q, what, probe=True, fields=None):
    """execute(n_closest_points=k) at the raw points Q: the single-field outputs, the probe unless probe=False, and the
    value fields [N, V] when given."""
    Q = np.asarray(Q, dtype=np.float64)
    z, ss = win.execute(k, Q)
    W = stations = zf = None
    if probe:
        stations = win.probe_stations(k, Q)
        W = win.probe(k, Q, stations)
    if fields is not None:
        zf = np.atleast_2d(win.execute(k, Q, fields)[0])
    Qa = win.frame(Q)
    SQ = kr.search_coords(Qa, win.geo)
    for i in range(Q.shape[0]):
        judge.point(win, k, Qa[i], SQ[i], i, what, z, ss, W, stations, None, fields, zf)


# ---- geometry of the cell grid (kb200_set_problem_knn) and the query placements -------------------------------------
def cell_grid(P):
    """(origin, cell, cells per axis) of the device's uniform cell grid over the adjusted points P."""
    lo, hi = P.min(axis=0), P.max(axis=0)
    ext = hi - lo
    live = int(np.sum(ext > 0.0))
    vol = float(np.prod(ext[ext > 0.0])) if live else 1.0
    cell = (vol * 2.0 / P.shape[0]) ** (1.0 / live) if live else 1.0
    while True:
        g = np.minimum(np.floor(ext / cell) + 1.0, 4096.0).astype(np.int64)
        if np.prod(g) <= (1 << 22):
            break
        cell *= 1.5
    for r in range(P.shape[1]):
        if g[r] == 4096:
            cell = max(cell, ext[r] / 4095.0)
    return lo, cell, g


def placements(win, rng, n_inside=10):
    """Raw query points: inside the data, on cell faces, just outside the box, and 10x the extent away beyond every
    side and corner (all faces in 3-D). Anisotropy is undone for the face points, so they sit on faces up to rounding."""
    raw = win.raw
    lo, hi = raw.min(axis=0), raw.max(axis=0)
    ext = np.where(hi > lo, hi - lo, 1.0)
    mid = (lo + hi) / 2.0
    out = [lo + rng.uniform(0.0, 1.0, (n_inside, win.dim)) * (hi - lo)]
    olo, cell, g = cell_grid(win.P)
    Minv = np.linalg.inv(win.M)
    for r in range(win.dim):                          # on interior cell faces of each axis
        if g[r] < 3:
            continue
        a = win.P[rng.choice(win.n, 2)].copy()
        a[:, r] = olo[r] + cell * rng.integers(1, g[r], 2)
        out.append(win.center + (a - win.center) @ Minv.T)
    for r in range(win.dim):                          # just outside
        for s in (-1.0, 1.0):
            p = mid.copy()
            p[r] = (lo[r] - 1e-3 * ext[r]) if s < 0 else (hi[r] + 1e-3 * ext[r])
            out.append(p[None, :])
    far = []                                          # 10x the extent away: sides and corners
    for sgn in np.ndindex(*([3] * win.dim)):
        o = np.asarray(sgn, dtype=np.float64) - 1.0
        if np.any(o != 0.0):
            far.append(mid + 10.0 * o * ext)
    out.append(np.asarray(far))
    return np.vstack(out)


def uniform(seed, n, dim=2, box=(1000.0, 1000.0, 250.0)):
    return cases.synth_data(seed, n, dim, box)


def lattice(n_side, dim=2):
    g = np.arange(float(n_side))
    X = np.stack(np.meshgrid(*([g] * dim), indexing="ij")[::-1], axis=-1).reshape(-1, dim)
    rng = np.random.default_rng(n_side)
    return X, 50.0 + 10.0 * np.sin(X[:, 0] / 3.0) + np.cos(X[:, 1] / 2.0) + rng.normal(0.0, 0.5, X.shape[0])


def lattice_queries(n_side, rng, m=8):
    """Lattice nodes, cell centres and edge midpoints (exact ties at many distances)."""
    nodes = rng.integers(0, n_side, (m, 2)).astype(np.float64)
    cells = rng.integers(0, n_side - 1, (m, 2)) + 0.5
    edges = np.column_stack([rng.integers(0, n_side - 1, m) + 0.5, rng.integers(0, n_side, m)])
    return np.vstack([nodes, cells, edges, [[0.0, 0.0], [n_side - 1.0, n_side - 1.0], [-3.0, 2.0]]])


# ---- k: every tile boundary of the Cholesky, the LU switch and the shared-memory ceiling ----------------------------
@pytest.mark.parametrize("k", K_SWEEP)
def test_k_sweep(pk, k):
    """Uniform scatter, N = 300 (all stations probed), queries inside, on cell faces, just outside and far outside."""
    xyz, val = uniform(1000 + k, 300)
    win = Window(pk, xyz, val)
    Q = placements(win, np.random.default_rng(k))
    j = Judge("k-sweep %s" % path_of(k, "exponential"), TOL[path_of(k, "exponential")])
    check_call(j, win, k, Q, "k=%d" % k)
    j.finish("k=%d" % k)


def test_k_equals_n(pk):
    """k = N: the search visits the whole grid and stops there; every station is a neighbour."""
    xyz, val = uniform(77, 40)
    win = Window(pk, xyz, val)
    Q = placements(win, np.random.default_rng(1), n_inside=4)
    j = Judge("k=N chol", TOL["chol"])
    check_call(j, win, 40, Q, "k=N=40")
    j.finish("k=N")


def test_k_limits_are_refused(pk):
    """k = 157 exceeds the shared memory of the local solver (NotImplementedError, the C ABI's KB200_EUNSUPPORTED);
    k = 1 and k = N + 1 are refused as arguments (ValueError)."""
    from pykrige_b200 import _cabi
    assert kr.k_supported(156) and not kr.k_supported(157)
    xyz, val = uniform(3, 200)
    win = Window(pk, xyz, val)
    q = xyz[:2] + 1.0
    with pytest.raises(NotImplementedError, match="n_closest_points too large"):
        win.execute(157, q)
    with pytest.raises(ValueError):
        win.execute(1, q)
    small = Window(pk, xyz[:20], val[:20])
    with pytest.raises(ValueError):
        small.execute(21, q)
    assert _cabi.KB200_EUNSUPPORTED == -2


# ---- launch shape: points per CTA ----------------------------------------------------------------------------------
SHAPE_K = [8, 64, 128, 129, 156]


@pytest.mark.parametrize("k", SHAPE_K)
def test_launch_shape(pk, k):
    """M = 1 and M = wpc c - 1, wpc c, wpc c + 1 (wpc points per CTA for this k, c = 3), as explicit points, as a grid
    and as a masked grid: the last CTA is partial, full, or holds one point."""
    chol = k <= kr.CHOL_K_MAX
    wpc = kr.points_per_cta(k, chol, 0, 1)
    xyz, val = uniform(2000 + k, 500)
    win = Window(pk, xyz, val)
    j = Judge("launch %s" % path_of(k, "exponential"), TOL[path_of(k, "exponential")])
    rng = np.random.default_rng(k)
    for M in (1, 3 * wpc - 1, 3 * wpc, 3 * wpc + 1):
        Q = rng.uniform(-50.0, 1050.0, (M, 2))
        check_call(j, win, k, Q, "points M=%d" % M, probe=M <= 4)
        gx, gy = np.sort(rng.uniform(0.0, 1000.0, M)), np.array([rng.uniform(0.0, 1000.0)])
        z, ss = win.model.execute("grid", gx, gy, backend="cuda", n_closest_points=k)
        Qg = np.column_stack([gx, np.full(M, gy[0])])
        Qa = win.frame(Qg)
        for i in range(M):
            j.point(win, k, Qa[i], Qa[i], i, "grid M=%d" % M, np.ravel(z), np.ravel(ss))
    gx, gy = np.linspace(0.0, 1000.0, wpc + 1), np.linspace(0.0, 1000.0, 3)
    mask = np.zeros((3, wpc + 1), bool)
    mask[1, ::2] = True
    z, ss = win.model.execute("masked", gx, gy, mask=mask, backend="cuda", n_closest_points=k)
    GX, GY = np.meshgrid(gx, gy)
    keep = ~mask.ravel()
    Qa = win.frame(np.column_stack([GX.ravel(), GY.ravel()])[keep])
    zk, sk = np.ma.getdata(z).ravel()[keep], np.ma.getdata(ss).ravel()[keep]
    assert np.array_equal(np.ma.getmaskarray(z).ravel(), mask.ravel())
    for i in range(Qa.shape[0]):
        j.point(win, k, Qa[i], Qa[i], i, "masked", zk, sk)
    j.finish("k=%d wpc=%d" % (k, wpc))


def test_staged_chunks(pk):
    """2^21 + 5 points: the outputs come back through three staged chunks of 2^20; points on both sides of each chunk
    boundary against the reference."""
    xyz, val = uniform(5, 300)
    win = Window(pk, xyz, val)
    M = (1 << 21) + 5
    rng = np.random.default_rng(9)
    Q = rng.uniform(0.0, 1000.0, (M, 2))
    z, ss = win.execute(8, Q)
    idx = np.unique(np.concatenate([[0, (1 << 20) - 1, 1 << 20, (1 << 21) - 1, 1 << 21, M - 1],
                                    rng.choice(M, 40, replace=False)]))
    Qa = win.frame(Q[idx])
    j = Judge("staged chol", TOL["chol"])
    for t, i in enumerate(idx):
        j.point(win, 8, Qa[t], Qa[t], t, "M=%d" % M, z[idx], ss[idx])
    j.finish("staged")


# ---- value fields: the augmented tile rows [c ; 1 ; Z_0 .. Z_{V-1}] --------------------------------------------------
V_SWEEP = [1, 5, 6, 7, 14, 15, 64]


@pytest.mark.parametrize("k", [8, 64, 128])
def test_value_rows(pk, k):
    """V fields step the augmented tile rows at V = 7, 15, ...; field v against lambda_ref . Z_v for every V."""
    xyz, val = uniform(3000 + k, 300)
    win = Window(pk, xyz, val)
    rng = np.random.default_rng(k)
    Q = rng.uniform(0.0, 1000.0, (12, 2))
    j = Judge("fields chol", TOL["chol"])
    for V in V_SWEEP:
        F = rng.normal(0.0, 1.0, (300, V)) * np.linspace(1.0, 100.0, V)[None, :]
        check_call(j, win, k, Q, "k=%d V=%d" % (k, V), probe=False, fields=F)
    j.finish("k=%d" % k)


def test_value_rows_lu_path(pk):
    """The hole-effect model is not positive definite on dense scatter: at k = 64 and 128 every local block of these
    points fails the Cholesky, which flags it, and the launch is repeated on the LU path, with V fields. The solve-launch
    count of each fields call shows it: 2 (Cholesky, then LU). At k = 8 the same model's blocks are positive definite
    (smallest eigenvalue 0.05 c0), the Cholesky result stands and the call makes 1 launch."""
    xyz, val = uniform(31, 300)
    win = Window(pk, xyz, val, "hole-effect", [1.0, 200.0, 0.0])
    rng = np.random.default_rng(2)
    Q = rng.uniform(0.0, 1000.0, (12, 2))
    for k, launches in ((8, 1), (64, 2), (128, 2)):
        p = "lu" if launches == 2 else "chol"
        j = Judge("fields hole-effect %s" % p, TOL[p])
        for V in (7, 15):
            F = rng.normal(0.0, 1.0, (300, V))
            check_call(j, win, k, Q, "k=%d V=%d" % (k, V), probe=(V == 7))
            win.model._kb_handle.reset_counters()
            zf = np.atleast_2d(win.execute(k, Q, F)[0])
            got = int(win.model._kb_handle.timings()["solve_launches"])
            assert got == launches, "hole-effect k=%d V=%d: %d solve launches, expected %d" % (k, V, got, launches)
            Qa = win.frame(Q)
            for i in range(Q.shape[0]):
                j.point(win, k, Qa[i], Qa[i], i, "k=%d V=%d fields" % (k, V), fields=F, zf=zf)
        j.finish("hole-effect k=%d" % k)


# ---- data layouts -------------------------------------------------------------------------------------------------
def _cluster(seed, n):
    rng = np.random.default_rng(seed)
    nc = int(0.9 * n)
    xyz = np.vstack([rng.uniform(450.0, 550.0, (nc, 2)), rng.uniform(0.0, 1000.0, (n - nc, 2))])
    return xyz, 50.0 + 10.0 * np.sin(xyz[:, 0] / 15.0) * np.cos(xyz[:, 1] / 20.0) + rng.normal(0.0, 0.3, n)


def _near_dups(seed):
    xyz, val = uniform(seed, 200)
    for q in range(4):
        xyz[199 - q] = xyz[q] + 1e-4 * np.array([1.0, 0.7])   # 1e-7 of the 1000 extent
    return xyz, val


def _coincident(seed):
    xyz, val = uniform(seed, 200)
    xyz[198] = xyz[197] = xyz[10]                              # a triple
    xyz[199] = xyz[20]                                         # a pair
    return xyz, val


def _offset(seed):
    rng = np.random.default_rng(seed)
    g = np.arange(18.0)
    X = np.column_stack([np.tile(g, 18), np.repeat(g, 18)]) + rng.uniform(-0.3, 0.3, (324, 2))
    X += np.array([5e5, 5e6])
    return X, 10.0 * np.sin(X[:, 0] - 5e5) + rng.normal(0.0, 0.5, 324)


LAYOUTS = {
    # name: (data builder, model, params, extra Window kwargs, ks, query builder)
    "lattice": (lambda: lattice(19), "exponential", [1.0, 6.0, 0.05], {}, [3, 7, 8, 16, 31, 64, 129],
                lambda w, rng: lattice_queries(19, rng)),
    "coincident_nugget": (lambda: _coincident(41), "exponential", [1.0, 300.0, 0.1], {}, [8, 64],
                          lambda w, rng: np.vstack([w.raw[[10, 20, 30]], placements(w, rng, 6)])),
    "coincident_nonexact": (lambda: _coincident(42), "exponential", [1.0, 300.0, 0.1], dict(exact=False), [8, 64],
                            lambda w, rng: np.vstack([w.raw[[10, 20, 30]], placements(w, rng, 6)])),
    "collinear": (lambda: (np.column_stack([np.random.default_rng(4).uniform(0, 1000, 300), np.full(300, 7.0)]),
                           np.random.default_rng(5).normal(0, 1, 300)), "exponential", EXP, {}, [8, 64, 156],
                  lambda w, rng: placements(w, rng)),
    "offset": (lambda: _offset(8), "exponential", [1.0, 6.0, 0.05], {}, [16, 64],
               lambda w, rng: placements(w, rng)),
    "aniso2d": (lambda: uniform(9, 300), "exponential", EXP, dict(aniso=([5.0], [35.0])), [8, 65, 129],
                lambda w, rng: placements(w, rng)),
    "uniform3d": (lambda: uniform(10, 350, 3), "spherical", [1.0, 400.0, 0.05], {}, [8, 64, 156],
                  lambda w, rng: placements(w, rng, 6)),
    "aniso3d": (lambda: uniform(11, 350, 3), "exponential", EXP, dict(aniso=([2.0, 0.5], [20.0, 35.0, 50.0])),
                [9, 64], lambda w, rng: placements(w, rng, 6)),
    "coplanar3d": (lambda: (np.column_stack([uniform(12, 300)[0], np.full(300, 3.0)]), uniform(12, 300)[1]),
                   "exponential", EXP, {}, [8, 64], lambda w, rng: placements(w, rng, 6)),
    "geographic": (lambda: (np.column_stack([np.random.default_rng(13).uniform(-180, 180, 350),
                                             np.degrees(np.arcsin(np.random.default_rng(14).uniform(-1, 1, 350)))]),
                            np.random.default_rng(15).normal(0, 1, 350)),
                   "exponential", [1.0, 40.0, 0.02], dict(geo=True), [8, 64, 129],
                   lambda w, rng: np.array([[179.999, 5.0], [-179.999, -5.0], [180.0, 0.0], [0.0, 89.99],
                                            [120.0, -89.99], [-45.0, 90.0], [10.0, -90.0], [33.0, 12.0]])),
}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_layout(pk, name):
    build, model, params, extra, ks, queries = LAYOUTS[name]
    xyz, val = build()
    win = Window(pk, xyz, val, model, params, **extra)
    rng = np.random.default_rng(len(name))
    Q = queries(win, rng)
    for k in ks:
        j = Judge("%s %s" % (name, path_of(k, model)), TOL[path_of(k, model)])
        check_call(j, win, k, Q, "k=%d" % k)
        j.finish("k=%d" % k)


def test_dense_cluster(pk):
    """90 % of N = 20000 stations in 1 % of the area: at k = 64 and 156 the candidate buffer is compacted again and
    again while the block grows. Probed on the 2k nearest of 12 points in, at the edge of and outside the cluster."""
    xyz, val = _cluster(17, 20000)
    win = Window(pk, xyz, val, "exponential", [1.0, 30.0, 0.02])
    Q = np.array([[500.0, 500.0], [450.0, 450.0], [550.0, 500.0], [449.9, 520.0], [560.0, 560.0], [300.0, 500.0],
                  [0.0, 0.0], [1000.0, 1000.0], [-5000.0, 500.0], [510.0, 5000.0], [523.4, 467.8], [700.0, 200.0]])
    for k in (64, 156):
        j = Judge("cluster %s" % path_of(k, "exponential"), TOL[path_of(k, "exponential")])
        check_call(j, win, k, Q, "k=%d" % k)
        j.finish("k=%d" % k)


def test_near_duplicates(pk):
    """Stations 1e-7 of the extent apart, nugget 0: the local systems are nearly singular. The result is the refined
    answer (to kappa * eps) or ValueError('Singular matrix'), never a silently wrong number."""
    xyz, val = _near_dups(43)
    for model, params in (("exponential", [1.0, 300.0, 0.0]), ("spherical", [1.0, 300.0, 0.0])):
        win = Window(pk, xyz, val, model, params)
        Q = np.vstack([xyz[:4] + 0.5, xyz[:4], placements(win, np.random.default_rng(3), 4)])
        for k in (8, 129):
            j = Judge("near-dup %s" % path_of(k, model), TOL[path_of(k, model)], ill=True)
            for i in range(Q.shape[0]):             # one point per call: a singular point does not hide the others
                try:
                    check_call(j, win, k, Q[i:i + 1], "%s k=%d Q[%d]" % (model, k, i))
                except ValueError as e:
                    assert str(e) == "Singular matrix"
            j.finish("%s k=%d" % (model, k))


def test_exact_duplicates_without_nugget(pk):
    """Coincident stations with nugget 0 make the local system exactly singular. The Cholesky pivot of such a block is
    rounding noise of either sign; the pivot floor (16 eps c0) sends every one of them to LU, which finds the exact zero
    pivot: ValueError('Singular matrix') as the reference's solver raises, at a Cholesky k and at an LU k. The same
    stations away from the duplicates krige normally."""
    xyz, val = uniform(44, 300)
    for q in range(12):
        xyz[299 - q] = xyz[q]
    win = Window(pk, xyz, val, "exponential", [1.0, 300.0, 0.0])
    silent = []
    for k in (8, 33, 129):
        for q in range(12):
            try:
                z, ss = win.execute(k, xyz[q:q + 1] + 0.25)
            except ValueError as e:
                assert str(e) == "Singular matrix"
                continue
            silent.append("k=%d duplicate pair %d: z=%r sigma^2=%r" % (k, q, float(z[0]), float(ss[0])))
    assert not silent, "exactly singular local systems returned numbers:\n" + "\n".join(silent)
    dups = np.r_[0:12, 288:300]
    far = np.array([p for p in cases.synth_points(44, 40, 2, xyz, n_hits=0)
                    if not np.isin(kr.neighbours(xyz, p, 8).sel, dups).any()][:6])
    assert far.shape[0] == 6
    j = Judge("exact-dup chol", TOL["chol"])
    check_call(j, win, 8, far, "away from the duplicates")
    j.finish("exact-dup")


# ---- variogram models ----------------------------------------------------------------------------------------------
MODELS = [
    ("exponential", [1.0, 300.0, 0.05], {}),
    ("spherical", [1.0, 3.0, 0.0], dict(lattice=True)),        # lattice distances exactly at the range
    ("gaussian", [1.0, 300.0, 0.01], dict(ill=True)),
    ("linear", [0.004, 0.05], {}),
    ("power", [0.02, 1.5, 0.05], {}),
    ("hole-effect", [1.0, 200.0, 0.0], {}),
    ("custom", [0.004, 0.05], {}),
    ("exponential", [1.0, 300.0, 0.2], dict(exact=False)),
]


@pytest.mark.parametrize("model,params,opt", MODELS,
                         ids=["%s%s" % (m[0], "_nonexact" if m[2].get("exact") is False else "") for m in MODELS])
def test_models(pk, model, params, opt):
    """Every model at a Cholesky k (8, 33), the last Cholesky k (128) and an LU k (140), with exact hits."""
    if opt.get("lattice"):
        xyz, val = lattice(17)
        Q = lattice_queries(17, np.random.default_rng(0))
    else:
        xyz, val = uniform(50, 300)
        Q = np.vstack([xyz[:4], cases.synth_points(50, 10, 2, xyz, n_hits=0)])
    win = Window(pk, xyz, val, model, params, exact=opt.get("exact", True))
    for k in (8, 33, 128, 140):
        p = path_of(k, model)
        j = Judge("model %s %s" % (model, p), TOL[p], ill=opt.get("ill", False))
        check_call(j, win, k, Q, "%s k=%d" % (model, k))
        j.finish("%s k=%d" % (model, k))


# ---- cross-validation: the held-out station and its group never enter ---------------------------------------------
CV = [("lattice", None), ("lattice", "blocks"), ("coincident", None), ("coincident", "blocks"), ("aniso", None),
      ("aniso", "blocks")]


@pytest.mark.parametrize("layout,groups", CV, ids=["%s_%s" % (a, b or "loo") for a, b in CV])
def test_cross_validation(pk, layout, groups):
    """leave_one_out / leave_group_out(n_closest_points=k) with probes: the held-out station (and its group) has weight
    exactly 0.0, the rest of the support is the nearest k outside the group, the weights and outputs are the
    reference's. Leave-one-out drops a station only where its d^2 to the query is exactly 0.0, which needs the data
    and the query through the same adjust arithmetic: the anisotropy case checks that under a rotation."""
    if layout == "lattice":
        xyz, val = lattice(15)
        win = Window(pk, xyz, val, "exponential", [1.0, 5.0, 0.05])
    elif layout == "coincident":
        xyz, val = _coincident(60)
        win = Window(pk, xyz, val, "exponential", [1.0, 300.0, 0.1])
    else:
        xyz, val = uniform(61, 220)
        win = Window(pk, xyz, val, "exponential", EXP, aniso=([5.0], [35.0]))
    n = win.n
    if groups == "blocks":
        lo, hi = xyz.min(axis=0), xyz.max(axis=0)
        b = np.floor((xyz - lo) / (hi - lo + 1e-9) * 4.0).astype(int)
        lab = b[:, 0] * 4 + b[:, 1]
        if layout == "coincident":
            lab[[197, 198]] = lab[10]
            lab[199] = lab[20]
    else:
        lab = None
    sizes = np.bincount(lab) if lab is not None else np.ones(n, int)
    for k in (7, 64, 129):
        if k > n - sizes.max():
            continue
        p = path_of(k, "exponential")
        j = Judge("cv %s %s" % (layout, p), TOL[p])
        z, ss = win.cross_validate(k, lab)
        stations = np.arange(n)
        W = np.atleast_2d(win.cross_validate(k, lab, values=np.eye(n))[0])
        for i in range(n):
            excl = np.flatnonzero(lab == lab[i]) if lab is not None else np.array([i])
            j.point(win, k, win.P[i], win.S[i], i, "%s k=%d" % (groups or "loo", k), z, ss, W, stations, excl)
        j.finish("%s k=%d" % (groups or "loo", k))


# ---- full size: BASELINE config 5 ---------------------------------------------------------------------------------
def test_full_size_cfg5(pk):
    """N = 1e5, k = 64, exponential [1, 50, 0.05]: z and sigma^2 of 256 points (corners, edges, outside the hull,
    exact hits, scatter) against the refined reference, and the probe at 16 of them."""
    xyz, val = cases.synth_data(1005, 100000, 2)
    win = Window(pk, xyz, val, "exponential", [1.0, 50.0, 0.05])
    rng = np.random.default_rng(56)
    edge = np.array([[0.0, 0.0], [1000.0, 0.0], [0.0, 1000.0], [1000.0, 1000.0], [-20.0, 500.0], [500.0, 1020.0],
                     [-3000.0, -3000.0], [5000.0, 400.0], [500.0, 0.0], [1000.0, 500.0]])
    Q = np.vstack([edge, xyz[:6], rng.uniform(0.0, 1000.0, (240, 2))])
    j = Judge("cfg5 chol", TOL["chol"])
    z, ss = win.execute(64, Q)
    Qa = win.frame(Q)
    for i in range(Q.shape[0]):
        j.point(win, 64, Qa[i], Qa[i], i, "cfg5", z, ss)
    sub = np.r_[0:10, 10:12, 100:104]
    stations = win.probe_stations(64, Q[sub])
    W = win.probe(64, Q[sub], stations)
    zs, ss_s = win.execute(64, Q[sub])
    for t, i in enumerate(sub):
        j.point(win, 64, Qa[i], Qa[i], t, "cfg5 probe", zs, ss_s, W, stations)
    j.finish("cfg5")
