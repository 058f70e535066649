"""The device factorisation of new and appended problems (factor.cu: kbk_cholesky_rows / kbk_inverse_rows, the dual
kernels) against extended-precision residuals (tests/factor_reference.py), at the shapes where the blocked path
branches. Run with -m gpu on an H100.

L is read through debug tap 1, W = L^-1 through tap 2, U = C^-1 [F | z], S^-1, phi and c0 through tap 3; only the
lower and the diagonal 64x64 tiles are read (the strict upper tiles are never written). Each case checks the
componentwise backward errors beta_L, beta_WL, beta_LW (and beta_U, beta_S, beta_phi of the dual vectors) against
factor_reference.TOL, and the structure the kernels rely on: the upper triangle of every diagonal tile of L and W is
exactly zero (append_l21_kernel and trtri_step2 read across it), the padding rows [n, n_pad) are exactly zero left of
column n and the padded diagonal block is the identity (gram_lower_kernel sums over them), and diag(L) > 0.

  * fresh: n from 1 to 4095, nb = 4 ... 64 tiles and 1 ... 16 outer panels of the look-ahead Cholesky, four models
    (exponential; spherical, exact zeros past the range; gaussian with a 1e-6 nugget, ill-conditioned; linear, c0 from
    the bounding box);
  * append splits (n_old, m), each chosen for the corner nc = n_pad - n0 it factors (n0 = n_old rounded down to the
    tile): a partial last outer panel, level doubling over a corner that is not a power of two, the extra doubling
    step with the held rows on top, the re-factored partial tile row [n0, n_old), and the stride change when n_pad
    grows; the held rows [0, n0) of L and W must come back bit for bit;
  * the 11-step chain of test_append_gpu.py, checked after every step;
  * kinds: OK 2-D and OK3D with anisotropy, a geographic problem, UK with regional-linear plus 13 functional columns
    (na = 17) at sizes around the 32-column blocks and the 128-row unrolled loop of dual_u_kernel, fresh and appended;
  * determinism: the same problem on two handles gives the same bits of L, W and U (the two-stream look-ahead).

The worst value of each metric per arm is printed at the end of the module (pytest -s). Worst values over the module
on one H100 80GB HBM3 at a 700 W power limit (u = 2^-53 = 1.11e-16), against factor_reference.TOL:
  beta_L   1.35e-14 (122 u, append 192+64 gaussian; every other case <= 33 u)          TOL 5e-14
  beta_WL  6.05e-14 (545 u, fresh n = 1025 gaussian)                                 TOL 2e-13
  beta_LW  4.73e-15 (43 u, append 4000+96 exponential)                               TOL 2e-14
  beta_U   2.34e-16 (2.1 u)   beta_S 3.74e-16 (3.4 u)   beta_phi 1.31e-15 (12 u, na = 17)  TOL 1e-15, 2e-15, 5e-15
All are below n u. The left residual beta_WL is the one that grows with the conditioning (the gaussian problems with
the 1e-6 nugget set it; the other models reach 177 u), while the right residual beta_LW stays small for every model: a triangular inverse built block row by block row from W21 = -W22 (L21 W11) is residual-stable on one
side only, as LAPACK's trtri is on the other (test_factor_reference.py)."""
import numpy as np
import pytest

import cases
import factor_reference as fr

pytestmark = pytest.mark.gpu

PARAMS = {"exponential": [1.0, 300.0, 0.05], "spherical": [1.0, 400.0, 0.05], "gaussian": [1.0, 300.0, 1e-6],
          "linear": [0.004, 0.05]}
MODEL_CYCLE = ("exponential", "spherical", "gaussian", "linear")
WORST = {}


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst backward error per arm and metric (in units of u = 2^-53; tolerance in brackets):")
        for key in sorted(WORST):
            val, what = WORST[key]
            print("  %-8s %-4s %10.3e  = %6.2f u  [%.1e]  at %s" % (key[0], key[1], val, val / 2.0 ** -53,
                                                                   fr.TOL[key[1]], what))


def _u(c):
    return (c - 500.0) / 500.0


_MONO = [(a, d - a) for d in (2, 3, 4) for a in range(d + 1)]
DRIFT13 = [(lambda x, y, a=a, b=b: _u(x) ** a * _u(y) ** b) for a, b in _MONO] + [lambda x, y: np.cos(_u(x) + _u(y))]


class Held:
    """One kriging object whose float64 global factorisation lives on its handle, and the host reference of its
    problem: C and F by the device's rules in the frame of the first set-up (the anisotropy centre, the drift
    rescale and c0 stay through appends)."""

    def __init__(self, pk, kind, xyz, val, model="exponential", params=None, **kw):
        self.kind, self.mname = kind, model
        self.geo = kw.get("coordinates_type") == "geographic"
        kw = dict(variogram_model=model, variogram_parameters=PARAMS[model] if params is None else params, **kw)
        cls = {"ok": pk.OrdinaryKriging, "uk": pk.UniversalKriging, "ok3d": pk.OrdinaryKriging3D}[kind]
        self.model = cls(*[xyz[:, c] for c in range(xyz.shape[1])], val, **kw)
        self.h = self.model._ensure_problem("float64")
        x, y, z, _, self.center, self.Mt = self.model._data_arrays()
        self.n_rl, cols = self.model._drift_spec()
        self.frame = fr.DriftFrame(self._coords(), self.n_rl, cols)
        self.n0 = self.n_old = 0
        self.fetch()

    def _coords(self):
        x, y, z, _, _, _ = self.model._data_arrays()
        X = np.column_stack([x, y] + ([z] if z is not None else []))
        return X if self.geo else fr.adjusted(X, self.center, self.Mt)

    def fetch(self):
        """L, W (strict upper tiles zeroed), U [n_pad, na], S^-1, phi and c0 of the handle."""
        m = self.model
        self.n = m._data_arrays()[0].size
        self.n_pad = -(-self.n // 256) * 256
        npd, nb = self.n_pad, self.n_pad // fr.TILE
        upper = np.kron(np.triu(np.ones((nb, nb), dtype=bool), 1), np.ones((fr.TILE, fr.TILE), dtype=bool))
        self.L = self.h.debug_fetch(1, npd * npd).reshape(npd, npd)
        self.W = self.h.debug_fetch(2, npd * npd).reshape(npd, npd)
        for A in (self.L, self.W):
            A[upper] = 0.0
        K1 = self.n_rl + len(m._drift_spec()[1]) + 1
        na = K1 + 1
        t3 = self.h.debug_fetch(3, na * npd + K1 * na + 1)
        assert t3.size == na * npd + K1 * na + 1
        self.K1, self.na = K1, na
        self.U = t3[:na * npd].reshape(na, npd).T
        self.Sinv = t3[na * npd:na * npd + K1 * K1].reshape(K1, K1)
        self.phi = t3[na * npd + K1 * K1:na * npd + K1 * na]
        self.c0 = t3[-1]

    def add(self, xyz, val):
        """add_data() through the device append: the held rows [0, n0) must come back unchanged."""
        L0, W0 = self.L, self.W
        self.n_old = self.n
        self.n0 = self.n // fr.TILE * fr.TILE
        self.model.add_data(*[xyz[:, c] for c in range(xyz.shape[1])], val)
        assert self.model._kb_key is not None, "add_data fell back to a new set-up"
        assert self.model._kb_handle is self.h
        self.fetch()
        n0 = self.n0
        assert np.array_equal(np.tril(self.L[:n0, :n0]), np.tril(L0[:n0, :n0])), "held rows of L changed"
        assert np.array_equal(np.tril(self.W[:n0, :n0]), np.tril(W0[:n0, :n0])), "held rows of W changed"

    def check(self, arm, what, duals=False):
        n, npd, L, W = self.n, self.n_pad, self.L, self.W
        for name, A in (("L", L), ("W", W)):
            for t in range(0, npd, fr.TILE):
                blk = A[t:t + fr.TILE, t:t + fr.TILE]
                assert not np.any(np.triu(blk, 1)), "%s: upper triangle of the diagonal tile of %s at %d" % (what, name, t)
            assert not np.any(A[n:, :n]), "%s: padding rows of %s left of column n" % (what, name)
            assert np.array_equal(np.tril(A[n:, n:]), np.eye(npd - n)), "%s: padded diagonal block of %s" % (what, name)
        assert np.all(np.diag(L)[:n] > 0.0), what
        P = self._coords()
        C = fr.KrigingMatrix(P, self.mname, self.model._device_model()[1], self.c0, geographic=self.geo)
        extra = (self.n0 - 1, self.n0, self.n_old - 1, self.n_old, n - 1, n) if self.n_old else (n - 1, n)
        I = fr.sample_rows(npd, extra, seed=n)
        got = {"L": fr.cholesky_backward_error(C, L, I)}
        got["WL"], got["LW"] = fr.inverse_residuals(W, L, I)
        F = self.frame.matrix(P, self.model._drift_spec()[1])
        v = self.model._data_arrays()[3]
        got["U"] = fr.dual_residual(C, np.column_stack([F, v]), self.U[:n], I)
        if duals:
            got["S"] = fr.sinv_residual(self.Sinv, F, self.U[:n, :self.K1])
            got["phi"] = fr.phi_residual(self.phi, F, self.U[:n, self.K1])
        bad = []
        for k, val in got.items():
            if val > WORST.get((arm, k), (-1.0,))[0]:
                WORST[(arm, k)] = (val, what)
            if not val <= fr.TOL[k]:
                bad.append("%s: beta_%s = %.3e > %.1e" % (what, k, val, fr.TOL[k]))
        assert not bad, "\n".join(bad)


# ---- fresh problems ---------------------------------------------------------------------------------------------------
FRESH = [1, 63, 64, 65, 255, 256, 257, 511, 513, 1023, 1025, 2049, 4095]


@pytest.mark.parametrize("n", FRESH)
def test_fresh_factor(pk, n):
    """nb = 4 ... 64 tiles, 1 ... 16 outer panels of 256 columns; the models cycle with the size."""
    model = MODEL_CYCLE[FRESH.index(n) % 4]
    xyz, val = cases.synth_data(30000 + n, n, 2)
    held = Held(pk, "ok", xyz, val, model)
    held.check("fresh", "n=%d %s" % (n, model))


# ---- appended stations ------------------------------------------------------------------------------------------------
SPLITS = [(64, 1), (100, 30), (192, 64), (255, 2), (256, 1), (128, 200), (700, 600), (1000, 1), (4000, 96),
          (3000, 1100)]


@pytest.mark.parametrize("n_old,m", SPLITS, ids=["%d+%d" % s for s in SPLITS])
def test_append_split(pk, n_old, m):
    """The corner nc = n_pad - n0 of each split: (64, 1) 192 = a partial outer panel and doubling over 3 tiles;
    (100, 30) the partial tile row [64, 100) re-factored; (192, 64) nc = 64; (255, 2), (256, 1), (128, 200) and
    (3000, 1100) a new stride; (700, 600) 3 full outer panels and 1 partial; (1000, 1), (4000, 96) small appends on a
    large held factor. The models cycle; the new stations lie in the box of the held ones (c0 of the linear model
    stays valid)."""
    model = MODEL_CYCLE[SPLITS.index((n_old, m)) % 4]
    xyz, val = cases.synth_data(40000 + n_old + 7 * m, n_old + m, 2)
    held = Held(pk, "ok", xyz[:n_old], val[:n_old], model)
    ld_old = held.n_pad
    held.add(xyz[n_old:], val[n_old:])
    what = "%d+%d %s nc=%d%s" % (n_old, m, model, held.n_pad - held.n0, " restride" if held.n_pad != ld_old else "")
    held.check("append", what)


def test_chain_of_appends(pk):
    """The 11 steps of test_append_gpu.test_chain_of_ten_appends_is_exact_and_repeatable (UK, regional-linear drift):
    every metric and the held rows after each step."""
    sizes = [500, 1, 13, 64, 65, 2, 100, 37, 63, 1, 120]
    xyz, val = cases.synth_data(99, sum(sizes), 2)
    n = sizes[0]
    held = Held(pk, "uk", xyz[:n], val[:n], drift_terms=["regional_linear"])
    held.check("chain", "n=%d" % n, duals=True)
    for m in sizes[1:]:
        held.add(xyz[n:n + m], val[n:n + m])
        n += m
        held.check("chain", "n=%d (+%d)" % (n, m), duals=True)


# ---- problem kinds ----------------------------------------------------------------------------------------------------
KINDS = [("ok2d_aniso", 600, 90), ("ok3d_aniso", 450, 70), ("geo", 300, 50)]


@pytest.mark.parametrize("name,n,m", KINDS, ids=[k[0] for k in KINDS])
def test_kinds(pk, name, n, m):
    """Anisotropy in 2-D and 3-D (the adjusted frame of the first set-up is kept by the append), and great-circle
    distances; fresh and appended."""
    if name == "geo":
        xyz, val = cases.synth_data(51, n + m, 2, (60.0, 45.0, 1.0))
        xyz = xyz + np.array([-20.0, 30.0])
        held = Held(pk, "ok", xyz[:n], val[:n], params=[1.0, 20.0, 0.05], coordinates_type="geographic")
    elif name == "ok3d_aniso":
        xyz, val = cases.synth_data(52, n + m, 3)
        held = Held(pk, "ok3d", xyz[:n], val[:n], "spherical", anisotropy_scaling_y=1.5, anisotropy_scaling_z=2.0,
                    anisotropy_angle_z=25.0, anisotropy_angle_x=10.0)
    else:
        xyz, val = cases.synth_data(53, n + m, 2)
        held = Held(pk, "ok", xyz[:n], val[:n], anisotropy_scaling=1.7, anisotropy_angle=35.0)
    held.check("kinds", "%s n=%d" % (name, n), duals=True)
    held.add(xyz[n:], val[n:])
    held.check("kinds", "%s n=%d+%d" % (name, n, m), duals=True)


UK17 = [(63, 33), (95, 2), (96, 1), (97, 31), (127, 1), (128, 1), (129, 32), (159, 2), (160, 97), (161, 1000)]


@pytest.mark.parametrize("n,m", UK17, ids=["%d+%d" % s for s in UK17])
def test_uk_seventeen_columns(pk, n, m):
    """na = 17 (KB_MAXAUX): regional-linear + 13 functional columns + ones + values. n and n + m around the
    32-column blocks and the i + 96 < n bound of dual_u_kernel; U, S^-1 and phi against the reference."""
    xyz, val = cases.synth_data(60000 + n, n + m, 2)
    held = Held(pk, "uk", xyz[:n], val[:n], drift_terms=["regional_linear", "functional"], functional_drift=DRIFT13)
    assert held.na == 17
    held.check("uk17", "n=%d" % n, duals=True)
    held.add(xyz[n:], val[n:])
    held.check("uk17", "n=%d+%d" % (n, m), duals=True)


# ---- determinism ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,m", [(4095, 0), (700, 600)], ids=["fresh4095", "append700+600"])
def test_two_handles_give_the_same_bits(pk, n, m):
    """The look-ahead Cholesky runs the panel chain on a second stream, ordered by events: the same problem on two
    handles must give the same bits of L, W and U."""
    xyz, val = cases.synth_data(70000 + n, n + m, 2)
    runs = []
    for _ in range(2):
        held = Held(pk, "ok", xyz[:n], val[:n])
        if m:
            held.add(xyz[n:], val[n:])
        runs.append(held)
    a, b = runs
    assert a.h is not b.h
    for name in ("L", "W", "U"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
