"""The residual metrics of factor_reference.py on host factorisations: a clean factor from LAPACK passes every metric at
the tolerances of test_factor_gpu.py, each seeded defect of the kind a blocked Cholesky / triangular inverse kernel
could have is flagged by at least 10^3 times the tolerance (on a full and on a sampled matrix), and the metrics do not
grow with the condition number of C."""
import numpy as np
import pytest
import scipy.linalg as sl
import scipy.linalg.lapack as lapack

import cases
import factor_reference as fr

T = fr.TILE
MARGIN = 1e3


def _factor(n, model="exponential", params=(1.0, 300.0, 0.05), n_pad=None, seed=3):
    """(C as a KrigingMatrix, C dense, L, W, coordinates, values) of n stations, padded to n_pad with the identity.
    W from LAPACK's blocked triangular inverse."""
    n_pad = n_pad or -(-n // T) * T
    xyz, val = cases.synth_data(seed, n, 2)
    Cm = fr.KrigingMatrix(xyz, model, list(params), params[0] + params[2])          # c0 = the sill
    C = Cm.block(np.arange(n_pad), np.arange(n_pad))
    L = sl.cholesky(C, lower=True)
    W, info = lapack.dtrtri(L, lower=1)
    assert info == 0
    return Cm, C, L, W, xyz, val


def _betas(C, L, W, I):
    b = {"L": fr.cholesky_backward_error(C, L, I)}
    b["WL"], b["LW"] = fr.inverse_residuals(W, L, I)
    return b


@pytest.fixture(scope="module", params=[(300, None), (1100, 1152)], ids=["full", "sampled"])
def clean(request):
    n, n_pad = request.param
    Cm, C, L, W, xyz, val = _factor(n, n_pad=n_pad)
    I = fr.sample_rows(L.shape[0], (n - 1, n), seed=1)
    assert (I.size == L.shape[0]) == (request.param[0] == 300)
    return dict(n=n, Cm=Cm, C=C, L=L, W=W, xyz=xyz, val=val, I=I)


def test_clean_factor_passes(clean):
    b = _betas(clean["Cm"], clean["L"], clean["W"], clean["I"])
    for k, v in b.items():
        assert v <= fr.TOL[k], (k, v)


def test_clean_dual_vectors_pass():
    """U = C^-1 [F | z] from LAPACK, S^-1 and phi for a regional-linear + 3 host columns drift."""
    n = 400
    Cm, C, L, W, xyz, val = _factor(n, n_pad=n)
    cols = [np.sin(xyz[:, 0] / 100.0), xyz[:, 1] ** 2, np.cos(xyz[:, 0] / 300.0) * 5.0 + 2.0]
    frame = fr.DriftFrame(xyz[:300], 2, [c[:300] for c in cols])      # an appended problem keeps the first frame
    F = frame.matrix(xyz, cols)
    Fz = np.column_stack([F, val])
    U = sl.cho_solve((L, True), Fz)
    K1 = F.shape[1]
    Sinv = np.linalg.inv(F.T @ U[:, :K1])
    phi = F.T @ U[:, K1]
    I = np.arange(n)
    assert fr.dual_residual(Cm, Fz, U, I) <= fr.TOL["U"]
    assert fr.sinv_residual(Sinv, F, U[:, :K1]) <= fr.TOL["S"]
    assert fr.phi_residual(phi, F, U[:, K1]) <= fr.TOL["phi"]
    # a wrong drift column, a stale S^-1 entry or a phi from the wrong column is flagged
    U2 = U.copy(); U2[:, 1] *= 1.0 + 1e-6
    assert fr.dual_residual(Cm, Fz, U2, I) >= MARGIN * fr.TOL["U"]
    S2 = Sinv.copy(); S2[0, 1] *= 1.0 + 1e-6
    assert fr.sinv_residual(S2, F, U[:, :K1]) >= MARGIN * fr.TOL["S"]
    assert fr.phi_residual(F.T @ U[:, 0], F, U[:, K1]) >= MARGIN * fr.TOL["phi"]


def _tile(A, i, j):
    return A[i * T:(i + 1) * T, j * T:(j + 1) * T]


def _missing_update(C, L, W):
    """L tile (4, 3) computed without the rank-64 update of chunk 1"""
    L = L.copy()
    _tile(L, 4, 3)[:] += _tile(L, 4, 1) @ _tile(L, 3, 1).T @ _tile(W, 3, 3).T
    return L, W


def _row_off(C, L, W):
    """L21 tile (3, 2) one row off: each row holds the one below"""
    L = L.copy()
    _tile(L, 3, 2)[:] = L[3 * T + 1:4 * T + 1, 2 * T:3 * T]
    return L, W


def _stale(C, L, W):
    """L21 tile (4, 1) still holding C: its value before the Schur update and the triangular solve"""
    L = L.copy()
    _tile(L, 4, 1)[:] = _tile(C, 4, 1)
    return L, W


def _short_k(C, L, W):
    """W21 tile (4, 1) whose k sum stops one 64-chunk early: W_41 = -W_44 sum_{K=1}^{2} L_4K W_K1, K = 3 dropped"""
    W = W.copy()
    _tile(W, 4, 1)[:] += _tile(W, 4, 4) @ _tile(L, 4, 3) @ _tile(W, 3, 1)
    return L, W


def _sign(C, L, W):
    """W21 tile (3, 0) with the wrong sign"""
    W = W.copy()
    _tile(W, 3, 0)[:] *= -1.0
    return L, W


def _upper(C, L, W, row):
    """one tiny non-zero above the diagonal of a W diagonal tile: an interior row, the last column of the tile"""
    W = W.copy()
    W[row, (row // T + 1) * T - 1] = 1e-12 * W[row, row]
    return L, W


def _fragment(C, L, W, row):
    """one element of a 16x16 fragment of L in an interior row holding its neighbour's value (a swapped column pair)"""
    L = L.copy()
    j = 2 * T + 16 + 6
    L[row, j], L[row, j + 1] = L[row, j + 1], L[row, j]
    return L, W


DEFECTS = [_missing_update, _row_off, _stale, _short_k, _sign, _upper, _fragment]


@pytest.mark.parametrize("defect", DEFECTS, ids=[d.__name__.strip("_") for d in DEFECTS])
def test_seeded_defects_are_flagged(clean, defect):
    C, L, W, I = clean["C"], clean["L"], clean["W"], clean["I"]
    if defect in (_upper, _fragment):
        tile = 2 if defect is _upper else 4
        row = next(i for i in I if i // T == tile and i % T not in (0, T - 1))     # a sampled interior row of the tile
        L2, W2 = defect(C, L, W, row)
    else:
        L2, W2 = defect(C, L, W)
    b = _betas(clean["Cm"], L2, W2, I)
    worst = max(b[k] / fr.TOL[k] for k in b)
    assert worst >= MARGIN, b


def test_metrics_do_not_depend_on_the_condition_number():
    """A well-conditioned problem and a gaussian one with a tiny nugget (kappa about 3e10) give beta_L and beta_WL of
    the same order (a few u), where an elementwise comparison of L or W with another factorisation would differ by a
    factor kappa. (Of the two residuals of a triangular inverse, a blocked method that builds W from W = L^-1 block rows
    bounds only one independently of kappa (Du Croz and Higham, 1992): beta_LW of LAPACK's trtri grows with kappa.)"""
    out = {}
    for name, model, params in (("well", "exponential", (1.0, 300.0, 0.3)), ("ill", "gaussian", (1.0, 300.0, 1e-9))):
        Cm, C, L, W, xyz, val = _factor(320, model, params)
        kappa = np.linalg.cond(C)
        I = np.arange(L.shape[0])
        out[name] = (kappa, _betas(Cm, L, W, I))
    (k_w, b_w), (k_i, b_i) = out["well"], out["ill"]
    assert k_w < 1e3 and k_i > 1e10, (k_w, k_i)
    for k in ("L", "WL"):
        assert b_i[k] <= fr.TOL[k] and b_w[k] <= fr.TOL[k]
        assert b_i[k] <= 30.0 * max(b_w[k], 2.0 ** -53) and b_w[k] <= 30.0 * max(b_i[k], 2.0 ** -53), (k, b_w, b_i)


def test_device_distance_rules_match_the_oracle():
    """The adjusted coordinates and great-circle distances of the reference C agree with the oracle's to rounding."""
    from oracle import krige_oracle as ko
    from pykrige_b200 import core
    xyz, _ = cases.synth_data(5, 200, 3)
    Mt = core.anisotropy_matrix(3, [1.5, 2.0], [10.0, 0.0, 25.0])
    center = (xyz.max(axis=0) + xyz.min(axis=0)) / 2.0
    P = fr.adjusted(xyz, center, Mt)
    assert np.allclose(P, ko.adjust_for_anisotropy(xyz, center, [1.5, 2.0], [10.0, 0.0, 25.0]), rtol=0, atol=1e-10)
    ll = cases.synth_data(6, 200, 2, (60.0, 45.0, 1.0))[0] + np.array([-20.0, 30.0])
    d = fr.great_circle_degrees(fr.unit_vectors(ll), fr.unit_vectors(ll))
    dr = ko.great_circle_distance(ll[:, 0][:, None], ll[:, 1][:, None], ll[:, 0][None, :], ll[:, 1][None, :])
    assert np.abs(d - dr).max() <= 1e-12 and np.all(np.diag(d) == 0.0)
