"""CPU model of the algebra the CUDA global path runs (DESIGN.md §3), in numpy — a white-box pin of the formulation,
not of the kernels: covariance form C = c0 11^T - Gamma with the covariance shift c0 chosen as csrc/api.cu does
(sill for bounded models, gamma(bounding-box diagonal) doubled until the Cholesky succeeds for linear / power),
Cholesky C = L L^T, W = L^-1, dual vectors U = C^-1 F, zeta = C^-1 Z on affinely rescaled drift columns (shift / scale
as api.cu: describe), and per prediction point

    q = ||W c||^2,  g = U^T c,  zc = zeta . c,  r = g - f,  mu = S^-1 r,  sigma^2 = c0 - q + r . mu,  z = zc - mu . phi.

Checked against the outputs of the unmodified imported reference (inverse x RHS on the gamma-form matrix) for the
randomised draws of tests/cases.py fuzz_config (tests/golden/ref_fuzz.npz): the two formulations must agree far inside
the 1e-5 parity tolerance, for every class, drift kind and anisotropy — if they did not for some draw, the device could
not either."""
import os
import warnings

import numpy as np
import pytest
import scipy.linalg

import cases
from conftest import GOLDEN
from oracle import krige_oracle as ko


def covariance_form_krige(P, values, model, m, Q, dcols, pcols, exact_values=True):
    """P [n, dim], Q [npt, dim] ADJUSTED coordinates; dcols / pcols: drift columns at the data / prediction points
    (without the unbiasedness column). Returns (z, sigma^2, attempts of the c0 search)."""
    n = P.shape[0]
    d = ko.cdist(P, P)
    gam = ko.variogram(model, m, d)
    np.fill_diagonal(gam, 0.0)                                  # ok.py:644: the nugget never sits on the diagonal
    if model in ("linear", "power"):
        lo, hi = P.min(axis=0), P.max(axis=0)
        c0 = float(ko.variogram(model, m, np.sqrt(np.sum((hi - lo) ** 2))))
        tries = 5
    else:
        c0, tries = float(m[0]) + float(m[2]), 1                # psill + nugget
    L = None
    for attempt in range(tries):
        try:
            L = np.linalg.cholesky(c0 - gam)
            break
        except np.linalg.LinAlgError:
            c0 *= 2.0
    if L is None:
        pytest.skip("covariance form not positive definite: the device takes the general path (DESIGN.md 3b)")
    # drift basis: columns shifted / scaled, then the constant (api.cu: describe; the span is unchanged)
    F = np.ones((n, len(dcols) + 1))
    Fq = np.ones((Q.shape[0], len(dcols) + 1))
    for c, (dc, pc) in enumerate(zip(dcols, pcols)):
        shift = 0.5 * (dc.max() + dc.min())
        half = 0.5 * (dc.max() - dc.min())
        scale = 1.0 / half if half > 0 else 1.0
        F[:, c] = (dc - shift) * scale
        Fq[:, c] = (pc - shift) * scale
    W = scipy.linalg.solve_triangular(L, np.eye(n), lower=True)
    U = W.T @ (W @ F)
    zeta = W.T @ (W @ values)
    S = F.T @ U
    phi = F.T @ zeta
    bd = ko.cdist(Q, P)
    b = -ko.variogram(model, m, bd)
    if exact_values:
        b[np.abs(bd) <= ko.EPS] = 0.0
    C = c0 + b                                                  # c_j = c0 1 + b_j[:n]
    q = np.sum((C @ W.T) ** 2, axis=1)
    r = C @ U - Fq
    mu = np.linalg.solve(S, r.T).T
    return C @ zeta - mu @ phi, c0 - q + np.sum(r * mu, axis=1), attempt + 1


def _adjusted(c, X):
    kw = c["kw"]
    dim = X.shape[1]
    data = np.column_stack(c["data"][:dim])
    center = (data.max(axis=0) + data.min(axis=0)) / 2.0
    if dim == 2:
        return ko.adjust_for_anisotropy(X, center, [kw.get("anisotropy_scaling", 1.0)], [kw.get("anisotropy_angle", 0.0)])
    return ko.adjust_for_anisotropy(X, center, [kw.get("anisotropy_scaling_y", 1.0), kw.get("anisotropy_scaling_z", 1.0)],
                                    [kw.get("anisotropy_angle_x", 0.0), kw.get("anisotropy_angle_y", 0.0),
                                     kw.get("anisotropy_angle_z", 0.0)])


@pytest.fixture(scope="module")
def ref_fuzz():
    return np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))


GLOBAL_DRAWS = [t for t in range(cases.N_FUZZ) if (cases.fuzz_config(t) or {}).get("knn", 1) is None]


@pytest.mark.parametrize("t", GLOBAL_DRAWS)
def test_covariance_form_reproduces_the_reference(t, ref_fuzz):
    c = cases.fuzz_config(t)
    kw, dim = c["kw"], len(c["data"]) - 1
    data = np.column_stack(c["data"][:dim])
    values = np.asarray(c["data"][dim], dtype=float)
    pts = [np.asarray(p, dtype=float) for p in c["pts"]]
    Qo = np.column_stack(pts) if c["style"] == "points" else ko.grid_points(pts)
    P, Q = _adjusted(c, data), _adjusted(c, Qo)
    terms = kw.get("drift_terms", [])
    dcols, pcols = [], []
    if "regional_linear" in terms:
        dcols += [P[:, k] for k in range(dim)]
        pcols += [Q[:, k] for k in range(dim)]
    if "point_log" in terms:                                    # wells live in the adjusted frame (uk.py:458-467)
        wells = np.asarray(kw["point_drift"], dtype=float)
        wa = _adjusted(c, wells[:, :2])
        for (wx, wy), s in zip(wa, wells[:, 2]):
            for X, out in ((P, dcols), (Q, pcols)):
                with np.errstate(divide="ignore"):
                    ld = np.log(np.sqrt((X[:, 0] - wx) ** 2 + (X[:, 1] - wy) ** 2))
                ld[np.isinf(ld)] = -100.0
                out.append(-s * ld)
    if "external_Z" in terms:                                   # sampled at the ORIGINAL coordinates
        from abi_emulator import _bilinear
        ax, ay, Zg = kw["external_drift_x"], kw["external_drift_y"], kw["external_drift"]
        dcols.append(_bilinear(ax, ay, Zg, data[:, 0], data[:, 1]))
        pcols.append(_bilinear(ax, ay, Zg, Qo[:, 0], Qo[:, 1]))
    if "specified" in terms:
        dcols.append(1e-3 * data[:, 0] * data[:, 1])
        pcols.append(1e-3 * Qo[:, 0] * Qo[:, 1])
    if "functional" in terms:                                   # callables see the adjusted coordinates (uk.py:906-910)
        f = kw["functional_drift"][0]
        dcols.append(np.asarray(f(*[P[:, k] for k in range(dim)]), dtype=float))
        pcols.append(np.asarray(f(*[Q[:, k] for k in range(dim)]), dtype=float))
    model = kw["variogram_model"]
    m = ko.stored_parameters(model, kw["variogram_parameters"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        z, ss, attempts = covariance_form_krige(P, values, model, m, Q, dcols, pcols, kw.get("exact_values", True))
    zr, sr = np.ravel(ref_fuzz["%d/z" % t]), np.ravel(ref_fuzz["%d/ss" % t])
    keep = np.ones(zr.size, bool)
    if c["style"] == "masked":
        keep = ~np.ravel(ref_fuzz["%d/mask" % t])
    if not keep.any():
        return
    tol = 1e-8       # three orders inside the parity tolerance; the draws have cond(A) <= 1.3e5
    np.testing.assert_allclose(z[keep], zr[keep], rtol=tol, atol=tol * np.abs(zr[keep]).max(), err_msg=c["text"])
    np.testing.assert_allclose(ss[keep], sr[keep], rtol=tol, atol=tol * max(np.abs(sr[keep]).max(), 1e-300), err_msg=c["text"])
    assert attempts <= 5


# ---- moving window (DESIGN.md §5): local covariance block C = c0 - gamma (c0 = sill, or gamma(2 d_k) for linear / power),
#      augmented Cholesky with the rows [c ; 1 ; Z] -> y_c, y_1, y_Z and NO back substitution:
#      mu = (y_1.y_c - 1) / (y_1.y_1),  z = y_c.y_Z - mu y_1.y_Z,  sigma^2 = c0 - (y_c.y_c - mu y_1.y_c) - mu
def moving_window_model(P, values, model, m, Q, k, exact_values=True):
    from scipy.spatial import cKDTree
    dist, idx = cKDTree(P).query(Q, k=k, eps=0.0)
    z = np.empty(Q.shape[0])
    ss = np.empty(Q.shape[0])
    for j in range(Q.shape[0]):
        S = P[idx[j]]
        gam = ko.variogram(model, m, ko.cdist(S, S))
        np.fill_diagonal(gam, 0.0)
        c0 = (float(ko.variogram(model, m, 2.0 * dist[j].max())) if model in ("linear", "power")
              else float(m[0]) + float(m[2]))
        L = np.linalg.cholesky(c0 - gam)
        b = -ko.variogram(model, m, dist[j])
        if exact_values:
            b[np.abs(dist[j]) <= ko.EPS] = 0.0
        y_c, y_1, y_z = (scipy.linalg.solve_triangular(L, v, lower=True) for v in (c0 + b, np.ones(k), values[idx[j]]))
        mu = (y_1 @ y_c - 1.0) / (y_1 @ y_1)
        z[j] = y_c @ y_z - mu * (y_1 @ y_z)
        ss[j] = c0 - (y_c @ y_c - mu * (y_1 @ y_c)) - mu
    return z, ss


KNN_DRAWS = [t for t in range(cases.N_FUZZ) if (cases.fuzz_config(t) or {}).get("knn") is not None]


@pytest.mark.parametrize("t", KNN_DRAWS)
def test_moving_window_model_reproduces_the_reference(t, ref_fuzz):
    c = cases.fuzz_config(t)
    kw, dim = c["kw"], len(c["data"]) - 1
    data = np.column_stack(c["data"][:dim])
    values = np.asarray(c["data"][dim], dtype=float)
    pts = [np.asarray(p, dtype=float) for p in c["pts"]]
    Qo = np.column_stack(pts) if c["style"] == "points" else ko.grid_points(pts)
    model = kw["variogram_model"]
    m = ko.stored_parameters(model, kw["variogram_parameters"])
    z, ss = moving_window_model(_adjusted(c, data), values, model, m, _adjusted(c, Qo), c["knn"], kw.get("exact_values", True))
    zr, sr = np.ravel(ref_fuzz["%d/z" % t]), np.ravel(ref_fuzz["%d/ss" % t])
    keep = ~np.ravel(ref_fuzz["%d/mask" % t]) if c["style"] == "masked" else np.ones(zr.size, bool)
    if not keep.any():
        return
    tol = 1e-8
    np.testing.assert_allclose(z[keep], zr[keep], rtol=tol, atol=tol * np.abs(zr[keep]).max(), err_msg=c["text"])
    np.testing.assert_allclose(ss[keep], sr[keep], rtol=tol, atol=tol * max(np.abs(sr[keep]).max(), 1e-300), err_msg=c["text"])


# ---- dtype='float64x' / 'float64x5' / 'float64x4' (csrc/solve_wgmma.cu): error-free slicing of W rows and RHS columns into
#      S signed base-128 digits (6 + 7 (S-1) bits), all digit products with d = s + t < S summed exactly in S int32
#      accumulators, exact int64 recombination, one conversion to fp64 ------------------------------------------------
def i8_slices(x, e, S):
    """Balanced digits of round(x * 2^(6 + 7 (S-1) - e)): x = 2^e sum_s out[s] 2^(-6-7s) + O(2^(e-7S)), out[s] in [-64, 64]
    (solve_wgmma.cu: i8_slice)."""
    v = np.rint(np.ldexp(np.asarray(x, dtype=np.float64), 6 + 7 * (S - 1) - e)).astype(np.int64)
    out = np.zeros((S,) + v.shape, dtype=np.int64)
    for s in range(S - 1, 0, -1):
        d = ((v + 64) & 127) - 64
        out[s] = d
        v = (v - d) >> 7
    out[0] = v
    return out


def i8_matvec_rows(W, c, S):
    """(W c)_r through the slice scheme: per-row exponents for W, one exponent for the column c."""
    ew = np.floor(np.log2(np.max(np.abs(W), axis=1))).astype(int) + 1          # |row| * 2^-ew < 1
    ec = int(np.floor(np.log2(np.max(np.abs(c))))) + 1
    ws = np.stack([i8_slices(W[r], int(ew[r]), S) for r in range(W.shape[0])], axis=1)     # [S, rows, n]
    cs = i8_slices(c, ec, S)                                                               # [S, n]
    assert np.abs(ws).max() <= 64 and np.abs(cs).max() <= 64
    V = np.zeros(W.shape[0], dtype=np.int64)
    for d in range(S):
        acc = np.zeros(W.shape[0], dtype=np.int64)
        for s in range(d + 1):
            acc += ws[s] @ cs[d - s]
        assert np.abs(acc).max() < 2 ** 31, "int32 accumulator would overflow"
        V = V * 128 + acc                                                                  # exact in int64
    return np.ldexp(V.astype(np.float64), ew + ec - 12 - 7 * (S - 1))


@pytest.mark.parametrize("S,bits,bound", [(6, 41, 1e-10), (5, 34, 1e-8), (4, 27, 1e-6)])
def test_int8_slice_scheme_is_error_free_and_fp64_class(S, bits, bound):
    rng = np.random.default_rng(99)
    x = rng.normal(size=2000) * np.exp(rng.uniform(-20, 20, 2000))
    e = int(np.floor(np.log2(np.abs(x).max()))) + 1
    sl = i8_slices(x, e, S)
    back = sum(np.ldexp(sl[s].astype(np.float64), e - 6 - 7 * s) for s in range(S))
    assert np.array_equal(back, np.ldexp(np.rint(np.ldexp(x, bits - e)), e - bits))        # the digits carry exactly `bits` bits
    # q = ||W c||^2 of a kriging problem (N = 600, exponential): W = chol(C)^-1, c = c0 + b for a few prediction points
    xyz, val = cases.synth_data(5, 600, 2)
    m = ko.stored_parameters("exponential", [1.0, 300.0, 0.05])
    gam = ko.variogram("exponential", m, ko.cdist(xyz, xyz))
    np.fill_diagonal(gam, 0.0)
    c0 = m[0] + m[2]
    W = scipy.linalg.solve_triangular(np.linalg.cholesky(c0 - gam), np.eye(600), lower=True)
    worst = 0.0
    for q in cases.synth_points(5, 6, 2, xyz, n_hits=1):
        c = c0 - ko.variogram("exponential", m, np.sqrt(np.sum((xyz - q) ** 2, axis=1)))
        exact = W @ c
        got = i8_matvec_rows(W, c, S)
        worst = max(worst, abs(np.sum(got ** 2) - np.sum(exact ** 2)) / np.sum(exact ** 2))
    # relative error of q here: 1.8e-11 / 1.9e-9 / 1.9e-7; sigma^2 = c0 - q + ... loses another ~20x to cancellation (bench.py on an
    # H100 at N=5000: 4e-10 / 4e-6 on sigma^2 for S = 6 / 4)
    assert worst < bound, worst


# ---- dtype='float32' (csrc/solve_wgmma.cu): 3xTF32 split W = Wh + Wl, c = ch + cl (each part representable in TF32:
#      10 explicit mantissa bits, cvt.rna), W c ~= Wh ch + Wh cl + Wl ch accumulated in fp32 ---------------------------
def tf32_round(x):
    """cvt.rna.tf32.f32: round a float32 to 10 mantissa bits, ties away from zero."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return u.view(np.float32)


def tf32x3_matvec(W, c):
    Wh = tf32_round(W.astype(np.float32))
    Wl = tf32_round((W - Wh.astype(np.float64)).astype(np.float32))
    cf = c.astype(np.float32)
    ch = tf32_round(cf)
    cl = tf32_round(cf - ch)
    # products of TF32 operands are exact in fp32's 24 bits x 2 = the tensor core keeps them exact and accumulates in fp32
    return (Wh @ ch + Wh @ cl + Wl @ ch).astype(np.float64), (Wh @ ch).astype(np.float64)


def test_three_tf32_products_recover_fp32_accuracy():
    xyz, val = cases.synth_data(5, 600, 2)
    m = ko.stored_parameters("exponential", [1.0, 300.0, 0.05])
    gam = ko.variogram("exponential", m, ko.cdist(xyz, xyz))
    np.fill_diagonal(gam, 0.0)
    c0 = m[0] + m[2]
    W = scipy.linalg.solve_triangular(np.linalg.cholesky(c0 - gam), np.eye(600), lower=True)
    err3 = err1 = 0.0
    for q in cases.synth_points(5, 6, 2, xyz, n_hits=1):
        c = c0 - ko.variogram("exponential", m, np.sqrt(np.sum((xyz - q) ** 2, axis=1)))
        exact = np.sum((W @ c) ** 2)
        y3, y1 = tf32x3_matvec(W, c)
        err3 = max(err3, abs(np.sum(y3 ** 2) - exact) / exact)
        err1 = max(err1, abs(np.sum(y1 ** 2) - exact) / exact)
    assert err3 < 2e-6, err3            # fp32 class: inside the 1e-2 tolerance of the fp32 arm by four orders
    assert err1 > 20 * err3             # a single TF32 product would not be (the reason for the split)
