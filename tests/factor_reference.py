"""Host reference for the device factorisation of the global path (factor.cu: assemble, blocked Cholesky, triangular
inverse, dual vectors): the kriging matrix C and the drift matrix F by the device's rules, and residual metrics of the
device's L, W = L^-1, U = C^-1 F, S^-1 and phi, accumulated in np.longdouble.

Every metric is a componentwise backward error, normalised by the matching product of absolute values, so it is a
small multiple of the unit roundoff u = 2^-53 for a correct kernel whatever the condition number of C, and of order 1
for a wrong tile, a missed update or a sign error:
  beta_L   max |C - L L^T|_ij / (|L| |L|^T + M)_ij,  M_ij = c0 + |gamma(d_ij)| off the diagonal (see KrigingMatrix)
  beta_WL  max |W L - I|_ij / (|W| |L|)_ij,   beta_LW  max |L W - I|_ij / (|L| |W|)_ij
  beta_U   max_i |F - C U|_i / ((|C| + M) |U| + |F|)_i         (Oettli-Prager, per column of U)
  beta_S   max |S^-1 S - I|_ij / (|S^-1| |F|^T |U|)_ij,  S = F^T U  (from the device's U)
  beta_phi max |phi - F^T zeta|_a / (|F|^T |zeta|)_a
The products are evaluated over the entries (i, j) of I x J in the lower block triangle (tile(i) >= tile(j), 64-row
tiles), so the upper triangle of the diagonal tiles counts: a non-zero there is read by the kernels and shows up here.
0 / 0 counts as 0. L and W are read as they are (their strict upper tiles must be zero). The sums run in longdouble
(64-bit mantissa) and the normalising products in float64: the denominators need no more than a few correct bits.

Full matrices up to n_pad = FULL_MAX; above, I = J = sample_rows(): both edges and one interior row of every 64-row
tile (the interior rows cycle through every residue mod 16, the row positions of the m8n8k4 and m16n8k16 fragments),
every row of two random tiles, and the rows on both sides of the append split. A defect that spans a tile, a tile row
or a fragment position repeated over the tiles always meets sampled rows; a single wrong element is seen when its row
(or, for L, its column) is sampled."""
import numpy as np

from oracle import krige_oracle as ko

TILE = 64
FULL_MAX = 1024
LD = np.longdouble

# Tolerances of tests/test_factor_gpu.py, a few times the worst values measured there (listed in its docstring)
TOL = {"L": 5e-14, "WL": 2e-13, "LW": 2e-14, "U": 1e-15, "S": 2e-15, "phi": 5e-15}


# ---- the device's matrices ------------------------------------------------------------------------------------------
def adjusted(X, center, Mt):
    """The device's adjusted coordinates (kb_adjust): c + Mt (x - c) per row of X [n, dim], in its order of rounded
    operations (no fused multiply-add), so that close pairs get the device's distances to the last bit or so."""
    X = np.asarray(X, dtype=np.float64)
    dim = X.shape[1]
    c = np.asarray(center, dtype=np.float64)
    m = np.asarray(Mt, dtype=np.float64).reshape(dim, dim)
    d = [X[:, j] - c[j] for j in range(dim)]
    out = np.empty_like(X)
    for i in range(dim):
        r = m[i, 0] * d[0]
        for j in range(1, dim):
            r = r + m[i, j] * d[j]
        out[:, i] = r + c[i]
    return out


def unit_vectors(lonlat):
    """Geographic stations on the device: unit vectors of (lon, lat) in degrees (kb_adjust<KB_GEO>)."""
    rad = 0.017453292519943295
    lon, lat = np.asarray(lonlat, dtype=np.float64)[:, 0] * rad, np.asarray(lonlat, dtype=np.float64)[:, 1] * rad
    return np.column_stack([np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)])


def great_circle_degrees(A, B):
    """Great-circle distances [len(A), len(B)] in degrees between unit vectors, the device's formula (kb_dist<KB_GEO>,
    core.py's great-circle distance written with unit vectors): atan2(|a x b|, a . b)."""
    a = [A[:, k][:, None] for k in range(3)]
    b = [B[:, k][None, :] for k in range(3)]
    cx, cy, cz = a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]
    return np.arctan2(np.sqrt(cx * cx + cy * cy + cz * cz), a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) * 57.29577951308232


class KrigingMatrix:
    """C of the assemble kernel (factor.cu): c0 - gamma(d_ij) off the diagonal, c0 on it, the identity in the padding
    rows [n, n_pad). P: adjusted coordinates [n, dim], or (geographic) lon / lat in degrees, whose great-circle
    distances (ko.great_circle_distance to rounding) are formed as the device forms them. params: the device's
    (stored) variogram parameters. block(rows, cols) builds only the entries asked for, so that sampled metrics never
    build the whole matrix, and leaves in last_mag the magnitude c0 + |gamma| of the two terms whose difference each
    off-diagonal entry is (0 on the diagonal and in the padding, which are exact): the device and the host round that
    difference differently, by up to u (c0 + |gamma|), which is far more than u |C_ij| for distant pairs."""

    def __init__(self, P, model, params, c0, geographic=False):
        self.P, self.model, self.params, self.c0, self.geo = np.asarray(P, dtype=np.float64), model, params, c0, geographic
        if geographic:
            self.P = unit_vectors(self.P)
        self.n = self.P.shape[0]

    def block(self, rows, cols):
        rows, cols = np.asarray(rows), np.asarray(cols)
        out = np.zeros((rows.size, cols.size))
        ri, ci = rows < self.n, cols < self.n
        A, B = self.P[rows[ri]], self.P[cols[ci]]
        if self.geo:
            d = great_circle_degrees(A, B)
        else:
            d = np.sqrt(((A[:, None, :] - B[None, :, :]) ** 2).sum(axis=2))
        g = ko.variogram(self.model, self.params, d)
        diag = rows[ri][:, None] == cols[ci][None, :]
        sub = self.c0 - g
        sub[diag] = self.c0
        out[np.ix_(ri, ci)] = sub
        pad = (rows[:, None] == cols[None, :]) & ~ri[:, None]
        out[pad] = 1.0
        mag = self.c0 + np.abs(g)
        mag[diag] = 0.0
        self.last_mag = np.zeros(out.shape)
        self.last_mag[np.ix_(ri, ci)] = mag
        return out


class DriftFrame:
    """The drift rescale the device fixes at the first set-up and keeps through appends (api.cu, describe()):
    regional-linear columns (x_adj - mid) / half of the adjusted bounding box, host drift columns (d - mean) / max|d -
    mean|. P_first: adjusted coordinates of the first set-up; cols_first: its host drift columns."""

    def __init__(self, P_first, n_rl, cols_first=()):
        P_first = np.asarray(P_first, dtype=np.float64)
        self.n_rl = n_rl
        lo, hi = P_first.min(axis=0), P_first.max(axis=0)
        self.shift = [0.5 * (hi[c] + lo[c]) for c in range(n_rl)]
        self.scale = [1.0 / (0.5 * (hi[c] - lo[c])) if hi[c] > lo[c] else 1.0 for c in range(n_rl)]
        for col in cols_first:
            col = np.asarray(col, dtype=np.float64)
            mean = col.sum() / col.size
            amax = np.abs(col - mean).max()
            self.shift.append(mean)
            self.scale.append(1.0 / amax if amax > 0.0 else 1.0)

    def matrix(self, P, cols=()):
        """F [n, K + 1]: the drift columns, then the ones column (build_fz_kernel)."""
        P = np.asarray(P, dtype=np.float64)
        out = [(P[:, c] - self.shift[c]) * self.scale[c] for c in range(self.n_rl)]
        out += [(np.asarray(d, dtype=np.float64) - self.shift[self.n_rl + c]) * self.scale[self.n_rl + c]
                for c, d in enumerate(cols)]
        return np.column_stack(out + [np.ones(P.shape[0])])


# ---- which entries ----------------------------------------------------------------------------------------------------
def sample_rows(n_pad, extra=(), seed=0):
    """All rows [0, n_pad) up to FULL_MAX; above, both edges of every tile, one interior row per tile whose residue
    mod 16 cycles with the tile index, every row of two random tiles, and `extra` (e.g. n0 - 1, n0, n_old - 1, n_old,
    n - 1, n), clipped to [0, n_pad)."""
    if n_pad <= FULL_MAX:
        return np.arange(n_pad)
    nt = n_pad // TILE
    t = np.arange(nt)
    rows = [t * TILE, t * TILE + TILE - 1, t * TILE + 16 + t % 16 + 16 * ((t // 16) % 2)]
    for r in np.random.default_rng(seed).choice(nt, 2, replace=False):
        rows.append(np.arange(r * TILE, r * TILE + TILE))
    rows.append(np.asarray([e for e in extra if 0 <= e < n_pad], dtype=np.int64))
    return np.unique(np.concatenate(rows))


def _groups(idx, size=128):
    """(positions, indices) of consecutive runs of `size` entries of the sorted index set idx"""
    return [(slice(s, s + size), idx[s:s + size]) for s in range(0, idx.size, size)]


def _tile_lo(i):
    return int(i) // TILE * TILE


def _tile_hi(i, n_pad):
    return min(n_pad, _tile_lo(i) + TILE)


def _lower_block_products(A, B, I, J, lower_b):
    """(A B)[I, J] in longdouble and (|A| |B|)[I, J] in float64 over the lower block triangle (tile(i) >= tile(j); other
    entries 0), for a lower block-triangular A [n_pad, n_pad] and B = L^T (lower_b False: k < end of tile(j)) or a
    lower block-triangular B (lower_b True: k in [start of tile(j), end of tile(i)))."""
    n_pad = A.shape[0]
    P = np.zeros((I.size, J.size), dtype=LD)
    Q = np.zeros((I.size, J.size))
    ti, tj = I // TILE, J // TILE
    for ri, gi in _groups(I):
        for ci, gj in _groups(J):
            if gi[-1] // TILE < gj[0] // TILE:
                continue
            k0 = _tile_lo(gj[0]) if lower_b else 0
            k1 = _tile_hi(gi[-1], n_pad) if lower_b else _tile_hi(gj[-1], n_pad)
            a = A[np.ix_(gi, np.arange(k0, k1))]
            b = B[np.ix_(np.arange(k0, k1), gj)]
            P[ri, ci] = a.astype(LD) @ b.astype(LD)
            Q[ri, ci] = np.abs(a) @ np.abs(b)
    mask = ti[:, None] >= tj[None, :]
    P[~mask] = 0
    Q[~mask] = 0.0
    return P, Q, mask


def _ratio(num, den, mask):
    num = np.abs(np.asarray(num, dtype=LD))
    den = np.asarray(den, dtype=LD)
    out = np.zeros(num.shape, dtype=LD)
    nz = den > 0
    out[nz] = num[nz] / den[nz]
    out[~nz & (num > 0)] = np.inf
    out[~mask] = 0
    return float(out.max()) if out.size else 0.0


# ---- metrics ----------------------------------------------------------------------------------------------------------
def _c_block(C, rows, cols):
    """C[rows, cols] and the magnitude of its rounding (KrigingMatrix.last_mag; 0 for a given array)"""
    if hasattr(C, "block"):
        return C.block(rows, cols), C.last_mag
    return C[np.ix_(rows, cols)], 0.0


def cholesky_backward_error(C, L, I):
    """beta_L over I x I: |C - L L^T| / (|L| |L|^T + (c0 + |gamma|)). C: a KrigingMatrix or an [n_pad, n_pad] array."""
    P, Q, mask = _lower_block_products(L, L.T, I, I, lower_b=False)
    Cb, mag = _c_block(C, I, I)
    return _ratio(Cb.astype(LD) - P, Q + mag, mask)


def inverse_residuals(W, L, I):
    """(beta_WL, beta_LW) over I x I."""
    eye = (I[:, None] == I[None, :]).astype(LD)
    P, Q, mask = _lower_block_products(W, L, I, I, lower_b=True)
    b_wl = _ratio(P - eye, Q, mask)
    P, Q, mask = _lower_block_products(L, W, I, I, lower_b=True)
    return b_wl, _ratio(P - eye, Q, mask)


def dual_residual(C, F, U, I):
    """beta_U over the rows I of [n, K + 1] F and U (the data rows; the padding carries no drift)."""
    n = F.shape[0]
    I = I[I < n]
    Cb, mag = _c_block(C, I, np.arange(n))
    r = F[I].astype(LD) - Cb.astype(LD) @ U.astype(LD)
    den = (np.abs(Cb) + mag) @ np.abs(U) + np.abs(F[I])
    return _ratio(r, den, np.ones(r.shape, dtype=bool))


def sinv_residual(Sinv, F, U):
    """beta_S: S^-1 of dual_small_kernel against S = F^T U formed in longdouble from the same U, normalised by
    |S^-1| |F|^T |U| (the device forms S by an n-term reduction, to within a few u of |F|^T |U|)."""
    S = F.astype(LD).T @ U.astype(LD)
    R = Sinv.astype(LD) @ S - np.eye(S.shape[0], dtype=LD)
    den = np.abs(Sinv) @ (np.abs(F).T @ np.abs(U))
    return _ratio(R, den, np.ones(R.shape, dtype=bool))


def phi_residual(phi, F, zeta):
    """beta_phi: phi = F^T zeta of dual_small_kernel."""
    r = np.asarray(phi, dtype=LD) - F.astype(LD).T @ zeta.astype(LD)
    return _ratio(r, np.abs(F).T @ np.abs(zeta), np.ones(r.shape, dtype=bool))
