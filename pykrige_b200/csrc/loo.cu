// loo.cu — leave-one-out cross-validation of every station from the factorisation kb200_set_problem holds
// (DESIGN.md §5e).
//
// M = inverse of the bordered covariance-form matrix [[C, F], [F^T, 0]] (F: rescaled drift columns + ones). Its
// top-left block is P = C^-1 - U S^-1 U^T (U = C^-1 F, S = F^T U), and with alpha_v = P Z_v = zeta_v - U S^-1 phi_v
// (Dubrule 1983):
//     sigma^2_-i = 1 / P_ii,    zhat_-i,v = Z_iv - alpha_iv / P_ii,
//     P_ii = ||W[:, i]||^2 - u_i^T S^-1 u_i     (W = L^-1, lower triangular; gform 1: G_ii instead of ||W[:, i]||^2).
// With exact_values, a station j within eps of station i gets gamma = 0 in the reduced problem's right-hand side, i.e.
// Delta_j = gamma(d_ij) more covariance; loo_dup_kernel adds that correction from P and alpha on {i} + D(i).
#include "common.cuh"
#include "kernels.h"
#include <climits>
#include <algorithm>

#define LOO_CB 128          // columns of W per CTA of the column-norm kernel (one per thread: coalesced row loads)

// part[c][j] = sum over rows r of chunk c (rows [c LOO_RC, (c + 1) LOO_RC) of W, r >= j, r < n) of W[r][j]^2.
// Fixed chunks and a fixed row order inside each: the sums do not depend on the launch.
__global__ void __launch_bounds__(LOO_CB) loo_colsq_kernel(const double* __restrict__ W, int ld, int n,
                                                           double* __restrict__ part) {
    const int j = blockIdx.x * LOO_CB + threadIdx.x;
    const int r0 = blockIdx.y * LOO_RC;
    if (r0 + LOO_RC <= (int)(blockIdx.x * LOO_CB)) return;          // chunk entirely above the diagonal (block-uniform)
    const int r1 = min(n, r0 + LOO_RC);
    double acc = 0.0;
    if (j < n) {
        const double* w = W + j;
#pragma unroll 8
        for (int r = max(r0, j); r < r1; ++r) {
            const double v = w[(size_t)r * ld];
            acc = fma(v, v, acc);
        }
        part[(size_t)blockIdx.y * n + j] = acc;
    }
}

// One thread per station: the diagonal term (chunk sums in chunk order, or G_ii), u_i^T S^-1 u_i, alpha_iv and the
// outputs. Every product and sum of field v is the same whatever nv is and wherever v sits.
__global__ void loo_finalize_kernel(CvParams P) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const int K1 = P.K1;
    double diag;
    if (P.gform == 1) {
        diag = P.G[(size_t)i * P.ld + i];
    } else {
        diag = 0.0;
        for (int c = i / LOO_RC; c < P.nchunks; ++c) diag += P.part[(size_t)c * P.n + i];
    }
    const double* Sinv = P.consts;
    double u[KB200_MAX_DRIFT + 1], wt[KB200_MAX_DRIFT + 1];
    for (int a = 0; a < K1; ++a) u[a] = P.Uz[(size_t)a * P.n_pad + i];
    for (int b = 0; b < K1; ++b) {                    // wt = u_i^T S^-1
        double s = 0.0;
        for (int a = 0; a < K1; ++a) s += u[a] * Sinv[a * K1 + b];
        wt[b] = s;
    }
    double usu = 0.0;
    for (int b = 0; b < K1; ++b) usu += wt[b] * u[b];
    const double pii = diag - usu;
    // drift not determined without station i: P_ii is rounding noise of the difference above
    if (!(fabs(pii) > P.tol * fmax(fabs(diag), fabs(usu)))) atomicMin(P.bad, i);
    P.pii[i] = pii;
    P.ss_out[i] = 1.0 / pii;
    for (int v = 0; v < P.nv; ++v) {
        const double* phi = P.consts + K1 * K1 + v * K1;
        double t = 0.0;
        for (int b = 0; b < K1; ++b) t += wt[b] * phi[b];
        const double alpha = P.Uz[(size_t)(K1 + v) * P.n_pad + i] - t;
        P.alpha[(size_t)v * P.n + i] = alpha;
        P.z_out[(size_t)v * P.n + i] = P.Z[(size_t)v * P.n + i] - alpha / pii;
    }
}

// Near pairs for exact_values: every j != i with |d_ij| <= eps, d as the solve kernels compute it for a data point and
// a prediction point (adjusted coordinates; great-circle degrees for geographic); with grp (leave-group-out) only the j
// of another group than i. One thread per station i walks all j in ascending order through shared-memory tiles: pass 0
// counts, pass 1 writes station i's list at off[i] in j order. GRP: grp is non-null (a template argument, so that the
// leave-one-out scan keeps its loop).
template <int DIM, bool GRP>
__global__ void __launch_bounds__(256) loo_pairs_kernel(int n, const double* __restrict__ ax, const double* __restrict__ ay,
                                                        const double* __restrict__ az, double eps,
                                                        const int* __restrict__ grp, int* __restrict__ cnt,
                                                        const int* __restrict__ off, int* __restrict__ pj,
                                                        double* __restrict__ pd) {
    __shared__ double sx[256], sy[256], sz[256];
    const int i = blockIdx.x * 256 + threadIdx.x;
    const double xi = i < n ? ax[i] : 0.0, yi = i < n ? ay[i] : 0.0, zi = i < n ? az[i] : 0.0;
    const int gi = (GRP && i < n) ? grp[i] : 0;
    int c = 0;
    const int o = (off && i < n) ? off[i] : 0;
    for (int j0 = 0; j0 < n; j0 += 256) {
        __syncthreads();
        const int jl = j0 + threadIdx.x;
        sx[threadIdx.x] = jl < n ? ax[jl] : 0.0; sy[threadIdx.x] = jl < n ? ay[jl] : 0.0; sz[threadIdx.x] = jl < n ? az[jl] : 0.0;
        __syncthreads();
        if (i >= n) continue;
        const int je = min(256, n - j0);
        for (int q = 0; q < je; ++q) {
            const int j = j0 + q;
            if (j == i) continue;
            const double d = kb_dist<DIM>(sx[q], sy[q], sz[q], xi, yi, zi);     // (data j, prediction point i)
            if (fabs(d) <= eps && !(GRP && grp[j] == gi)) {
                if (off) { pj[o + c] = j; pd[o + c] = d; }
                ++c;
            }
        }
    }
    if (i < n && !off) cnt[i] = c;
}

// u_j^T S^-1 u_l (U: the first K1 columns of Uz, S^-1: the first K1 x K1 constants)
__device__ double cv_usu(const CvParams& P, int j, int l) {
    const int K1 = P.K1;
    double usu = 0.0;
    for (int a = 0; a < K1; ++a) {
        double t = 0.0;
        for (int b = 0; b < K1; ++b) t += P.consts[a * K1 + b] * P.Uz[(size_t)b * P.n_pad + l];
        usu += P.Uz[(size_t)a * P.n_pad + j] * t;
    }
    return usu;
}

// sum over the 32 lanes of a warp by a fixed xor tree (every lane gets the same bits)
__device__ __forceinline__ double cv_warp_sum(double s) {
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

__device__ double loo_gamma(const VgParams& v, double d) {
    switch (v.model) {
        case KB200_VG_LINEAR: return kb_gamma<KB200_VG_LINEAR>(v, d);
        case KB200_VG_POWER: return kb_gamma<KB200_VG_POWER>(v, d);
        case KB200_VG_GAUSSIAN: return kb_gamma<KB200_VG_GAUSSIAN>(v, d);
        case KB200_VG_EXPONENTIAL: return kb_gamma<KB200_VG_EXPONENTIAL>(v, d);
        case KB200_VG_SPHERICAL: return kb_gamma<KB200_VG_SPHERICAL>(v, d);
        case KB200_VG_TABLE: return kb_gamma<KB200_VG_TABLE>(v, d);
        default: return kb_gamma<KB200_VG_HOLE_EFFECT>(v, d);
    }
}

// P_jl by one warp: W[:, j] . W[:, l] over rows >= max(j, l) (lanes over rows, fixed xor tree), minus u_j^T S^-1 u_l;
// gform 1: G_jl - u_j^T S^-1 u_l.
__device__ double loo_pjl(const CvParams& P, int j, int l, int lane) {
    double s;
    if (P.gform == 1) {
        s = P.G[(size_t)j * P.ld + l];
    } else {
        s = 0.0;
        for (int r = max(j, l) + lane; r < P.n; r += 32) s = fma(P.W[(size_t)r * P.ld + j], P.W[(size_t)r * P.ld + l], s);
        s = cv_warp_sum(s);
    }
    return s - cv_usu(P, j, l);
}

// Exact-hit correction of station i (one warp per station that has near pairs), D = D(i), Delta_j = gamma(d_ij):
//     zhat_v  += sum_j Delta_j (alpha_jv - alpha_iv P_ij / P_ii)
//     sigma^2 += 2 sum_j Delta_j P_ij / P_ii - sum_{j,l} Delta_j Delta_l (P_jl - P_ij P_il / P_ii)
// m = |D(i)| <= LOO_MAXDUP (the host checks); sums run in list order (ascending j).
__global__ void __launch_bounds__(256) loo_dup_kernel(CvParams P, int nst, const int* __restrict__ st,
                                                      const int* __restrict__ off, const int* __restrict__ pj,
                                                      const double* __restrict__ pd) {
    const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= nst) return;
    const int i = st[w], o = off[i], m = off[i + 1] - o;
    double pij[LOO_MAXDUP], dl[LOO_MAXDUP];
    const double pii = P.pii[i];
    for (int a = 0; a < m; ++a) {
        pij[a] = loo_pjl(P, i, pj[o + a], lane);
        dl[a] = loo_gamma(P.vg, pd[o + a]);
    }
    double ds = 0.0;
    for (int a = 0; a < m; ++a) ds += dl[a] * pij[a] / pii;
    double quad = 0.0;
    for (int a = 0; a < m; ++a)
        for (int b = 0; b < m; ++b) {
            const double pab = (a <= b) ? loo_pjl(P, pj[o + a], pj[o + b], lane) : loo_pjl(P, pj[o + b], pj[o + a], lane);
            quad += dl[a] * dl[b] * (pab - pij[a] * pij[b] / pii);
        }
    if (lane == 0) {
        P.ss_out[i] += 2.0 * ds - quad;
        for (int v = 0; v < P.nv; ++v) {
            const double ai = P.alpha[(size_t)v * P.n + i];
            double dz = 0.0;
            for (int a = 0; a < m; ++a) dz += dl[a] * (P.alpha[(size_t)v * P.n + pj[o + a]] - ai * pij[a] / pii);
            P.z_out[(size_t)v * P.n + i] += dz;
        }
    }
}

cudaError_t kbk_loo_colsq(const double* W, int ld, int n, double* part, cudaStream_t st) {
    const dim3 g((n + LOO_CB - 1) / LOO_CB, (n + LOO_RC - 1) / LOO_RC);
    loo_colsq_kernel<<<g, LOO_CB, 0, st>>>(W, ld, n, part);
    return cudaGetLastError();
}

cudaError_t kbk_loo_finalize(const CvParams& p, cudaStream_t st) {
    loo_finalize_kernel<<<(p.n + 127) / 128, 128, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t kbk_loo_pairs(int dim, int n, const double* ax, const double* ay, const double* az, double eps,
                          const int* grp, int* cnt, const int* off, int* pj, double* pd, cudaStream_t st) {
    return KbDims::dispatch(dim, [&](auto D) {
        return KbBools::dispatch(grp != nullptr, [&](auto GRP) {
            loo_pairs_kernel<D, bool(GRP)><<<(n + 255) / 256, 256, 0, st>>>(n, ax, ay, az, eps, grp, cnt, off, pj, pd);
            return cudaGetLastError();
        });
    });
}

cudaError_t kbk_loo_dup(const CvParams& p, int nst, const int* st_list, const int* off, const int* pj, const double* pd,
                        cudaStream_t st) {
    if (nst == 0) return cudaSuccess;
    loo_dup_kernel<<<(nst + 7) / 8, 256, 0, st>>>(p, nst, st_list, off, pj, pd);
    return cudaGetLastError();
}

// ---- leave-group-out (DESIGN.md §5f) --------------------------------------------------------------------------------
// For a group S (T: the other stations), with P and alpha as above and G = C^-1 held as a lower triangle:
//     e_S,v = P_SS^-1 alpha_S,v,   zhat_S,v = Z_S,v - e_S,v,   sigma^2_S = diag(P_SS^-1).
// The blocks P_SS of all groups are gathered into one array (group g: m_g x m_g, row-major, stations ascending), each is
// replaced by its inverse (lgo_small_kernel in shared memory, or the blocked factor kernels on a padded copy for a
// large group), then lgo_finalize_kernel forms e, zhat and sigma^2 and lgo_dup_kernel the exact-hit correction.

// P_jl = G_jl - u_j^T S^-1 u_l, evaluated in the order (max(j, l), min(j, l)) so that P is exactly symmetric;
// *usu_out = u_j^T S^-1 u_l
__device__ double lgo_p(const CvParams& P, int j, int l, double* usu_out = nullptr) {
    const int hi = max(j, l), lo = min(j, l);
    const double s = P.G[(size_t)hi * P.ld + lo];
    const double usu = cv_usu(P, hi, lo);
    if (usu_out) *usu_out = usu;
    return s - usu;
}

// blk[boff[g] + a m + b] = P_{S_a S_b} for every group g = blockIdx.y (grid-stride over its m^2 entries); the diagonal also
// gives scale[goff[g] + a] = max(|G_ii|, |u_i^T S^-1 u_i|), the terms whose difference P_ii is
__global__ void __launch_bounds__(256) lgo_gather_kernel(CvParams P) {
    const int g = blockIdx.y, o = P.goff[g], m = P.goff[g + 1] - o;
    double* blk = P.blk + P.boff[g];
    for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < (long long)m * m; e += (long long)gridDim.x * 256) {
        const int a = (int)(e / m), b = (int)(e % m);
        const int i = P.mem[o + a], j = P.mem[o + b];
        double usu;
        blk[e] = lgo_p(P, i, j, &usu);
        if (a == b) P.scale[o + a] = fmax(fabs(P.G[(size_t)i * P.ld + i]), fabs(usu));
    }
}

// In-place Gauss-Jordan inverse of one small block (m <= LGO_SMALL) in shared memory, one CTA per group: partial
// pivoting (largest |value|, ties to the lower row), the column swaps in reverse order at the end. A pivot at or below
// tol * scale of its station means the drift is not determined without the group: *bad = lowest such group.
__global__ void __launch_bounds__(256) lgo_small_kernel(CvParams P, const int* __restrict__ glist) {
    extern __shared__ __align__(16) double lsm[];
    __shared__ double wv[8]; __shared__ int wi[8];
    __shared__ int fail;
    const int g = glist[blockIdx.x], o = P.goff[g], m = P.goff[g + 1] - o;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* A = lsm;                                 // m x m
    double* col = A + (size_t)m * m;                 // column k before the update
    int* piv = reinterpret_cast<int*>(col + m);      // row swapped with row k at step k
    int* rid = piv + m;                              // position in the group of the row's station
    double* blk = P.blk + P.boff[g];
    for (int e = tid; e < m * m; e += 256) A[e] = blk[e];
    for (int t = tid; t < m; t += 256) rid[t] = t;
    if (tid == 0) fail = 0;
    __syncthreads();
    for (int k = 0; k < m; ++k) {
        double bv = -1.0; int bi = m;
        for (int r = k + tid; r < m; r += 256) {
            const double v = fabs(A[r * m + k]);
            if (v > bv || (v == bv && r < bi)) { bv = v; bi = r; }
        }
        for (int s = 16; s > 0; s >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, s);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < 8; ++w)
                if (wv[w] > bv || (wv[w] == bv && wi[w] < bi)) { bv = wv[w]; bi = wi[w]; }
            piv[k] = bi;
        }
        __syncthreads();
        const int p = piv[k];
        if (p != k) {
            for (int c = tid; c < m; c += 256) { const double t = A[k * m + c]; A[k * m + c] = A[p * m + c]; A[p * m + c] = t; }
            if (tid == 0) { const int t = rid[k]; rid[k] = rid[p]; rid[p] = t; }
        }
        __syncthreads();
        const double pv = A[k * m + k];
        const double inv = 1.0 / pv;
        if (tid == 0 && !(fabs(pv) > P.tol * P.scale[o + rid[k]])) fail = 1;
        for (int r = tid; r < m; r += 256) col[r] = A[r * m + k];
        __syncthreads();
        for (int c = tid; c < m; c += 256) A[k * m + c] = (c == k) ? inv : A[k * m + c] * inv;
        __syncthreads();
        for (int e = tid; e < m * m; e += 256) {
            const int r = e / m, c = e - r * m;
            if (r == k) continue;
            A[e] = (c == k) ? -col[r] * inv : A[e] - col[r] * A[k * m + c];
        }
        __syncthreads();
    }
    for (int k = m - 1; k >= 0; --k) {
        const int p = piv[k];
        if (p != k)
            for (int r = tid; r < m; r += 256) { const double t = A[r * m + k]; A[r * m + k] = A[r * m + p]; A[r * m + p] = t; }
        __syncthreads();
    }
    for (int e = tid; e < m * m; e += 256) blk[e] = A[e];
    if (tid == 0 && fail) atomicMin(P.bad, g);
}

// padded copy of a large block for the blocked factor kernels: dst (ld x ld) = [[blk, 0], [0, d I]]
__global__ void lgo_pad_kernel(const double* __restrict__ blk, int m, double* __restrict__ dst, int ld, double d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= ld) return;
    dst[(size_t)r * ld + c] = (r < m && c < m) ? blk[(size_t)r * m + c] : (r == c ? d : 0.0);
}

// ... and back: blk[r][c] = src[max(r, c)][min(r, c)] (the lower triangle of the inverse)
__global__ void lgo_unpad_kernel(const double* __restrict__ src, int ld, double* __restrict__ blk, int m) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= m) return;
    blk[(size_t)r * m + c] = src[(size_t)max(r, c) * ld + min(r, c)];
}

// One thread per station i (group g, position a): e_v = row a of P_SS^-1 . alpha_S,v (b ascending), zhat = Z - e,
// sigma^2 = (P_SS^-1)_aa. Every product and sum of field v is the same whatever nv is and wherever v sits.
__global__ void lgo_finalize_kernel(CvParams P) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const int g = P.grp[i], o = P.goff[g], m = P.goff[g + 1] - o, a = P.pos[i];
    const double* row = P.blk + P.boff[g] + (size_t)a * m;
    P.ss_out[i] = row[a];
    for (int v = 0; v < P.nv; ++v) {
        const double* al = P.alpha + (size_t)v * P.n;
        double e = 0.0;
        for (int b = 0; b < m; ++b) e += row[b] * al[P.mem[o + b]];
        P.e[(size_t)v * P.n + i] = e;
        P.z_out[(size_t)v * P.n + i] = P.Z[(size_t)v * P.n + i] - e;
    }
}

// Exact-hit correction of station i in S (one warp per station with near stations outside its group), D = D(i) at
// pj/pd + off[i] (ascending j, at most LOO_MAXDUP), Delta_j = gamma(d_ij), Q = P_SS^-1:
//     zhat_v  += sum_j Delta_j (alpha_jv - P_jS e_S,v)
//     sigma^2 += 2 sum_j Delta_j (P_jS Q)_a - sum_{j,l} Delta_j Delta_l (P_jl - P_jS Q P_Sl)
// scratch + soff[w]: P_jS (|D| x m), then P_jS Q (|D| x m). Lanes split b; sums over b close with a fixed xor tree.
__global__ void __launch_bounds__(256) lgo_dup_kernel(CvParams P, int nst, const int* __restrict__ st,
                                                      const int* __restrict__ off, const int* __restrict__ pj,
                                                      const double* __restrict__ pd, const long long* __restrict__ soff,
                                                      double* __restrict__ scratch) {
    const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= nst) return;
    const int i = st[w], d0 = off[i], cnt = off[i + 1] - d0;
    const int g = P.grp[i], o = P.goff[g], m = P.goff[g + 1] - o, a = P.pos[i];
    const double* Q = P.blk + P.boff[g];
    double* ps = scratch + soff[w];                  // [cnt][m] P_jS
    double* qs = ps + (size_t)cnt * m;               // [cnt][m] P_jS Q
    double dl[LOO_MAXDUP];
    for (int t = 0; t < cnt; ++t) {
        dl[t] = loo_gamma(P.vg, pd[d0 + t]);
        for (int b = lane; b < m; b += 32) ps[(size_t)t * m + b] = lgo_p(P, pj[d0 + t], P.mem[o + b]);
    }
    __syncwarp();
    for (int t = 0; t < cnt; ++t)
        for (int b = lane; b < m; b += 32) {
            double s = 0.0;
            for (int c = 0; c < m; ++c) s += ps[(size_t)t * m + c] * Q[(size_t)c * m + b];
            qs[(size_t)t * m + b] = s;
        }
    __syncwarp();
    double ds = 0.0, quad = 0.0;
    for (int t = 0; t < cnt; ++t) {
        ds += dl[t] * qs[(size_t)t * m + a];
        for (int u = 0; u < cnt; ++u) {
            double s = 0.0;
            for (int b = lane; b < m; b += 32) s += qs[(size_t)t * m + b] * ps[(size_t)u * m + b];
            s = cv_warp_sum(s);
            quad += dl[t] * dl[u] * (lgo_p(P, pj[d0 + t], pj[d0 + u]) - s);
        }
    }
    double dz[KB200_MAX_FIELDS];
    for (int v = 0; v < P.nv; ++v) {
        const double* e = P.e + (size_t)v * P.n;
        double acc = 0.0;
        for (int t = 0; t < cnt; ++t) {
            double s = 0.0;
            for (int b = lane; b < m; b += 32) s += ps[(size_t)t * m + b] * e[P.mem[o + b]];
            s = cv_warp_sum(s);
            acc += dl[t] * (P.alpha[(size_t)v * P.n + pj[d0 + t]] - s);
        }
        dz[v] = acc;
    }
    if (lane == 0) {
        P.ss_out[i] += 2.0 * ds - quad;
        for (int v = 0; v < P.nv; ++v) P.z_out[(size_t)v * P.n + i] += dz[v];
    }
}

cudaError_t kbk_lgo_gather(const CvParams& p, int n_groups, int max_m, cudaStream_t st) {
    const long long e = (long long)max_m * max_m;
    const int bx = (int)std::min<long long>(64, (e + 255) / 256);
    lgo_gather_kernel<<<dim3(bx, n_groups), 256, 0, st>>>(p);
    return cudaGetLastError();
}

size_t kbk_lgo_small_smem(int m) { return (size_t)m * m * sizeof(double) + (size_t)m * (sizeof(double) + 2 * sizeof(int)); }

cudaError_t kbk_lgo_small(const CvParams& p, int count, const int* glist, int max_m, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const size_t smem = kbk_lgo_small_smem(max_m);
    KB_CUDA_OK(cudaFuncSetAttribute(lgo_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lgo_small_kernel<<<count, 256, smem, st>>>(p, glist);
    return cudaGetLastError();
}

cudaError_t kbk_lgo_pad(const double* blk, int m, double* dst, int ld, double d, cudaStream_t st) {
    lgo_pad_kernel<<<dim3((ld + 255) / 256, ld), 256, 0, st>>>(blk, m, dst, ld, d);
    return cudaGetLastError();
}

cudaError_t kbk_lgo_unpad(const double* src, int ld, double* blk, int m, cudaStream_t st) {
    lgo_unpad_kernel<<<dim3((m + 255) / 256, m), 256, 0, st>>>(src, ld, blk, m);
    return cudaGetLastError();
}

cudaError_t kbk_lgo_finalize(const CvParams& p, cudaStream_t st) {
    lgo_finalize_kernel<<<(p.n + 127) / 128, 128, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t kbk_lgo_dup(const CvParams& p, int nst, const int* st_list, const int* off, const int* pj, const double* pd,
                        const long long* soff, double* scratch, cudaStream_t st) {
    if (nst == 0) return cudaSuccess;
    lgo_dup_kernel<<<(nst + 7) / 8, 256, 0, st>>>(p, nst, st_list, off, pj, pd, soff, scratch);
    return cudaGetLastError();
}
