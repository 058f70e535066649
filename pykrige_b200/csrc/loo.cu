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
__global__ void loo_finalize_kernel(LooParams P) {
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
// a prediction point (adjusted coordinates; great-circle degrees for geographic). One thread per station i walks all j
// in ascending order through shared-memory tiles: pass 0 counts, pass 1 writes station i's list at off[i] in j order.
template <int DIM>
__global__ void __launch_bounds__(256) loo_pairs_kernel(int n, const double* __restrict__ ax, const double* __restrict__ ay,
                                                        const double* __restrict__ az, double eps, int* __restrict__ cnt,
                                                        const int* __restrict__ off, int* __restrict__ pj,
                                                        double* __restrict__ pd) {
    __shared__ double sx[256], sy[256], sz[256];
    const int i = blockIdx.x * 256 + threadIdx.x;
    const double xi = i < n ? ax[i] : 0.0, yi = i < n ? ay[i] : 0.0, zi = i < n ? az[i] : 0.0;
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
            if (fabs(d) <= eps) {
                if (off) { pj[o + c] = j; pd[o + c] = d; }
                ++c;
            }
        }
    }
    if (i < n && !off) cnt[i] = c;
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
__device__ double loo_pjl(const LooParams& P, int j, int l, int lane) {
    double s;
    if (P.gform == 1) {
        s = P.G[(size_t)j * P.ld + l];
    } else {
        s = 0.0;
        for (int r = max(j, l) + lane; r < P.n; r += 32) s = fma(P.W[(size_t)r * P.ld + j], P.W[(size_t)r * P.ld + l], s);
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    const int K1 = P.K1;
    double usu = 0.0;
    for (int a = 0; a < K1; ++a) {
        double t = 0.0;
        for (int b = 0; b < K1; ++b) t += P.consts[a * K1 + b] * P.Uz[(size_t)b * P.n_pad + l];
        usu += P.Uz[(size_t)a * P.n_pad + j] * t;
    }
    return s - usu;
}

// Exact-hit correction of station i (one warp per station that has near pairs), D = D(i), Delta_j = gamma(d_ij):
//     zhat_v  += sum_j Delta_j (alpha_jv - alpha_iv P_ij / P_ii)
//     sigma^2 += 2 sum_j Delta_j P_ij / P_ii - sum_{j,l} Delta_j Delta_l (P_jl - P_ij P_il / P_ii)
// m = |D(i)| <= LOO_MAXDUP (the host checks); sums run in list order (ascending j).
__global__ void __launch_bounds__(256) loo_dup_kernel(LooParams P, int nst, const int* __restrict__ st,
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

cudaError_t kbk_loo_finalize(const LooParams& p, cudaStream_t st) {
    loo_finalize_kernel<<<(p.n + 127) / 128, 128, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t kbk_loo_pairs(int dim, int n, const double* ax, const double* ay, const double* az, double eps, int* cnt,
                          const int* off, int* pj, double* pd, cudaStream_t st) {
    return KbDims::dispatch(dim, [&](auto D) {
        loo_pairs_kernel<D><<<(n + 255) / 256, 256, 0, st>>>(n, ax, ay, az, eps, cnt, off, pj, pd);
        return cudaGetLastError();
    });
}

cudaError_t kbk_loo_dup(const LooParams& p, int nst, const int* st_list, const int* off, const int* pj, const double* pd,
                        cudaStream_t st) {
    if (nst == 0) return cudaSuccess;
    loo_dup_kernel<<<(nst + 7) / 8, 256, 0, st>>>(p, nst, st_list, off, pj, pd);
    return cudaGetLastError();
}
