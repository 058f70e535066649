// factor.cu — one-off (per problem) device work of the global kriging path:
//   K1  assemble the shifted covariance matrix C = c0*11^T - Gamma     (ok.py:626-648, uk.py:861-875)
//   K2a blocked Cholesky  C = L L^T  (DMMA trailing updates)            replaces scipy.linalg.inv, ok.py:663
//   K2b blocked triangular inverse  W = L^-1 (DMMA GEMMs)
//   K2c dual vectors  Uz = C^-1 [F | Z],  S = F^T C^-1 F, S^-1, phi
//   K2d pack W (+ dual rows) into the fragment-ordered tile stream read by the solve kernel
// See DESIGN.md §3-§4 for the algebra (covariance-form kriging; results equal the
// reference's inverse x RHS, ok.py:679-681, to rounding).
#include "common.cuh"
#include "kernels.h"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

// ---------------------------------------------------------------------------
// adjusted data coordinates (core.py:120-193 applied to the data, ok.py:284-289)
template <int DIM>
__global__ void adjust_data_kernel(Aniso an, int n, const double* __restrict__ x,
                                   const double* __restrict__ y, const double* __restrict__ z,
                                   double* __restrict__ ax, double* __restrict__ ay, double* __restrict__ az) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double ox, oy, oz;
    kb_adjust<DIM>(an, x[i], y[i], DIM == 3 ? z[i] : 0.0, ox, oy, oz);
    ax[i] = ox; ay[i] = oy; az[i] = oz;
}

// ---------------------------------------------------------------------------
// K1: C[i][j] = c0 - gamma(|p_i - p_j|) (i != j), c0 on the diagonal; identity in the
// padding. Only tiles on/below the diagonal are written (Cholesky reads the lower triangle), and only those of the
// tile rows [it0, n_pad / 64): it0 = 0 for a new factorisation, the first new tile row for appended stations.
// HBM-write bound: n_pad^2/2 * 8 bytes.
template <int DIM, int MODEL>
__global__ void __launch_bounds__(256) assemble_kernel(VgParams vg, int n, int ld, int it0,
                                                        const double* __restrict__ ax,
                                                        const double* __restrict__ ay,
                                                        const double* __restrict__ az,
                                                        double* __restrict__ C) {
    // blockIdx.x -> lower-triangular tile (it >= jt) of 64x64, counted from the first tile of row it0
    int t = blockIdx.x + it0 * (it0 + 1) / 2;
    int it = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while ((long long)(it + 1) * (it + 2) / 2 <= t) ++it;
    while ((long long)it * (it + 1) / 2 > t) --it;
    int jt = t - (int)((long long)it * (it + 1) / 2);
    __shared__ double sx[64], sy[64], sz[64];   // column (j) points
    int tid = threadIdx.x;
    if (tid < 64) {
        int j = jt * 64 + tid;
        bool ok = j < n;
        sx[tid] = ok ? ax[j] : 0.0;
        sy[tid] = ok ? ay[j] : 0.0;
        sz[tid] = (ok && KB_HASZ(DIM)) ? az[j] : 0.0;
    }
    __syncthreads();
    int jl = tid & 63;          // column within tile (contiguous -> coalesced stores)
    int i0 = tid >> 6;          // 0..3
    int j = jt * 64 + jl;
    for (int r = i0; r < 64; r += 4) {
        int i = it * 64 + r;
        double v;
        if (i < n && j < n) {
            if (i == j) v = vg.c0;
            else {
                double d = kb_dist<DIM>(ax[i], ay[i], KB_HASZ(DIM) ? az[i] : 0.0, sx[jl], sy[jl], sz[jl]);
                v = vg.c0 - kb_gamma<MODEL>(vg, d);
            }
        } else {
            v = (i == j) ? 1.0 : 0.0;
        }
        C[(size_t)i * ld + j] = v;
    }
}

// ---------------------------------------------------------------------------
// 64x64 DMMA GEMM tile core used by the Cholesky trailing update, the
// triangular inverse and the Gram product W^T W: acc(64x64) += A(64 x [k0,k1)) * B([k0,k1) x 64).
//   A row-major (lda);  TA -> At[k*lda + i].  B: NN -> B[k*ldb + j];  NT -> Bt[j*ldb + k].
// 128 threads = 4 warps (2x2), each warp a 32x32 sub-tile = 4x4 m8n8k4 tiles.
// smem rows are padded (+4 doubles) so the 8x4 / 4x8 fragment reads are conflict-free.
#define GT_LDS_A 20
#define GT_LDS_BN 68
struct GemmSmem {
    double a[64 * GT_LDS_A];
    double b[64 * GT_LDS_A > 16 * GT_LDS_BN ? 64 * GT_LDS_A : 16 * GT_LDS_BN];
};

template <bool NT, bool TA = false>
__device__ __forceinline__ void gemm_tile_64(double (&acc)[4][4][2], GemmSmem& sm,
                                             const double* __restrict__ A, int lda,
                                             const double* __restrict__ B, int ldb,
                                             int k0, int k1) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1;
    // global->register staging: A (and NT-B) tile 64x16: thread -> row tid/2, half (tid&1)*8
    const int ar = tid >> 1, ah = (tid & 1) * 8;
    // NN-B tile 16x64: thread -> k = tid/8, j0 = (tid&7)*8
    const int bk = tid >> 3, bj = (tid & 7) * 8;
    double ra[8], rb[8];
    auto gload = [&](int k) {
        if (TA) {                                      // At tile 16x64: the NN-B mapping
            const double* pa = A + (size_t)(k + bk) * lda + bj;
#pragma unroll
            for (int q = 0; q < 8; ++q) ra[q] = pa[q];
        } else {
            const double* pa = A + (size_t)ar * lda + k + ah;
#pragma unroll
            for (int q = 0; q < 8; ++q) ra[q] = pa[q];
        }
        if (NT) {
            const double* pb = B + (size_t)ar * ldb + k + ah;
#pragma unroll
            for (int q = 0; q < 8; ++q) rb[q] = pb[q];
        } else {
            const double* pb = B + (size_t)(k + bk) * ldb + bj;
#pragma unroll
            for (int q = 0; q < 8; ++q) rb[q] = pb[q];
        }
    };
    if (k0 >= k1) return;
    gload(k0);
    for (int k = k0; k < k1; k += 16) {
        __syncthreads();   // previous tile fully consumed
        if (TA) {
#pragma unroll
            for (int q = 0; q < 8; ++q) sm.a[(bj + q) * GT_LDS_A + bk] = ra[q];
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) sm.a[ar * GT_LDS_A + ah + q] = ra[q];
        }
        if (NT) {
#pragma unroll
            for (int q = 0; q < 8; ++q) sm.b[ar * GT_LDS_A + ah + q] = rb[q];
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) sm.b[bk * GT_LDS_BN + bj + q] = rb[q];
        }
        __syncthreads();
        if (k + 16 < k1) gload(k + 16);
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
            double fa[4], fb[4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
                fa[mt] = sm.a[(wm * 32 + mt * 8 + (lane >> 2)) * GT_LDS_A + k4 * 4 + (lane & 3)];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                int col = wn * 32 + nt * 8 + (lane >> 2);
                fb[nt] = NT ? sm.b[col * GT_LDS_A + k4 * 4 + (lane & 3)]
                            : sm.b[(k4 * 4 + (lane & 3)) * GT_LDS_BN + col];
            }
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
                    kb_dmma(acc[mt][nt][0], acc[mt][nt][1], fa[mt], fb[nt]);
        }
    }
}

// out = alpha*acc + beta*out   (64x64 tile at `out`, row-major ldc)
__device__ __forceinline__ void gemm_tile_store(const double (&acc)[4][4][2], double* out, int ldc,
                                                double alpha, double beta) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp >> 1, wn = warp & 1;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            int r = wm * 32 + mt * 8 + (lane >> 2);
            int c = wn * 32 + nt * 8 + 2 * (lane & 3);
            double2* p = reinterpret_cast<double2*>(out + (size_t)r * ldc + c);
            double2 v;
            if (beta != 0.0) {
                v = *p;
                v.x = alpha * acc[mt][nt][0] + beta * v.x;
                v.y = alpha * acc[mt][nt][1] + beta * v.y;
            } else {
                v.x = alpha * acc[mt][nt][0];
                v.y = alpha * acc[mt][nt][1];
            }
            *p = v;
        }
}

// ---------------------------------------------------------------------------
// K2a.1  fused panel step of the blocked Cholesky (one launch per 64-column step; replaces the potf2 / trsm /
// thin-update launch triple of round 1). Block column kb of the outer panel that starts at block ob:
//   every CTA   D = C[kb][kb] - A_d A_d^T   (A_d = C[kb rows][ob*64 .. kb*64): the updates of the earlier steps of
//               this outer panel, applied left-looking),  L = chol(D),  Winv = L^-1     -- redundantly, in shared memory:
//               the 64^3/3 flops are nothing, the point is that no CTA waits for another one;
//   CTA 0       writes Winv into the diagonal block of W (the starting point of the triangular inverse K2b), L into a
//               STAGING tile (the other CTAs of this launch may still be reading D from C: the diagonal blocks of C are
//               overwritten by diag_writeback_kernel after the factorisation), and reports a non-positive pivot;
//   CTA b >= 1  its 64-row slab X = C[slab][kb] - A_s A_d^T, then X <- X Winv^T (= X L^-T) on the DMMA pipe.
// potf2 and the triangular inverse are blocked by 16 inside the 64x64 tile: the 16x16 diagonal blocks are done by
// one warp without block-wide barriers, everything else is small dense updates by all 256 threads (12 + 6 barriers
// instead of 256). A pivot at or below dtol (16 eps c0: the rounding noise of c0 - sum l^2, so exactly redundant
// points are caught like scipy's exact zero pivot) sets *flag = 1 + global column index.
#define PN_LD 65
#define PN_SMEM ((3 * 64 * PN_LD + 64) * sizeof(double))

// acc(8 rows of this warp x 64 cols) (+)= sign * A[r][k] * B[c][k], k in [0, 64): A, B row-major [64][PN_LD] in smem
__device__ __forceinline__ void pn_mma_nt(double (&acc)[8][2], const double* A, const double* B, int warp, int lane, int kend) {
#pragma unroll 4
    for (int k4 = 0; k4 < kend; k4 += 4) {
        const double fa = A[(warp * 8 + (lane >> 2)) * PN_LD + k4 + (lane & 3)];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const double fb = B[(nt * 8 + (lane >> 2)) * PN_LD + k4 + (lane & 3)];
            kb_dmma(acc[nt][0], acc[nt][1], fa, fb);
        }
    }
}

// the same restricted to the column tiles nt <= warp (lower block triangle of a symmetric product)
__device__ __forceinline__ void pn_mma_nt_lower(double (&acc)[8][2], const double* A, const double* B, int warp, int lane) {
#pragma unroll 4
    for (int k4 = 0; k4 < 64; k4 += 4) {
        const double fa = A[(warp * 8 + (lane >> 2)) * PN_LD + k4 + (lane & 3)];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            if (nt <= warp) {
                const double fb = B[(nt * 8 + (lane >> 2)) * PN_LD + k4 + (lane & 3)];
                kb_dmma(acc[nt][0], acc[nt][1], fa, fb);
            }
        }
    }
}

__global__ void __launch_bounds__(256) panel_kernel(double* __restrict__ C, double* __restrict__ W, double* __restrict__ Lstage,
                                                     int ld, int kb, int ob, int* __restrict__ flag, double dtol) {
    extern __shared__ double pn_sm[];
    double* a = pn_sm;                       // D -> L
    double* b1 = pn_sm + 64 * PN_LD;         // chunk of A_d, later Winv
    double* b2 = pn_sm + 2 * 64 * PN_LD;     // chunk of A_s, later the slab X
    double* dnv = pn_sm + 3 * 64 * PN_LD;    // 1 / L[j][j]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool owner = blockIdx.x == 0;
    const size_t drow = (size_t)kb * 64;
    const size_t srow = owner ? drow : (size_t)(kb + blockIdx.x) * 64;        // slab rows (CTA 0: the diagonal block itself)
    // fragment ownership of the 64x64 results: warp -> rows 8w..8w+7, lane -> row (lane>>2), cols nt*8 + 2*(lane&3) + {0,1}
    double accD[8][2], accX[8][2];
    {
        const double* Dg = C + (drow + warp * 8 + (lane >> 2)) * ld + drow;
        const double* Xg = C + (srow + warp * 8 + (lane >> 2)) * ld + drow;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int c = nt * 8 + 2 * (lane & 3);
            const double2 d = *reinterpret_cast<const double2*>(Dg + c);
            accD[nt][0] = -d.x; accD[nt][1] = -d.y;          // accumulate the NEGATIVE: acc = A A^T - D
            if (!owner) {
                const double2 x = *reinterpret_cast<const double2*>(Xg + c);
                accX[nt][0] = -x.x; accX[nt][1] = -x.y;
            } else { accX[nt][0] = 0.0; accX[nt][1] = 0.0; }
        }
    }
    for (int pc = ob; pc < kb; ++pc) {                       // pending 64-column chunks of this outer panel
        __syncthreads();
        for (int e = tid; e < 64 * 32; e += 256) {
            const int r = e >> 5, c = (e & 31) * 2;
            const double2 vd = *reinterpret_cast<const double2*>(C + (drow + r) * ld + (size_t)pc * 64 + c);
            b1[r * PN_LD + c] = vd.x; b1[r * PN_LD + c + 1] = vd.y;
            if (!owner) {
                const double2 vs = *reinterpret_cast<const double2*>(C + (srow + r) * ld + (size_t)pc * 64 + c);
                b2[r * PN_LD + c] = vs.x; b2[r * PN_LD + c + 1] = vs.y;
            }
        }
        __syncthreads();
        pn_mma_nt_lower(accD, b1, b1, warp, lane);           // only the tiles on/below the diagonal of D are used
        if (!owner) pn_mma_nt(accX, b2, b1, warp, lane, 64);
    }
    __syncthreads();
    {   // D (updated, lower part) -> a ; slab X -> b2
        const int r = warp * 8 + (lane >> 2);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int c = nt * 8 + 2 * (lane & 3);
            a[r * PN_LD + c] = -accD[nt][0]; a[r * PN_LD + c + 1] = -accD[nt][1];
            b2[r * PN_LD + c] = -accX[nt][0]; b2[r * PN_LD + c + 1] = -accX[nt][1];
        }
    }
    __syncthreads();
    // ---- potf2 of a (lower triangle), blocked by 16 ----
    for (int jb = 0; jb < 4; ++jb) {
        const int j0 = jb * 16;
        if (warp == 0) {                                     // 16x16 diagonal block in registers: lane & 15 = row, shuffles
            const int r = lane & 15;                         // (both half-warps compute the same thing)
            double d[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) d[c] = (c <= r) ? a[(j0 + r) * PN_LD + j0 + c] : 0.0;
            double dinv = 1.0;
#pragma unroll
            for (int pc = 0; pc < 16; ++pc) {
                double piv = __shfl_sync(0xffffffffu, d[pc], pc, 16);
                if (!(piv > dtol)) { if (owner && lane == 0 && *flag == 0) *flag = 1 + kb * 64 + j0 + pc; piv = 1.0; }
                const double inv = rsqrt(piv);
                const double l = d[pc] * inv;                // lane pc: sqrt(piv); lanes below: L[r][pc]
                d[pc] = (r == pc) ? piv * inv : l;
                if (r == pc) dinv = inv;
#pragma unroll
                for (int c = pc + 1; c < 16; ++c) d[c] = fma(-l, __shfl_sync(0xffffffffu, l, c, 16), d[c]);
            }
            if (lane < 16) {
#pragma unroll
                for (int c = 0; c < 16; ++c) if (c <= r) a[(j0 + r) * PN_LD + j0 + c] = d[c];
                dnv[j0 + r] = dinv;
            }
        }
        __syncthreads();
        const int below = 64 - j0 - 16;                      // rows under the diagonal block
        if (below > 0) {
            if (tid < below) {                               // X <- X L16^-T: one thread per row, 16-step substitution
                double* xr = a + (j0 + 16 + tid) * PN_LD + j0;
                double x[16];
#pragma unroll
                for (int c = 0; c < 16; ++c) x[c] = xr[c];
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    double sacc = x[c];
#pragma unroll
                    for (int j = 0; j < c; ++j) sacc = fma(-x[j], a[(j0 + c) * PN_LD + j0 + j], sacc);
                    x[c] = sacc * dnv[j0 + c];
                }
#pragma unroll
                for (int c = 0; c < 16; ++c) xr[c] = x[c];
            }
            __syncthreads();
            for (int i = warp; i < below; i += 8) {          // rank-16 update of the trailing lower triangle: warp = row
                const double* pi = a + (j0 + 16 + i) * PN_LD + j0;
                for (int k = lane; k <= i; k += 32) {
                    const double* pk = a + (j0 + 16 + k) * PN_LD + j0;
                    double sacc = 0.0;
#pragma unroll
                    for (int j = 0; j < 16; ++j) sacc = fma(pi[j], pk[j], sacc);
                    a[(j0 + 16 + i) * PN_LD + j0 + 16 + k] -= sacc;
                }
            }
            __syncthreads();
        }
    }
    // ---- Winv = L^-1 into b1, blocked by 16 ----
    for (int e = tid; e < 64 * 64; e += 256) b1[(e >> 6) * PN_LD + (e & 63)] = 0.0;
    __syncthreads();
    if (tid < 64) {                                          // the four 16x16 diagonal inverses: thread = (block, column)
        const int blk = tid >> 4, c = tid & 15, o = blk * 16;
        double x[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            double sacc = (i == c) ? 1.0 : 0.0;
#pragma unroll
            for (int k = 0; k < i; ++k) if (k >= c) sacc -= a[(o + i) * PN_LD + o + k] * x[k];
            x[i] = (i >= c) ? sacc * dnv[o + i] : 0.0;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) b1[(o + i) * PN_LD + o + c] = x[i];
    }
    __syncthreads();
    for (int ib = 1; ib < 4; ++ib) {                         // block row ib: X_ij = -X_ii (sum_{k=j}^{ib-1} L_ik X_kj), j < ib
        // T_ij goes (transposed) into the strict upper triangle of `a`, which nothing reads: rows < ib*16, columns >= ib*16
        for (int e = tid; e < 16 * 16 * ib; e += 256) {
            const int j = e >> 8, r = (e >> 4) & 15, c = e & 15;          // block column j, element (r, c)
            double sacc = 0.0;
            for (int k = j * 16; k < ib * 16; ++k) sacc += a[(ib * 16 + r) * PN_LD + k] * b1[k * PN_LD + j * 16 + c];
            a[(j * 16 + c) * PN_LD + ib * 16 + r] = sacc;
        }
        __syncthreads();
        for (int e = tid; e < 16 * 16 * ib; e += 256) {
            const int j = e >> 8, r = (e >> 4) & 15, c = e & 15;
            double sacc = 0.0;
#pragma unroll
            for (int k = 0; k < 16; ++k) sacc += b1[(ib * 16 + r) * PN_LD + ib * 16 + k] * a[(j * 16 + c) * PN_LD + ib * 16 + k];
            b1[(ib * 16 + r) * PN_LD + j * 16 + c] = -sacc;
        }
        __syncthreads();
    }
    if (owner) {
        for (int e = tid; e < 64 * 64; e += 256) {
            const int r = e >> 6, c = e & 63;
            Lstage[(size_t)kb * 4096 + e] = (c <= r) ? a[r * PN_LD + c] : 0.0;
            W[(drow + r) * ld + drow + c] = b1[r * PN_LD + c];
        }
        return;
    }
    // ---- slab: X <- X Winv^T  (out[i][c] = sum_{j <= c} X[i][j] Winv[c][j]) ----
    double acc[8][2];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { acc[nt][0] = 0.0; acc[nt][1] = 0.0; }
    pn_mma_nt(acc, b2, b1, warp, lane, 64);
    {
        double* Xg = C + (srow + warp * 8 + (lane >> 2)) * ld + drow;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
            *reinterpret_cast<double2*>(Xg + nt * 8 + 2 * (lane & 3)) = make_double2(acc[nt][0], acc[nt][1]);
    }
}

// staged diagonal factors -> the diagonal blocks of C (after the last panel step; one CTA per block)
__global__ void __launch_bounds__(256) diag_writeback_kernel(double* __restrict__ C, const double* __restrict__ Lstage, int ld) {
    const size_t drow = (size_t)blockIdx.x * 64;
    for (int e = threadIdx.x; e < 4096; e += 256)
        C[(drow + (e >> 6)) * ld + drow + (e & 63)] = Lstage[(size_t)blockIdx.x * 4096 + e];
}

// K2a.3  rank-(64*pkw) update:  C[it][jt] -= P_it P_jt^T  with  P_x = C[x-rows][pk0*64 .. (pk0+pkw)*64),
// for the tiles jt in [jt0, jt1), it in [jt, nb).  Used twice per outer panel of 256 columns:
//   * "thin" (pkw = 1): after each inner 64-column step, bring the remaining columns of the outer panel
//     up to date (a few tile columns only);
//   * "trailing" (pkw = 4): ONE pass over the trailing matrix per 256 factored columns - a quarter of
//     the memory traffic of updating after every 64-column step (the update is memory-bound).
__global__ void __launch_bounds__(128) syrk_kernel(double* __restrict__ C, int ld, int pk0, int pkw, int jt0, int nb) {
    __shared__ GemmSmem sm;
    const int jt = jt0 + blockIdx.y;
    const int it = jt + blockIdx.x;
    if (it >= nb) return;
    const double* A = C + (size_t)it * 64 * ld + pk0 * 64;
    const double* B = C + (size_t)jt * 64 * ld + pk0 * 64;
    double acc[4][4][2] = {};
    gemm_tile_64<true>(acc, sm, A, ld, B, ld, 0, 64 * pkw);
    gemm_tile_store(acc, C + (size_t)it * 64 * ld + jt * 64, ld, -1.0, 1.0);
}

// ---------------------------------------------------------------------------
// K2b  triangular inverse by level doubling.  At level m (block size m = 64*2^s),
// pair p covers rows [r0, r0+m) (top) and [r0+m, r0+m+m2) (bottom), r0 = 2*p*m, m2 = min(mb, n_pad - r0 - m):
//     W21 = -W22 * (L21 * W11)
// step 1: T1 = L21 * W11   (W11 lower-triangular: k >= first column of the tile)
// step 2: W21 = -W22 * T1  (W22 lower-triangular: k <= last row of the tile)
// Level doubling passes mb = m; appended stations run one pair with the held rows on top (m = n0, mb = n_pad - n0).
__global__ void __launch_bounds__(128) trtri_step1_kernel(const double* __restrict__ L, const double* __restrict__ W,
                                                           double* __restrict__ T1, int ld, int n_pad, int m, int mb) {
    __shared__ GemmSmem sm;
    int r0 = 2 * blockIdx.z * m;
    int m2 = min(mb, n_pad - r0 - m);
    int ti = blockIdx.y, tj = blockIdx.x;
    if (m2 <= 0 || ti * 64 >= m2) return;
    const double* A = L + (size_t)(r0 + m + ti * 64) * ld + r0;        // L21 rows
    const double* B = W + (size_t)r0 * ld + r0 + tj * 64;              // W11 (NN), column tile tj
    double acc[4][4][2] = {};
    gemm_tile_64<false>(acc, sm, A, ld, B, ld, tj * 64, m);
    gemm_tile_store(acc, T1 + (size_t)(r0 + m + ti * 64) * ld + r0 + tj * 64, ld, 1.0, 0.0);
}

__global__ void __launch_bounds__(128) trtri_step2_kernel(double* __restrict__ W, const double* __restrict__ T1,
                                                           int ld, int n_pad, int m, int mb) {
    __shared__ GemmSmem sm;
    int r0 = 2 * blockIdx.z * m;
    int m2 = min(mb, n_pad - r0 - m);
    int ti = blockIdx.y, tj = blockIdx.x;
    if (m2 <= 0 || ti * 64 >= m2) return;
    const double* A = W + (size_t)(r0 + m + ti * 64) * ld + (r0 + m);  // W22 rows of tile ti
    const double* B = T1 + (size_t)(r0 + m) * ld + r0 + tj * 64;       // T1 (NN)
    double acc[4][4][2] = {};
    gemm_tile_64<false>(acc, sm, A, ld, B, ld, 0, ti * 64 + 64);
    gemm_tile_store(acc, W + (size_t)(r0 + m + ti * 64) * ld + r0 + tj * 64, ld, -1.0, 0.0);
}

// ---------------------------------------------------------------------------
// Gram product of the triangular inverse (LAPACK lauum): G = W^T W = C^-1 for W = L^-1, lower tiles only,
//     G_IJ = sum_{K >= I} W_KI^T W_KJ    (I >= J; W_KI = 0 for K < I, and the diagonal tiles of W are lower triangular)
// One CTA per lower tile, k over the rows [64 I, n_pad) of W in a fixed order (leave-group-out, DESIGN.md §5f).
__global__ void __launch_bounds__(128) gram_lower_kernel(const double* __restrict__ W, int ld, int n_pad,
                                                         double* __restrict__ G, int ldg) {
    __shared__ GemmSmem sm;
    const int tj = blockIdx.x, ti = blockIdx.y;
    if (tj > ti) return;
    double acc[4][4][2] = {};
    gemm_tile_64<false, true>(acc, sm, W + ti * 64, ld, W + tj * 64, ld, ti * 64, n_pad);
    gemm_tile_store(acc, G + (size_t)ti * 64 * ldg + tj * 64, ldg, 1.0, 0.0);
}

// ---------------------------------------------------------------------------
// Appended stations (kb200_append_data, DESIGN.md §5g): L21 = C21 W11^T, the new rows [n0, n_pad) of L from the held
// W11 of rows [0, n0). One 64x64 output tile (ti, tj) per CTA; W11[j][k] = 0 for k > j, so k stops at the end of the
// column tile. C21 and L21 point at the first new row, column 0.
__global__ void __launch_bounds__(128) append_l21_kernel(const double* __restrict__ C21, const double* __restrict__ W11,
                                                         double* __restrict__ L21, int ld) {
    __shared__ GemmSmem sm;
    const int tj = blockIdx.x, ti = blockIdx.y;
    double acc[4][4][2] = {};
    gemm_tile_64<true>(acc, sm, C21 + (size_t)ti * 64 * ld, ld, W11 + (size_t)tj * 64 * ld, ld, 0, (tj + 1) * 64);
    gemm_tile_store(acc, L21 + (size_t)ti * 64 * ld + tj * 64, ld, 1.0, 0.0);
}

// ---------------------------------------------------------------------------
// K2c  dual vectors.  Fz (n x na, column-major, column stride n_pad) holds the drift
// columns, the ones column and the data values.  Hz = W Fz ; Uz = W^T Hz = C^-1 Fz.
// Regional-linear columns are built on device from the adjusted coordinates
// (uk.py:877-883, uk3d.py:708-717) with an affine rescale (a change of drift basis,
// which leaves lambda, z and sigma^2 unchanged because the constant is in the span).
// values: nv columns (column-major, stride n) -> Fz columns K+1 .. K+nv
__global__ void build_fz_kernel(int n, int n_pad, int n_rl, int n_hd, int nv,
                                const double* __restrict__ ax, const double* __restrict__ ay,
                                const double* __restrict__ az,
                                DriftScale ds, const double* __restrict__ hd, const double* __restrict__ values,
                                double* __restrict__ Fz) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    int K = n_rl + n_hd;
    bool in = i < n;
    for (int c = 0; c < n_rl; ++c) {
        double v = c == 0 ? (in ? ax[i] : 0.0) : (c == 1 ? (in ? ay[i] : 0.0) : (in ? az[i] : 0.0));
        Fz[(size_t)c * n_pad + i] = in ? (v - ds.shift[c]) * ds.scale[c] : 0.0;
    }
    for (int c = 0; c < n_hd; ++c)
        Fz[(size_t)(n_rl + c) * n_pad + i] = in ? (hd[(size_t)c * n + i] - ds.shift[n_rl + c]) * ds.scale[n_rl + c] : 0.0;
    Fz[(size_t)K * n_pad + i] = in ? 1.0 : 0.0;
    for (int v = 0; v < nv; ++v) Fz[(size_t)(K + 1 + v) * n_pad + i] = in ? values[(size_t)v * n + i] : 0.0;
}

// Hz[i][c] = sum_{k<=i} W[i][k] Fz[k][c]   (one warp per row)
__global__ void __launch_bounds__(256) dual_h_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                      const double* __restrict__ Fz, double* __restrict__ Hz) {
    int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= n) return;
    double acc[KB_MAXAUX];
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) acc[c] = 0.0;
    const double* wr = W + (size_t)row * ld;
    for (int k = lane; k <= row; k += 32) {
        double w = wr[k];
#pragma unroll
        for (int c = 0; c < KB_MAXAUX; ++c)
            if (c < na) acc[c] += w * Fz[(size_t)c * n_pad + k];
    }
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) {
        if (c < na) {
            double v = acc[c];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) Hz[(size_t)c * n_pad + row] = v;
        }
    }
}

// Uz[k][c] = sum_{i>=k} W[i][k] Hz[i][c]   (block: 32 columns x 32 row slices; W is read ONCE for all na columns,
// four independent row loads in flight per thread: the kernel is a memory-bound pass over the lower triangle)
__global__ void __launch_bounds__(1024) dual_u_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                       const double* __restrict__ Hz, double* __restrict__ Uz) {
    __shared__ double red[32][33];
    const int kx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + kx;
    const int kfirst = blockIdx.x * 32;
    double acc[KB_MAXAUX];
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) acc[c] = 0.0;
    if (k < n) {
        int i = kfirst + ty;
        for (; i + 96 < n; i += 128) {
            double w[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { const int ii = i + 32 * u; w[u] = (ii >= k) ? W[(size_t)ii * ld + k] : 0.0; }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int ii = i + 32 * u;
#pragma unroll
                for (int c = 0; c < KB_MAXAUX; ++c) if (c < na) acc[c] = fma(w[u], Hz[(size_t)c * n_pad + ii], acc[c]);
            }
        }
        for (; i < n; i += 32) {
            if (i >= k) {
                const double w = W[(size_t)i * ld + k];
#pragma unroll
                for (int c = 0; c < KB_MAXAUX; ++c) if (c < na) acc[c] = fma(w, Hz[(size_t)c * n_pad + i], acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) {
        if (c < na) {                                   // na is uniform: every thread takes the same branches
            red[ty][kx] = acc[c];
            __syncthreads();
            if (ty == 0) {
                double v = 0.0;
#pragma unroll
                for (int q = 0; q < 32; ++q) v += red[q][kx];
                if (k < n_pad) Uz[(size_t)c * n_pad + k] = (k < n) ? v : 0.0;
            }
            __syncthreads();
        }
    }
}

// S = F^T U (K1 x K1), phi_v = F^T zeta_v (v < nv), S^-1 by Gauss-Jordan with partial pivoting.
// consts layout: [0 .. K1*K1) Sinv, then phi_0 .. phi_{nv-1}, K1 each. Singular S sets *flag = -1.
__global__ void __launch_bounds__(256) dual_small_kernel(int n, int n_pad, int K1, int nv,
                                                          const double* __restrict__ Fz, const double* __restrict__ Uz,
                                                          double* __restrict__ consts, int* __restrict__ flag) {
    __shared__ double red[256];
    __shared__ double S[16 * 17];
    const int tid = threadIdx.x;
    for (int a = 0; a < K1; ++a) {
        for (int b = 0; b < K1 + nv; ++b) {     // b >= K1 -> zeta columns
            double s = 0.0;
            for (int k = tid; k < n; k += 256) s += Fz[(size_t)a * n_pad + k] * Uz[(size_t)b * n_pad + k];
            red[tid] = s;
            __syncthreads();
            for (int o = 128; o > 0; o >>= 1) { if (tid < o) red[tid] += red[tid + o]; __syncthreads(); }
            if (tid == 0) { if (b < K1) S[a * 17 + b] = red[0]; else consts[K1 * K1 + (b - K1) * K1 + a] = red[0]; }
            __syncthreads();
        }
    }
    if (tid == 0) {
        double M[16][32];
        for (int a = 0; a < K1; ++a)
            for (int b = 0; b < K1; ++b) {
                M[a][b] = 0.5 * (S[a * 17 + b] + S[b * 17 + a]);
                M[a][K1 + b] = (a == b) ? 1.0 : 0.0;
            }
        bool bad = false;
        for (int c = 0; c < K1; ++c) {
            int p = c; double best = fabs(M[c][c]);
            for (int r = c + 1; r < K1; ++r) if (fabs(M[r][c]) > best) { best = fabs(M[r][c]); p = r; }
            if (!(best > 0.0)) { bad = true; break; }
            if (p != c) for (int q = 0; q < 2 * K1; ++q) { double t = M[c][q]; M[c][q] = M[p][q]; M[p][q] = t; }
            double inv = 1.0 / M[c][c];
            for (int q = 0; q < 2 * K1; ++q) M[c][q] *= inv;
            for (int r = 0; r < K1; ++r) if (r != c) {
                double f = M[r][c];
                if (f != 0.0) for (int q = 0; q < 2 * K1; ++q) M[r][q] -= f * M[c][q];
            }
        }
        if (bad) { if (*flag == 0) *flag = -1; }
        for (int a = 0; a < K1; ++a)
            for (int b = 0; b < K1; ++b) consts[a * K1 + b] = bad ? 0.0 : M[a][K1 + b];
    }
}

// ---------------------------------------------------------------------------
// K2d  pack: tile (row block I, k tile kt) -> 4096 values in the fp64 solve kernel's order: element (r, k) of the tile
//   lives at ((r/16)*4 + k/4)*64 + ((r%8)*4 + k%4)*2 + (r/8)%2, the m16n8k16 A-fragment order of common.cuh.
// rows < n: W (lower triangle); rows [n, n+na): dual rows Uz^T; other rows 0.
__device__ __forceinline__ void pack_rk(int I, int kt, int e, int& r, int& k) {
    // e = ((m16 tile * 4 + k/4) * 32 + lane) * 2 + (r/8)%2, lane = (r%8)*4 + k%4
    const int h = e & 1, lane = (e >> 1) & 31, k4 = (e >> 6) & 3, mt = e >> 8;
    r = I * KB_BM + mt * 16 + 8 * h + (lane >> 2);
    k = kt * KB_BK + k4 * 4 + (lane & 3);
}
__global__ void __launch_bounds__(256) pack_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                    const double* __restrict__ Uz, PackMap pm, double* __restrict__ out) {
    int I = blockIdx.y, kt = blockIdx.x;
    if (kt >= pm.ktiles[I]) return;
    double* o = out + ((size_t)pm.tile_off[I] + kt) * (KB_BM * KB_BK);
    for (int e = threadIdx.x; e < KB_BM * KB_BK; e += 256) {
        int r, k;
        pack_rk(I, kt, e, r, k);
        double v = 0.0;
        if (r < n) { if (k <= r) v = W[(size_t)r * ld + k]; }
        else if (r < n + na) { if (k < n) v = Uz[(size_t)(r - n) * n_pad + k]; }
        o[e] = v;
    }
}

// ---------------------------------------------------------------------------
// host-side launchers
cudaError_t kbk_adjust_data(int dim, const Aniso& an, int n, const double* x, const double* y, const double* z,
                            double* ax, double* ay, double* az, cudaStream_t st) {
    return KbDims::dispatch(dim, [&](auto D) {
        adjust_data_kernel<D><<<(n + 255) / 256, 256, 0, st>>>(an, n, x, y, z, ax, ay, az);
        return cudaGetLastError();
    });
}

cudaError_t kbk_assemble(int dim, const VgParams& vg, int n, int n_pad, int ld, int it0,
                         const double* ax, const double* ay, const double* az, double* C, cudaStream_t st) {
    const int nb = n_pad / 64;
    return KbDims::dispatch(dim, [&](auto D) {
        return KbModels::dispatch(vg.model, [&](auto M) {
            const int tiles = nb * (nb + 1) / 2 - it0 * (it0 + 1) / 2;
            assemble_kernel<D, M><<<tiles, 256, 0, st>>>(vg, n, ld, it0, ax, ay, az, C);
            return cudaGetLastError();
        });
    });
}

cudaError_t kbk_factor_init() {
    return cudaFuncSetAttribute(panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PN_SMEM);
}

// Blocked right-looking Cholesky with one level of look-ahead. Outer panels of OW = 4 block columns (256 columns):
//   panel(ob)   four fused panel steps (left-looking inside the outer panel)            -> side stream `hi`
//   T_look(ob)  update of the NEXT outer panel's columns with this panel (k = 256)        -> side stream `hi`
//   T_rest(ob)  update of everything to the right of the next panel (k = 256): the bulk
//               of the flops, one pass over the trailing matrix per 256 factored columns  -> main stream `st`
// panel(ob+1) and T_look(ob) depend only on T_look / T_rest of earlier panels, so the latency-bound panel chain runs on
// the high-priority stream `hi` UNDER the DMMA-bound trailing update of the previous panel. Events (ev[0..2*nob)) order
// the read-modify-write passes over shared regions:
//   T_look(ob) after T_rest(ob-1);  T_rest(ob) after panel(ob).
// The diagonal-block inverses land in W's diagonal blocks (input of kbk_inverse_rows).
static cudaError_t cholesky(double* C, double* W, double* Lstage, int ld, int n_pad, int* flag, double dtol, cudaStream_t st,
                            cudaStream_t hi, cudaEvent_t* ev, int n_ev, int* launches) {
    const int nb = n_pad / 64;
    const int OW = 4;
    const int nob = (nb + OW - 1) / OW;
    if (2 * nob + 1 > n_ev) return cudaErrorInvalidValue;
    cudaEvent_t* evP = ev;               // panel(ob) complete            (recorded on hi)
    cudaEvent_t* evR = ev + nob;         // T_rest(ob) complete           (recorded on st)
    KB_CUDA_OK(cudaEventRecord(ev[2 * nob], st));                 // everything before (assemble) precedes the panel chain
    KB_CUDA_OK(cudaStreamWaitEvent(hi, ev[2 * nob], 0));
    for (int ob = 0, o = 0; ob < nb; ob += OW, ++o) {
        const int oe = ob + OW < nb ? ob + OW : nb;     // end of the outer panel (tile units)
        for (int kb = ob; kb < oe; ++kb) {
            panel_kernel<<<nb - kb, 256, PN_SMEM, hi>>>(C, W, Lstage, ld, kb, ob, flag, dtol);
            ++*launches;
        }
        KB_CUDA_OK(cudaEventRecord(evP[o], hi));
        if (oe < nb) {
            const int le = oe + OW < nb ? oe + OW : nb; // end of the look-ahead columns
            if (o > 0) KB_CUDA_OK(cudaStreamWaitEvent(hi, evR[o - 1], 0));
            {
                dim3 g(nb - oe, le - oe);
                syrk_kernel<<<g, 128, 0, hi>>>(C, ld, ob, oe - ob, oe, nb);
                ++*launches;
            }
            KB_CUDA_OK(cudaStreamWaitEvent(st, evP[o], 0));
            if (le < nb) {
                dim3 g(nb - le, nb - le);
                syrk_kernel<<<g, 128, 0, st>>>(C, ld, ob, oe - ob, le, nb);
                ++*launches;
            }
            KB_CUDA_OK(cudaEventRecord(evR[o], st));
        } else {
            KB_CUDA_OK(cudaStreamWaitEvent(st, evP[o], 0));      // join: the main stream continues after the last panel
        }
    }
    diag_writeback_kernel<<<nb, 256, 0, st>>>(C, Lstage, ld);
    ++*launches;
    return cudaGetLastError();
}

// Rows [n0, n_pad) of L and W from the held L11 (in C) and W11 = L11^-1 of rows [0, n0); n0 = 0 factors all of C:
//   kbk_cholesky_rows  L21 = C21 W11^T, S = C22 - L21 L21^T, L22 = chol(S)      (the Cholesky above, on the corner)
//   kbk_inverse_rows   W22 = L22^-1 (level doubling on the corner), W21 = -W22 (L21 W11): one more doubling step whose
//                      top block is the n0 held rows
// T is scratch of C's shape. L21 goes there first (its tiles read whole rows of C21), then into C21 for the Schur
// update; afterwards T holds the corner's staged diagonal factors, then T1 of the inverse.
cudaError_t kbk_cholesky_rows(double* C, double* W, double* T, int ld, int n_pad, int n0, int* flag, double dtol,
                              cudaStream_t st, cudaStream_t hi, cudaEvent_t* ev, int n_ev, int* launches) {
    const int nb0 = n0 / 64, nb = n_pad / 64;
    const size_t r0 = (size_t)n0 * ld;
    if (nb0 > 0) {
        append_l21_kernel<<<dim3(nb0, nb - nb0), 128, 0, st>>>(C + r0, W, T + r0, ld);
        KB_CUDA_OK(cudaMemcpy2DAsync(C + r0, (size_t)ld * 8, T + r0, (size_t)ld * 8, (size_t)n0 * 8, n_pad - n0,
                                     cudaMemcpyDeviceToDevice, st));
        syrk_kernel<<<dim3(nb - nb0, nb - nb0), 128, 0, st>>>(C, ld, 0, nb0, nb0, nb);
        *launches += 2;
    }
    return cholesky(C + r0 + n0, W + r0 + n0, T, ld, n_pad - n0, flag, dtol, st, hi, ev, n_ev, launches);
}

cudaError_t kbk_inverse_rows(const double* L, double* W, double* T, int ld, int n_pad, int n0, cudaStream_t st,
                             int* launches) {
    const size_t c0 = (size_t)n0 * ld + n0;
    const int nc = n_pad - n0;
    for (int m = 64; m < nc; m *= 2) {
        dim3 grid(m / 64, m / 64, (nc + 2 * m - 1) / (2 * m));
        trtri_step1_kernel<<<grid, 128, 0, st>>>(L + c0, W + c0, T + c0, ld, nc, m, m);
        trtri_step2_kernel<<<grid, 128, 0, st>>>(W + c0, T + c0, ld, nc, m, m);
        *launches += 2;
    }
    if (n0 > 0) {
        dim3 grid(n0 / 64, nc / 64, 1);
        trtri_step1_kernel<<<grid, 128, 0, st>>>(L, W, T, ld, n_pad, n0, nc);
        trtri_step2_kernel<<<grid, 128, 0, st>>>(W, T, ld, n_pad, n0, nc);
        *launches += 2;
    }
    return cudaGetLastError();
}

cudaError_t kbk_gram_lower(const double* W, int ld, int n_pad, double* G, int ldg, cudaStream_t st) {
    const int nb = n_pad / 64;
    gram_lower_kernel<<<dim3(nb, nb), 128, 0, st>>>(W, ld, n_pad, G, ldg);
    return cudaGetLastError();
}

// The dual kernels keep KB_MAXAUX accumulators per thread in registers: more columns (value fields) run as further
// launches over column chunks of KB_MAXAUX. Every column's arithmetic is the same in whichever chunk it lands.
cudaError_t kbk_dual(const double* W, int ld, int n, int n_pad, int n_rl, int n_hd, int nv,
                     const double* ax, const double* ay, const double* az, const DriftScale& ds,
                     const double* hd, const double* values,
                     double* Fz, double* Hz, double* Uz, double* consts, int* flag, cudaStream_t st, int* launches) {
    int K1 = n_rl + n_hd + 1, na = K1 + nv;
    build_fz_kernel<<<(n_pad + 255) / 256, 256, 0, st>>>(n, n_pad, n_rl, n_hd, nv, ax, ay, az, ds, hd, values, Fz);
    for (int c0 = 0; c0 < na; c0 += KB_MAXAUX) {
        const int nc = na - c0 < KB_MAXAUX ? na - c0 : KB_MAXAUX;
        const size_t o = (size_t)c0 * n_pad;
        dual_h_kernel<<<(n + 7) / 8, 256, 0, st>>>(W, ld, n, n_pad, nc, Fz + o, Hz + o);
        dual_u_kernel<<<(n_pad + 31) / 32, 1024, 0, st>>>(W, ld, n, n_pad, nc, Hz + o, Uz + o);
        *launches += 2;
    }
    dual_small_kernel<<<1, 256, 0, st>>>(n, n_pad, K1, nv, Fz, Uz, consts, flag);
    *launches += 2;
    return cudaGetLastError();
}

cudaError_t kbk_build_fz(int n, int n_pad, int n_rl, int n_hd, const double* ax, const double* ay, const double* az,
                         const DriftScale& ds, const double* hd, const double* values, double* Fz, cudaStream_t st) {
    build_fz_kernel<<<(n_pad + 255) / 256, 256, 0, st>>>(n, n_pad, n_rl, n_hd, 1, ax, ay, az, ds, hd, values, Fz);
    return cudaGetLastError();
}

cudaError_t kbk_pack(const double* W, int ld, int n, int n_pad, int na, const double* Uz,
                     const PackMap& pm, void* out, cudaStream_t st) {
    pack_kernel<<<kb_pack_grid(pm), 256, 0, st>>>(W, ld, n, n_pad, na, Uz, pm, (double*)out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// General fallback when C is not positive definite (a variogram that is not conditionally negative
// definite in the working dimension, e.g. hole-effect on dense 2-D scatter; the reference's LU still
// inverts such systems, ok.py:663): in-place Gauss-Jordan inversion with partial pivoting, blocked by 64 columns
// ("Blocked Gauss-Jordan" below), followed by the column swaps in reverse order. The result G = C^-1 is then used in
// the quadratic-form variant of the solve kernel (q = c^T G c through the lower triangle with doubled
// off-diagonals, DESIGN.md §3b).
__global__ void gj_colswap_kernel(double* __restrict__ A, int ld, int n, const int* __restrict__ piv) {
    // one thread per row: apply the recorded swaps as column swaps in reverse order
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double* row = A + (size_t)i * ld;
    for (int k = n - 1; k >= 0; --k) {
        int p = piv[k];
        if (p != k) { double t = row[k]; row[k] = row[p]; row[p] = t; }
    }
}

// Uz[i][c] = sum_k G[i][k] Fz[k][c]  (full symmetric G; one warp per row)
__global__ void __launch_bounds__(256) dual_g_kernel(const double* __restrict__ G, int ld, int n, int n_pad, int na,
                                                      const double* __restrict__ Fz, double* __restrict__ Uz) {
    int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= n_pad) return;
    double acc[KB_MAXAUX];
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) acc[c] = 0.0;
    if (row < n) {
        const double* gr = G + (size_t)row * ld;
        for (int k = lane; k < n; k += 32) {
            double w = gr[k];
#pragma unroll
            for (int c = 0; c < KB_MAXAUX; ++c)
                if (c < na) acc[c] += w * Fz[(size_t)c * n_pad + k];
        }
    }
#pragma unroll
    for (int c = 0; c < KB_MAXAUX; ++c) {
        if (c < na) {
            double v = acc[c];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) Uz[(size_t)c * n_pad + row] = v;
        }
    }
}

// pack for the quadratic-form variant: T = lower triangle of the symmetrised G with doubled off-diagonals
__global__ void __launch_bounds__(256) pack_gform_kernel(const double* __restrict__ G, int ld, int n, int n_pad, int na,
                                                          const double* __restrict__ Uz, PackMap pm,
                                                          double* __restrict__ out) {
    int I = blockIdx.y, kt = blockIdx.x;
    if (kt >= pm.ktiles[I]) return;
    double* o = out + ((size_t)pm.tile_off[I] + kt) * (KB_BM * KB_BK);
    for (int e = threadIdx.x; e < KB_BM * KB_BK; e += 256) {
        int r, k;
        pack_rk(I, kt, e, r, k);                 // fp64 solve kernel order, as pack_kernel
        double v = 0.0;
        if (r < n) {
            if (k < r) v = G[(size_t)r * ld + k] + G[(size_t)k * ld + r];
            else if (k == r) v = G[(size_t)r * ld + r];
        } else if (r < n + na) { if (k < n) v = Uz[(size_t)(r - n) * n_pad + k]; }
        o[e] = v;
    }
}

// full symmetric assemble for the fallback (upper tiles too): mirror the lower triangle
__global__ void symmetrize_kernel(double* __restrict__ C, int ld, int n_pad) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    int i = blockIdx.y;
    if (j < n_pad && j > i) C[(size_t)i * ld + j] = C[(size_t)j * ld + i];
}

// ---------------------------------------------------------------------------
// Blocked Gauss-Jordan. 64 consecutive column steps of the elimination (step k: pivot search in column k, row swap,
// scaling of the pivot row, a[i][j] -= a[i][k] a[k][j] for i != k) compose into the block exchange of the pivot block K
// against the rest R (after the row swaps):
//     A_KK <- A_KK^-1,  A_RK <- -A_RK A_KK^-1,  A_KR <- A_KK^-1 A_KR,  A_RR <- A_RR - A_RK A_KK^-1 A_KR
// (tests/test_host.py::test_blocked_gauss_jordan_algebra pins this against the column steps in numpy), so one 64-column
// step is
//   gj_panel_kernel      the 64 column steps with partial pivoting restricted to the n_pad x 64 column panel. The rows
//                        are dealt to the CTAs of ONE cooperative grid, each CTA keeps its rows of the panel in shared
//                        memory; per step every CTA publishes its best pivot candidate (|value|, row index, the row's 64
//                        panel entries) and the owner of row k publishes that row, ONE grid barrier, then every CTA
//                        picks the same winner, swaps and eliminates locally. Double-buffered slots: the barrier of step
//                        j+1 separates the reads of step j from the writes of step j+2.
//   gj_swap_copy_kernel  the recorded row swaps on all other columns, then T = A[K rows][other columns] to a buffer
//   gj_gemm_kernel       A[:, other] = (rows K: 0, else A[:, other]) + Panel * T   -- rank-64 update on the DMMA pipe
// i.e. 3 launches and 64 grid barriers per 64 columns. The padded rows/columns (identity) take part, so every block is
// full. A pivot at or below ptol is reported as singular: ptol is rounding noise, as the pivot row is scaled, so a
// redundant row cancels to ~1 ulp, not 0.
#define GJ_PLD 65
#define GJ_MAX_CTAS 256

struct GjWork {
    double* Tbuf;       // [64][n_pad]
    double* cand_row;   // [2][GJ_MAX_CTAS][64]
    double* krow;       // [2][64]
    double* cand_val;   // [2][GJ_MAX_CTAS]
    int* cand_idx;      // [2][GJ_MAX_CTAS]
    int* piv;           // [n_pad]
};

size_t kbk_general_inverse_workspace_bytes(int n_pad) {
    size_t d = (size_t)64 * n_pad + 2 * GJ_MAX_CTAS * 64 + 128 + 2 * GJ_MAX_CTAS;
    return d * sizeof(double) + (2 * GJ_MAX_CTAS + (size_t)n_pad + 64) * sizeof(int);
}

static GjWork gj_carve(void* work, int n_pad) {
    GjWork w;
    double* d = reinterpret_cast<double*>(work);
    w.Tbuf = d; d += (size_t)64 * n_pad;
    w.cand_row = d; d += 2 * GJ_MAX_CTAS * 64;
    w.krow = d; d += 128;
    w.cand_val = d; d += 2 * GJ_MAX_CTAS;
    int* i = reinterpret_cast<int*>(d);
    w.cand_idx = i; i += 2 * GJ_MAX_CTAS;
    w.piv = i;
    return w;
}

static size_t gj_panel_smem(int rpc) { return ((size_t)rpc * (GJ_PLD + 1) + 3 * 64) * sizeof(double); }

// candidates (|v|, row): larger |v| wins, ties go to the lower row index (the first maximum, as LAPACK's getrf)
__device__ __forceinline__ bool gj_better(double v, int i, double bv, int bi) { return v > bv || (v == bv && i < bi); }

__global__ void __launch_bounds__(256) gj_panel_kernel(double* A, int ld, int n_pad, int k0, int rpc,
                                                        double* cand_row, double* krow, double* cand_val, int* cand_idx,
                                                        int* __restrict__ piv, int* flag, double ptol) {
    cg::grid_group grid = cg::this_grid();
    extern __shared__ double gj_sm[];
    double* P = gj_sm;                          // [rpc][GJ_PLD]: this CTA's rows of the panel
    double* colv = P + (size_t)rpc * GJ_PLD;    // [rpc]  column j before the step
    double* prow = colv + rpc;                  // [64]   pivot row
    double* kr = prow + 64;                     // [64]   row k before the swap
    double* rv = kr + 64;                       // [64]   scaled pivot row
    __shared__ double s_val[8];
    __shared__ int s_idx[8];
    __shared__ int s_win[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    const int row0 = cta * rpc;
    const int R = max(0, min(rpc, n_pad - row0));
    for (int e = tid; e < R * 64; e += 256) {
        const int r = e >> 6, c = e & 63;
        P[r * GJ_PLD + c] = A[(size_t)(row0 + r) * ld + k0 + c];
    }
    __syncthreads();
    for (int j = 0; j < 64; ++j) {
        const int kk = k0 + j, par = j & 1;
        // (1) this CTA's candidate among its rows >= kk
        double best = -1.0; int bi = 0x7fffffff;
        for (int r = tid; r < R; r += 256) {
            const int g = row0 + r;
            if (g >= kk) {
                const double v = fabs(P[r * GJ_PLD + j]);
                if (gj_better(v, g, best, bi)) { best = v; bi = g; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (gj_better(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) { s_val[warp] = best; s_idx[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            best = lane < 8 ? s_val[lane] : -1.0;
            bi = lane < 8 ? s_idx[lane] : 0x7fffffff;
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (gj_better(ov, oi, best, bi)) { best = ov; bi = oi; }
            }
            if (lane == 0) { s_val[0] = best; s_idx[0] = bi; }
        }
        __syncthreads();
        best = s_val[0]; bi = s_idx[0];
        // (2) publish: candidate (+ its panel row), and row kk by its owner
        if (tid == 0) { __stcg(&cand_val[par * G + cta], best); __stcg(&cand_idx[par * G + cta], bi); }
        if (best >= 0.0 && tid < 64) __stcg(&cand_row[((size_t)(par * G + cta)) * 64 + tid], P[(bi - row0) * GJ_PLD + tid]);
        if (kk >= row0 && kk < row0 + R && tid >= 64 && tid < 128)
            __stcg(&krow[par * 64 + tid - 64], P[(kk - row0) * GJ_PLD + tid - 64]);
        grid.sync();
        // (3) every CTA picks the same winner (L1 is bypassed: the slots are rewritten every other step)
        if (warp == 0) {
            double bv = -1.0; int bx = 0x7fffffff, bc = 0;
            for (int c = lane; c < G; c += 32) {
                const double v = __ldcg(&cand_val[par * G + c]);
                const int ix = __ldcg(&cand_idx[par * G + c]);
                if (gj_better(v, ix, bv, bx)) { bv = v; bx = ix; bc = c; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bx, o);
                const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
                if (gj_better(ov, oi, bv, bx)) { bv = ov; bx = oi; bc = oc; }
            }
            if (lane == 0) {
                if (bx == 0x7fffffff) {             // no comparable candidate at all (NaN in the data): report, keep indices sane
                    bx = kk;
                    if (cta == 0 && *flag == 0) *flag = 1 + kk;
                }
                s_win[0] = bc; s_win[1] = bx;
            }
        }
        __syncthreads();
        const int wc = s_win[0], p = s_win[1];
        if (tid < 64) {
            prow[tid] = __ldcg(&cand_row[((size_t)(par * G + wc)) * 64 + tid]);
            kr[tid] = __ldcg(&krow[par * 64 + tid]);
        }
        __syncthreads();
        const double d0 = prow[j];
        double d = d0;
        if (!(fabs(d) > 0.0)) d = 1.0;
        const double inv = 1.0 / d;
        if (cta == 0 && tid == 0) {
            piv[kk] = p;
            if (!(fabs(d0) > ptol) && *flag == 0) *flag = 1 + kk;
        }
        if (tid < 64) rv[tid] = (tid == j) ? inv : prow[tid] * inv;
        // (4) swap rows kk <-> p inside the panel
        if (p != kk) {
            if (p >= row0 && p < row0 + R && tid < 64) P[(p - row0) * GJ_PLD + tid] = kr[tid];
            if (kk >= row0 && kk < row0 + R && tid >= 64 && tid < 128) P[(kk - row0) * GJ_PLD + tid - 64] = prow[tid - 64];
        }
        __syncthreads();
        for (int r = tid; r < R; r += 256) colv[r] = P[r * GJ_PLD + j];
        __syncthreads();
        // (5) column step kk on this CTA's rows: row kk becomes the scaled pivot row, column j the negated multipliers
        for (int e = tid; e < R * 64; e += 256) {
            const int r = e >> 6, c = e & 63;
            double v;
            if (row0 + r == kk) v = rv[c];
            else {
                const double cv = colv[r];
                v = (c == j) ? -(cv * inv) : P[r * GJ_PLD + c] - cv * rv[c];
            }
            P[r * GJ_PLD + c] = v;
        }
        __syncthreads();
    }
    for (int e = tid; e < R * 64; e += 256) {
        const int r = e >> 6, c = e & 63;
        A[(size_t)(row0 + r) * ld + k0 + c] = P[r * GJ_PLD + c];
    }
}

// one thread per column outside the panel: the 64 row swaps in order, then the K rows of that column to Tbuf
__global__ void __launch_bounds__(256) gj_swap_copy_kernel(double* __restrict__ A, int ld, int n_pad, int k0,
                                                            const int* __restrict__ piv, double* __restrict__ Tbuf) {
    __shared__ int sp[64];
    if (threadIdx.x < 64) sp[threadIdx.x] = piv[k0 + threadIdx.x];
    __syncthreads();
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= n_pad || (c >= k0 && c < k0 + 64)) return;
    for (int j = 0; j < 64; ++j) {
        const int p = sp[j], kk = k0 + j;
        if (p != kk) {
            const double t = A[(size_t)kk * ld + c];
            A[(size_t)kk * ld + c] = A[(size_t)p * ld + c];
            A[(size_t)p * ld + c] = t;
        }
    }
    for (int j = 0; j < 64; ++j) Tbuf[(size_t)j * n_pad + c] = A[(size_t)(k0 + j) * ld + c];
}

__global__ void __launch_bounds__(128) gj_gemm_kernel(double* C, int ld, int n_pad, int kb, const double* __restrict__ Tbuf) {
    __shared__ GemmSmem sm;
    const int J = blockIdx.x, I = blockIdx.y;
    if (J == kb) return;
    const double* A = C + (size_t)I * 64 * ld + (size_t)kb * 64;     // this row block of the panel
    const double* B = Tbuf + (size_t)J * 64;                         // T[0..64)[J columns], row stride n_pad
    double acc[4][4][2] = {};
    gemm_tile_64<false>(acc, sm, A, ld, B, n_pad, 0, 64);
    gemm_tile_store(acc, C + (size_t)I * 64 * ld + (size_t)J * 64, ld, 1.0, I == kb ? 0.0 : 1.0);
}

// grid of the panel kernel: rows per CTA and CTA count, 0 if the device cannot co-schedule it
static int gj_plan(int n_pad, int* rpc_out) {
    int dev = 0, sms = 0, coop = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if (!coop || sms <= 0) return 0;
    int max_ctas = sms < GJ_MAX_CTAS ? sms : GJ_MAX_CTAS;
    int rpc = (n_pad + max_ctas - 1) / max_ctas;
    if (rpc < 32) rpc = 32;
    const size_t smem = gj_panel_smem(rpc);
    if (smem > 227 * 1024) return 0;
    if (cudaFuncSetAttribute(gj_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 0;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gj_panel_kernel, 256, smem) != cudaSuccess || per_sm < 1) return 0;
    *rpc_out = rpc;
    return (n_pad + rpc - 1) / rpc;
}

cudaError_t kbk_general_inverse(double* C, int ld, int n_pad, void* work, int* flag, double ptol,
                                cudaStream_t st, int* launches) {
    // C holds the assembled lower triangle (+ diagonal, identity in the padding); build the full matrix, then invert
    int rpc = 0;
    const int G = gj_plan(n_pad, &rpc);
    if (G == 0) return cudaErrorNotSupported;
    GjWork w = gj_carve(work, n_pad);
    symmetrize_kernel<<<dim3((n_pad + 255) / 256, n_pad), 256, 0, st>>>(C, ld, n_pad);
    ++*launches;
    const int nbk = n_pad / 64;
    const size_t smem = gj_panel_smem(rpc);
    for (int kb = 0; kb < nbk; ++kb) {
        int k0 = kb * 64;
        void* args[] = {&C, &ld, &n_pad, &k0, &rpc, &w.cand_row, &w.krow, &w.cand_val, &w.cand_idx, &w.piv, &flag, &ptol};
        KB_CUDA_OK(cudaLaunchCooperativeKernel((const void*)gj_panel_kernel, dim3(G), dim3(256), args, smem, st));
        ++*launches;
        if (nbk > 1) {
            gj_swap_copy_kernel<<<(n_pad + 255) / 256, 256, 0, st>>>(C, ld, n_pad, k0, w.piv, w.Tbuf);
            gj_gemm_kernel<<<dim3(nbk, nbk), 128, 0, st>>>(C, ld, n_pad, kb, w.Tbuf);
            *launches += 2;
        }
    }
    gj_colswap_kernel<<<(n_pad + 127) / 128, 128, 0, st>>>(C, ld, n_pad, w.piv);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t kbk_dual_gform(const double* G, int ld, int n, int n_pad, int n_rl, int n_hd, int nv,
                           const double* ax, const double* ay, const double* az, const DriftScale& ds,
                           const double* hd, const double* values,
                           double* Fz, double* Uz, double* consts, int* flag, cudaStream_t st, int* launches) {
    int K1 = n_rl + n_hd + 1, na = K1 + nv;
    build_fz_kernel<<<(n_pad + 255) / 256, 256, 0, st>>>(n, n_pad, n_rl, n_hd, nv, ax, ay, az, ds, hd, values, Fz);
    for (int c0 = 0; c0 < na; c0 += KB_MAXAUX) {      // column chunks, as kbk_dual
        const int nc = na - c0 < KB_MAXAUX ? na - c0 : KB_MAXAUX;
        const size_t o = (size_t)c0 * n_pad;
        dual_g_kernel<<<(n_pad + 7) / 8, 256, 0, st>>>(G, ld, n, n_pad, nc, Fz + o, Uz + o);
        *launches += 1;
    }
    dual_small_kernel<<<1, 256, 0, st>>>(n, n_pad, K1, nv, Fz, Uz, consts, flag);
    *launches += 2;
    return cudaGetLastError();
}

cudaError_t kbk_pack_gform(const double* G, int ld, int n, int n_pad, int na, const double* Uz,
                           const PackMap& pm, void* out, cudaStream_t st) {
    pack_gform_kernel<<<kb_pack_grid(pm), 256, 0, st>>>(G, ld, n, n_pad, na, Uz, pm, (double*)out);
    return cudaGetLastError();
}
