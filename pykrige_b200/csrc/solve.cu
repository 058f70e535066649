// solve.cu — K3: the per-grid-point hot kernel of the global kriging path (fp64 DMMA), finalize fused.
//
// Reference semantics (ok.py:665-681, uk.py:942-1007): for every prediction point j
//     b_j = [-gamma(|p_j - x_k|) (0 on an exact hit) ; drift(p_j) ; 1],  x_j = A^-1 b_j,
//     z_j = x_j[:n] . Z,   sigma2_j = -x_j . b_j .
// Here (DESIGN.md §3), with c_j = c0 + b_j[:n] and W = chol(C)^-1:
//     q_j  = || W c_j ||^2            <- the O(n^2) contraction, a triangular GEMM on the fp64 tensor pipe
//     g_j  = U^T c_j, zc_j = zeta . c_j   <- extra dense "dual rows" appended to W (same GEMM)
//     finalize: r = g - f_j, mu = S^-1 r, sigma2 = c0 - q + r.mu, z = zc - mu.phi
//
// Kernels in this file (all fp64, mma.sync.m8n8k4 = SASS DMMA):
//   solve_kernel_pt   (K3 v3, the product path) persistent CTAs, one CTA = 64 points x all rows of W, RHS column
//                     block generated once per tile, W/RHS tiles streamed by cp.async.bulk + mbarrier, fused
//                     finalize. See the comment above the kernel.
// The wgmma variants live in solve_tf32.cu (dtype float32) and solve_i8.cu (dtype float64x).
#include "common.cuh"
#include "kernels.h"
#include <cstdlib>

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    // bounded spin: a lost transaction traps instead of hanging the GPU
    for (uint32_t it = 0; it < (1u << 26); ++it)
        if (mbar_try_wait(bar, parity)) return;
    __trap();
}
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------------------------------------
// K3 v3: persistent, warp-specialised, one CTA = one tile of 64 prediction points x ALL rows of W.
//
// v1 (one CTA per (row block, point tile)) regenerates every RHS tile once per row block - a 10x
// recompute of sqrt+exp at N=5000 - and alternates generation with the tensor work (measured: DMMA pipe
// 54 % active). v2 (warp-specialised but still regenerating) was slower: four producer warps cannot
// hide the fp64 sqrt/exp latency. v3 removes the recompute instead:
//   phase G  all 12 warps evaluate the RHS column block c[k][j] of the tile ONCE (n x 64 values) and
//            park it, already in MMA-fragment order, in a per-CTA scratch ring (L2-resident, re-used for
//            every tile the CTA processes; size independent of M);
//   phase M  warp 0 streams W tiles (32 KB) and RHS tiles (8 KB) with cp.async.bulk + mbarrier into a
//            4-stage ring; warps 4..11 do nothing but LDS + DMMA, walking all row blocks and keeping the
//            per-point sum of squares in registers;
//   phase F  the (K+1)x(K+1) drift solve and the two outputs per point are produced in the same CTA:
//            no partial buffers, no separate finalize pass, fixed summation order (deterministic).
#define PT_STAGES 5
#define PT_THREADS 384
#define PT_STAGE_BYTES ((KB_BM * KB_BK + KB_BK * KB_TN) * 8)

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(smem_u32(bar)) : "memory");
}

// NT = n-tiles (of 8 points) per point tile: 8 (64 points) is the default. Narrower tiles (NT = 4, 2: 32 / 16 points) are used by
// the host for the TAIL of a launch: the points left over after the last full round of 64-point tiles would keep only a few of
// the persistent CTAs (one per SM) busy for a whole tile time (1953 tiles on 132 SMs = 14.8 rounds at 125 000 points per
// GPU); as narrow tiles they spread over all SMs and a tile costs little more than streaming W once. The per-point arithmetic
// does not depend on NT (tests/test_parity_gpu.py::test_tile_width_is_invisible).
template <int DIM, int MODEL, int NT>
__global__ void __launch_bounds__(PT_THREADS, 1) solve_kernel_pt(const __grid_constant__ SolvePtParams P) {
    constexpr int TN = NT * 8;                                          // points per tile
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* Ts = reinterpret_cast<double*>(smem_raw);                   // PT_STAGES * BM*BK
    double* Bs = Ts + PT_STAGES * KB_BM * KB_BK;                        // PT_STAGES * BK*TN
    double* qred = Bs + PT_STAGES * KB_BK * TN;                      // 8 * 64
    double* auxs = qred + 8 * TN;                                    // KB_MAXAUX * 64
    uint64_t* full = reinterpret_cast<uint64_t*>(auxs + KB_MAXAUX * TN);   // PT_STAGES
    uint64_t* empty = full + PT_STAGES;                                 // PT_STAGES

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nk = (P.n + KB_BK - 1) / KB_BK;                           // k tiles of a full column block
    double* scratch = P.scratch + (size_t)blockIdx.x * nk * (KB_BK * TN);
    const double* gt = reinterpret_cast<const double*>(P.tiles);
    const long long ntiles = (P.m + TN - 1) / TN;

    if (tid == 0) {
        for (int s = 0; s < PT_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    }
    __syncthreads();

    uint32_t git = 0;                 // running stage counter (same sequence in producer and consumers)
    const int cw = warp - 4;          // consumer warp 0..7

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        // ---------------- phase G: RHS column block of this tile, once ----------------
        {
            const int pl = tid % TN;                 // point within the tile
            const int ks = tid / TN;                 // k-tile slice (6 slices at 64 points, 8 at 48)
            const long long pj = tile * TN + pl;
            const bool pvalid = pj < P.m;
            double px = 0.0, py = 0.0, pz = 0.0;
            if (pvalid) kb_load_point<DIM>(P.ps, P.an, pj, px, py, pz);
            for (int t = ks; t < nk; t += PT_THREADS / TN) {
                double* bt = scratch + (size_t)t * (KB_BK * TN);
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) {
                    double v[4];
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const int k = t * KB_BK + k4 * 4 + kk;
                        double val = 0.0;
                        if (pvalid && k < P.n) {
                            double d = kb_dist<DIM>(__ldg(P.ax + k), __ldg(P.ay + k), KB_HASZ(DIM) ? __ldg(P.az + k) : 0.0,
                                                    px, py, pz);
                            val = kb_cov_rhs<MODEL>(P.vg, d);
                        }
                        v[kk] = val;
                    }
                    // fragment order ((k4*NT + n/8)*32 + (n%8)*4 + k%4): 4 consecutive k = 32 contiguous bytes
                    double2* dst = reinterpret_cast<double2*>(bt + (k4 * NT + (pl >> 3)) * 32 + (pl & 7) * 4);
                    dst[0] = make_double2(v[0], v[1]);
                    dst[1] = make_double2(v[2], v[3]);
                }
            }
            // generic-proxy global writes -> later read by the async proxy (bulk copies) of this CTA
            __threadfence();
            asm volatile("fence.proxy.async.global;\n" ::: "memory");
        }
        __syncthreads();

        // ---------------- phase M ----------------
        if (warp == 0) {
            if (lane == 0) {
                uint32_t g = git;
                const uint64_t pol_w = kb_policy_evict_last(), pol_c = kb_policy_evict_first();
                long long tau = 0;                   // W tiles are stored contiguously in (I, t) order
                for (int I = 0; I < P.nrb; ++I) {
                    const int kt = P.pm.ktiles[I];
                    for (int t = 0; t < kt; ++t, ++tau, ++g) {
                        const int s = g % PT_STAGES;
                        mbar_wait(&empty[s], (uint32_t)(((g / PT_STAGES) & 1) ^ 1));
                        mbar_expect_tx(&full[s], (KB_BM * KB_BK + KB_BK * TN) * 8);
                        kb_bulk_g2s_hint(Ts + (size_t)s * KB_BM * KB_BK, gt + (size_t)tau * (KB_BM * KB_BK),
                                         KB_BM * KB_BK * 8, &full[s], pol_w);
                        kb_bulk_g2s_hint(Bs + (size_t)s * KB_BK * TN, scratch + (size_t)t * (KB_BK * TN),
                                         KB_BK * TN * 8, &full[s], pol_c);
                    }
                }
            }
        } else if (warp >= 4) {
            uint32_t g = git;
            double qs[NT][2];
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) { qs[nt][0] = 0.0; qs[nt][1] = 0.0; }
            for (int I = 0; I < P.nrb; ++I) {
                const int kt = P.pm.ktiles[I];
                // this warp owns the m-tiles cw, cw+8, cw+16, cw+24 of the 256-row block (8 rows each):
                // interleaving keeps the eight warps equally busy inside the triangular diagonal block and
                // lets every m-tile skip the k tiles above the diagonal (W rows are lower-triangular, the
                // dual rows are dense, padding rows need nothing)
                int kmax[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int r0 = I * KB_BM + (cw + 8 * q) * 8;
                    if (r0 + 7 >= P.n && r0 < P.n + P.na) kmax[q] = 0x7fffffff;
                    else if (r0 >= P.n + P.na) kmax[q] = -1;
                    else kmax[q] = r0 + 7;
                }
                double acc[4][NT][2];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < NT; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
                for (int t = 0; t < kt; ++t, ++g) {
                    const int s = g % PT_STAGES;
                    // every consumer waits for every stage (also the ones it skips) so that no warp can lap
                    // the ring and arrive twice on empty[s] within one phase
                    mbar_wait(&full[s], (uint32_t)((g / PT_STAGES) & 1));
                    const int k0 = t * KB_BK;
                    if (k0 <= kmax[3] || k0 <= kmax[2] || k0 <= kmax[1] || k0 <= kmax[0]) {
                        const double* ts = Ts + (size_t)s * KB_BM * KB_BK;
                        const double* bs = Bs + (size_t)s * KB_BK * TN;
#pragma unroll
                        for (int k4 = 0; k4 < 4; ++k4) {
                            double fb[NT];
#pragma unroll
                            for (int nt = 0; nt < NT; ++nt) fb[nt] = bs[(k4 * NT + nt) * 32 + lane];
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                if (k0 <= kmax[q]) {
                                    const double fa = ts[(k4 * 32 + cw + 8 * q) * 32 + lane];
#pragma unroll
                                    for (int nt = 0; nt < NT; ++nt)
                                        kb_dmma(acc[q][nt][0], acc[q][nt][1], fa, fb[nt]);
                                }
                            }
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[s]);
                }
                // row-block epilogue: W rows -> running sum of squares; dual rows -> shared memory
#pragma unroll
                for (int mt = 0; mt < 4; ++mt) {
                    const int r = I * KB_BM + (cw + 8 * mt) * 8 + (lane >> 2);
                    if (r < P.n) {
                        if (!P.gform) {
#pragma unroll
                            for (int nt = 0; nt < NT; ++nt) {
                                qs[nt][0] += acc[mt][nt][0] * acc[mt][nt][0];
                                qs[nt][1] += acc[mt][nt][1] * acc[mt][nt][1];
                            }
                        } else {
                            // quadratic form c^T G c: multiply row r of T c by c[r] (read back from the
                            // scratch ring: tile r/16, fragment order)
                            const double* bt = scratch + (size_t)(r >> 4) * (KB_BK * TN) + ((r & 15) >> 2) * (NT * 32) + (r & 3);
#pragma unroll
                            for (int nt = 0; nt < NT; ++nt) {
                                const int c0i = nt * 8 + 2 * (lane & 3);
                                qs[nt][0] += acc[mt][nt][0] * bt[(c0i >> 3) * 32 + (c0i & 7) * 4];
                                qs[nt][1] += acc[mt][nt][1] * bt[((c0i + 1) >> 3) * 32 + ((c0i + 1) & 7) * 4];
                            }
                        }
                    } else if (r < P.n + P.na) {
                        double* ao = auxs + (r - P.n) * TN + 2 * (lane & 3);
#pragma unroll
                        for (int nt = 0; nt < NT; ++nt) {
                            ao[nt * 8] = acc[mt][nt][0];
                            ao[nt * 8 + 1] = acc[mt][nt][1];
                        }
                    }
                }
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    double v = qs[nt][i];
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    v += __shfl_xor_sync(0xffffffffu, v, 8);
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                    qs[nt][i] = v;
                }
            if ((lane >> 2) == 0) {
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    qred[cw * TN + nt * 8 + 2 * lane] = qs[nt][0];
                    qred[cw * TN + nt * 8 + 2 * lane + 1] = qs[nt][1];
                }
            }
        }
        // every role advances the ring counter by the same amount
        for (int I = 0; I < P.nrb; ++I) git += (uint32_t)P.pm.ktiles[I];
        __syncthreads();

        // ---------------- phase F: per-point finalize (DESIGN.md §3) ----------------
        if (tid < TN) {
            const long long pj = tile * TN + tid;
            if (pj < P.m) {
                double q = 0.0;
#pragma unroll
                for (int w = 0; w < 8; ++w) q += qred[w * TN + tid];     // fixed order: deterministic
                kb_finalize_point<DIM, double>(P, pj, q, auxs + tid, TN);
            }
        }
        __syncthreads();      // qred / auxs / scratch are re-used by the next tile
    }
}

static size_t solve_smem_pt() {     // sized for the 64-point tile (the 48-point variant needs less)
    return (size_t)PT_STAGES * (KB_BM * KB_BK + KB_BK * KB_TN) * sizeof(double) + 8 * KB_TN * sizeof(double) +
           KB_MAXAUX * KB_TN * sizeof(double) + 2 * PT_STAGES * sizeof(uint64_t) + 64;
}
size_t kbk_solve_pt_scratch_doubles(int n, int grid) {
    return (size_t)grid * ((n + KB_BK - 1) / KB_BK) * (KB_BK * KB_TN);
}


template <int DIM, int MODEL>
static cudaError_t solve_set_attr() {
    KB_CUDA_OK(cudaFuncSetAttribute(solve_kernel_pt<DIM, MODEL, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)solve_smem_pt()));
    KB_CUDA_OK(cudaFuncSetAttribute(solve_kernel_pt<DIM, MODEL, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)solve_smem_pt()));
    return cudaFuncSetAttribute(solve_kernel_pt<DIM, MODEL, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)solve_smem_pt());
}

cudaError_t kbk_solve_init() {
#define KB_ATTR(M) KB_CUDA_OK((solve_set_attr<2, M>())); KB_CUDA_OK((solve_set_attr<3, M>())); KB_CUDA_OK((solve_set_attr<KB_GEO, M>()));
    KB_ATTR(KB200_VG_LINEAR) KB_ATTR(KB200_VG_POWER) KB_ATTR(KB200_VG_GAUSSIAN)
    KB_ATTR(KB200_VG_EXPONENTIAL) KB_ATTR(KB200_VG_SPHERICAL) KB_ATTR(KB200_VG_HOLE_EFFECT) KB_ATTR(KB200_VG_TABLE)
#undef KB_ATTR
    return cudaSuccess;
}

template <int DIM>
static cudaError_t solve_pt_dim(const SolvePtParams& p, int grid, int tile_points, cudaStream_t st) {
    size_t sm = solve_smem_pt();
    switch (p.vg.model) {
#define KB_CASE(M) case M: if (tile_points == 16) solve_kernel_pt<DIM, M, 2><<<grid, PT_THREADS, sm, st>>>(p); \
                           else if (tile_points == 32) solve_kernel_pt<DIM, M, 4><<<grid, PT_THREADS, sm, st>>>(p); \
                           else solve_kernel_pt<DIM, M, 8><<<grid, PT_THREADS, sm, st>>>(p); break;
        KB_CASE(KB200_VG_LINEAR) KB_CASE(KB200_VG_POWER) KB_CASE(KB200_VG_GAUSSIAN)
        KB_CASE(KB200_VG_EXPONENTIAL) KB_CASE(KB200_VG_SPHERICAL) KB_CASE(KB200_VG_HOLE_EFFECT) KB_CASE(KB200_VG_TABLE)
#undef KB_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t kbk_solve_pt(int dim, const SolvePtParams& p, int grid, int tile_points, cudaStream_t st) {
    if (tile_points != 64 && tile_points != 32 && tile_points != 16) return cudaErrorInvalidValue;
    if (dim == KB_GEO) return solve_pt_dim<KB_GEO>(p, grid, tile_points, st);
    return dim == 2 ? solve_pt_dim<2>(p, grid, tile_points, st) : solve_pt_dim<3>(p, grid, tile_points, st);
}

