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
// Kernels in this file (all fp64, mma.sync.m16n8k16 = SASS DMMA.16x8x16; on H100 the 16x8xK shapes run at twice the
// per-FMA rate of m8n8k4, 127 vs 64 FMA/clk/SM, scripts/dmma_rate.py):
//   solve_kernel_pt   (K3 v3, the product path) persistent CTAs, one CTA = 64 points x all rows of W, RHS column
//                     block generated once per tile, W/RHS tiles streamed by cp.async.bulk + mbarrier, fused
//                     finalize. See the comment above the kernel.
// The wgmma variants (dtype float32 and float64x) live in solve_wgmma.cu.
#include "common.cuh"
#include "kernels.h"

// ---------------------------------------------------------------------------------------------
// K3 v3: persistent, warp-specialised, one CTA = one tile of 64 prediction points x ALL rows of W.
//
// v1 (one CTA per (row block, point tile)) regenerates every RHS tile once per row block - a 10x
// recompute of sqrt+exp at N=5000 - and alternates generation with the tensor work (measured: DMMA pipe
// 54 % active). v2 (warp-specialised but still regenerating) was slower: four producer warps cannot
// hide the fp64 sqrt/exp latency. v3 removes the recompute instead:
//   phase G  the 8 consumer warps evaluate the RHS column block c[k][j] of the tile ONCE (n x 64 values) and
//            park it, already in MMA-fragment order, in a per-CTA scratch ring (L2-resident, re-used for
//            every tile the CTA processes; size independent of M);
//   phase M  warp 0 streams W tiles (32 KB) and RHS tiles (8 KB) with cp.async.bulk + mbarrier into a
//            5-stage ring; warps 4..11 do nothing but LDS + m16n8k16 DMMA, walking all row blocks; each owns
//            the 16-row m-tiles j and 15 - j of a block (2 x NT x 4 accumulators) and adds its per-point sums
//            of squares to shared memory at the end of every row block (a CTA of 12 warps gets 168 registers
//            per thread; warps 0..3 need few and hand theirs to the consumers with setmaxnreg: 56 / 224);
//   phase F  the (K+1)x(K+1) drift solve and the two outputs per point are produced in the same CTA:
//            no partial buffers, no separate finalize pass, fixed summation order (deterministic).
#define PT_STAGES 5
#define PT_THREADS 384
#define PT_CONS0 (PT_THREADS / 32 - 8)    // first of the 8 consumer warps
#define PT_STAGE_BYTES ((KB_BM * KB_BK + KB_BK * KB_TN) * 8)
// registers per thread of warpgroup 0 and of the consumer warpgroups (setmaxnreg) and at launch (__launch_bounds__):
// 128 x 56 + 256 x 224 = 384 x 168
#define PT_REGS_PRODUCER 56
#define PT_REGS_CONSUMER 224

// Sum of v[0..CNT) over the 8 lanes of a warp that share lane & 3 (the row lanes of an MMA C fragment), halving the
// values at each of the butterfly steps xor 16, 8, 4: afterwards v[0..max(CNT/8, 1)) hold this lane's share of the sums.
// Every sum is added up in the same tree ((l + l^16) + (l^8 + ...)) + ... whatever CNT is, so a point's result does
// not depend on the tile width.
template <int C>
__device__ __forceinline__ void pt_reduce_scatter_step(double* v, int lane, int mask) {
    if constexpr (C >= 2) {
        const bool up = (lane & mask) != 0;
#pragma unroll
        for (int h = 0; h < C / 2; ++h) {
            const double send = up ? v[h] : v[h + C / 2];
            const double keep = up ? v[h + C / 2] : v[h];
            v[h] = keep + __shfl_xor_sync(0xffffffffu, send, mask);
        }
    } else {
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], mask);
    }
}
template <int CNT>
__device__ __forceinline__ void pt_reduce_scatter(double* v, int lane) {
    pt_reduce_scatter_step<CNT>(v, lane, 16);
    pt_reduce_scatter_step<(CNT >= 2 ? CNT / 2 : 1)>(v, lane, 8);
    pt_reduce_scatter_step<(CNT >= 4 ? CNT / 4 : 1)>(v, lane, 4);
}
// which of the CNT sums v[i] holds after pt_reduce_scatter<CNT> (-1: a duplicate another lane also holds)
template <int CNT>
__device__ __forceinline__ int pt_reduce_scatter_index(int i, int lane) {
    int o = i, c = CNT;
    for (int mask = 16; mask >= 4; mask >>= 1) {
        if (c >= 2) { c /= 2; if (lane & mask) o += c; }
        else if (lane & mask) return -1;
    }
    return o;
}

// Phase M of one consumer warp over the stages [g, gto) of the ring: wait for each, run one m16n8k16 per (m-tile,
// n-tile) for the m-tiles in ON (bit q: m-tile mt[q]), release the stage. ON is a template argument, so no mma.sync sits
// behind a branch the compiler cannot prove warp-uniform (that costs a WARPSYNC before every DMMA).
template <int NT, int ON>
__device__ __forceinline__ void pt_stages(uint32_t& g, uint32_t gto, double (&acc)[2][NT][4], const double* Ts,
                                          const double* Bs, uint64_t* full, uint64_t* empty, const int (&mt)[2], int lane) {
    for (; g < gto; ++g) {
        const int s = g % PT_STAGES;
        // every consumer waits for every stage (also the ones it skips) so that no warp can lap the ring and arrive
        // twice on empty[s] within one phase
        kb_mbar_wait(&full[s], (uint32_t)((g / PT_STAGES) & 1));
        if constexpr (ON != 0) {
            const double2* ts = reinterpret_cast<const double2*>(Ts + (size_t)s * KB_BM * KB_BK);
            const double* bs = Bs + (size_t)s * KB_BK * NT * 8;
            double fa[2][8];
#pragma unroll
            for (int q = 0; q < 2; ++q)
                if (ON >> q & 1)
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4) {
                        const double2 v = ts[(mt[q] * 4 + k4) * 32 + lane];
                        fa[q][2 * k4] = v.x; fa[q][2 * k4 + 1] = v.y;
                    }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                double fb[4];
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) fb[k4] = bs[(k4 * NT + nt) * 32 + lane];
                if (ON & 1) kb_dmma_16x8x16(acc[0][nt], fa[0], fb);
                if (ON & 2) kb_dmma_16x8x16(acc[1][nt], fa[1], fb);
            }
        }
        __syncwarp();
        if (lane == 0) kb_mbar_arrive(&empty[s]);
    }
}

// NT = n-tiles (of 8 points) per point tile: 8 (64 points) is the default. Narrower tiles (NT = 4, 2: 32 / 16 points) are used by
// the host for the TAIL of a launch: the points left over after the last full round of 64-point tiles would keep only a few of
// the persistent CTAs (one per SM) busy for a whole tile time (1953 tiles on 132 SMs = 14.8 rounds at 125 000 points per
// GPU); as narrow tiles they spread over all SMs and a tile costs little more than streaming W once. The per-point arithmetic
// does not depend on NT (tests/test_parity_gpu.py::test_tile_width_is_invisible).
// FIELDS (kb200_set_values): the dual rows are K + 1 + V rows, staged per CTA in global memory (P.fstage) instead of
// shared memory; a separate instantiation, so that the single-field kernels keep their code and registers.
template <int DIM, int MODEL, int NT, bool FIELDS>
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
        for (int s = 0; s < PT_STAGES; ++s) { kb_mbar_init(&full[s], 1); kb_mbar_init(&empty[s], 8); }
        kb_fence_mbar_init();
    }
    __syncthreads();

    // stages of one tile (W tiles of all row blocks); the running stage counter of a tile starts at (tiles this CTA
    // already did) x this, the same sequence in producer and consumers (recomputed per tile: no register held)
    const uint32_t stages_per_tile = (uint32_t)(P.pm.tile_off[P.nrb - 1] + P.pm.ktiles[P.nrb - 1]);
    // consumer warp 0..7, read from lane 0 so that the compiler knows it (and the m-tile limits of phase M computed
    // from it) to be warp-uniform
    const int cw = __shfl_sync(0xffffffffu, warp - PT_CONS0, 0);

    // ---------------- phase G: RHS column block of a tile, once, by the 8 consumer warps ----------------
    auto phase_g = [&](long long tile) {
        const int ct = tid - PT_CONS0 * 32;
        const int pl = ct % TN;                  // point within the tile
        const int ks = ct / TN;                  // k-tile slice (4 slices at 64 points)
        const long long pj = tile * TN + pl;
        const bool pvalid = pj < P.m;
        double px = 0.0, py = 0.0, pz = 0.0;
        if (pvalid) kb_load_point<DIM>(P.ps, P.an, pj, px, py, pz);
        for (int t = ks; t < nk; t += (PT_THREADS - PT_CONS0 * 32) / TN) {
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
        kb_fence_publish_async();      // the bulk copies of this CTA read the ring
    };

    // The warps keep one role for the whole kernel. In warpgroup 0 (warps 0..3) warp 0 streams the ring in phase M and
    // the others wait; it lends registers to the consumer warpgroups (warps 4..11), which hold the accumulators and the
    // operand fragments of two m-tiles in phase M and run phases G and F (ptxas 12.9 crashes on phase G's geographic
    // distance code in warpgroup 0's register-reduced region). Both loops pass the same three barriers per tile. The loops count this CTA's
    // tiles in 32 bits and form the 64-bit tile index where it is used.
    if (warp < PT_CONS0) {
        kb_setmaxnreg_dec<PT_REGS_PRODUCER>();
        for (uint32_t it = 0; blockIdx.x + (long long)it * gridDim.x < ntiles; ++it) {
            __syncthreads();      // phase G
            // ---------------- phase M: the producer ----------------
            const uint32_t git = it * stages_per_tile;
            if (warp == 0 && lane == 0) {
                uint32_t g = git;
                const uint64_t pol_w = kb_policy_evict_last(), pol_c = kb_policy_evict_first();
                long long tau = 0;                   // W tiles are stored contiguously in (I, t) order
                for (int I = 0; I < P.nrb; ++I) {
                    const int kt = P.pm.ktiles[I];
                    for (int t = 0; t < kt; ++t, ++tau, ++g) {
                        const int s = g % PT_STAGES;
                        kb_mbar_wait(&empty[s], (uint32_t)(((g / PT_STAGES) & 1) ^ 1));
                        kb_mbar_expect_tx(&full[s], (KB_BM * KB_BK + KB_BK * TN) * 8);
                        kb_bulk_g2s_hint(Ts + (size_t)s * KB_BM * KB_BK, gt + (size_t)tau * (KB_BM * KB_BK),
                                         KB_BM * KB_BK * 8, &full[s], pol_w);
                        kb_bulk_g2s_hint(Bs + (size_t)s * KB_BK * TN, scratch + (size_t)t * (KB_BK * TN),
                                         KB_BK * TN * 8, &full[s], pol_c);
                    }
                }
            }
            __syncthreads();
            __syncthreads();      // phase F
        }
    } else {
        kb_setmaxnreg_inc<PT_REGS_CONSUMER>();
        for (uint32_t it = 0; blockIdx.x + (long long)it * gridDim.x < ntiles; ++it) {
            const long long tile = blockIdx.x + (long long)it * gridDim.x;
            phase_g(tile);
            __syncthreads();
            // ---------------- phase M: the consumers ----------------
            const uint32_t git = it * stages_per_tile;
            uint32_t g = git;
            // running per-point sums of this warp, kept in its row of qred (registers are spent on the accumulators):
            // after the reduce-scatter of each row-block epilogue, sum v of this lane belongs to (n-tile, column)
            // o = pt_reduce_scatter_index(v), or is a duplicate another lane owns (o < 0)
            constexpr int QV = NT >= 4 ? NT / 4 : 1;
            double* qrow = qred + cw * TN;
#pragma unroll
            for (int v = 0; v < QV; ++v) {
                const int o = pt_reduce_scatter_index<2 * NT>(v, lane);     // sum 2 nt + i: point nt*8 + 2 t + i
                if (o >= 0) qrow[(o >> 1) * 8 + 2 * (lane & 3) + (o & 1)] = 0.0;
            }
            // this warp owns the 16-row m-tiles cw and 15 - cw of every 256-row block: the pair keeps the eight warps
            // equally busy inside the triangular diagonal block (cw + 1 and 16 - cw k tiles), and every m-tile skips
            // the k tiles above its diagonal (W rows are lower-triangular, the dual rows dense, padding rows empty)
            const int mtl[2] = {cw, 15 - cw};
            for (int I = 0; I < P.nrb; ++I) {
                const uint32_t gend = g + (uint32_t)P.pm.ktiles[I];
                // stage counter bound of each m-tile: its k tiles 0 .. (k up to its last row) of the block
                uint32_t glim[2];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int r0 = I * KB_BM + mtl[q] * 16;
                    if (r0 + 15 >= P.n && r0 < P.n + P.na) glim[q] = gend;
                    else if (r0 >= P.n + P.na) glim[q] = g;
                    else glim[q] = g + (uint32_t)(r0 / KB_BK + 1);
                }
                double acc[2][NT][4];
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int b = 0; b < NT; ++b)
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.0;
                // each m-tile's k tiles are a prefix of the block's stages: both m-tiles up to the smaller limit, then
                // the one with the larger limit alone, then neither (the stages are still waited for and released)
                const uint32_t glo = min(min(glim[0], glim[1]), gend), ghi = min(max(glim[0], glim[1]), gend);
                pt_stages<NT, 3>(g, glo, acc, Ts, Bs, full, empty, mtl, lane);
                if (glim[0] > glim[1]) pt_stages<NT, 1>(g, ghi, acc, Ts, Bs, full, empty, mtl, lane);
                else pt_stages<NT, 2>(g, ghi, acc, Ts, Bs, full, empty, mtl, lane);
                pt_stages<NT, 0>(g, gend, acc, Ts, Bs, full, empty, mtl, lane);
                // row-block epilogue, in place: every accumulator of a W row becomes its term of the point's sum (square,
                // or c[r] times it for the quadratic form), dual rows go to shared memory and, like padding rows, add 0;
                // then the warp's per-point sums (fixed order: m-tile, row g before g + 8) are reduced over the 8 row
                // lanes and added to the running sums
#pragma unroll
                for (int q = 0; q < 2; ++q)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int r = I * KB_BM + mtl[q] * 16 + 8 * h + (lane >> 2);
                        if (r < P.n) {
                            if (!P.gform) {
#pragma unroll
                                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                                    for (int i = 0; i < 2; ++i) acc[q][nt][2 * h + i] *= acc[q][nt][2 * h + i];
                            } else {
                                // quadratic form c^T G c: multiply row r of T c by c[r] (read back from the scratch
                                // ring: tile r/16, fragment order)
                                const double* bt = P.scratch + ((size_t)blockIdx.x * nk + (r >> 4)) * (KB_BK * TN) +
                                                   ((r & 15) >> 2) * (NT * 32) + (r & 3);
#pragma unroll
                                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                                    for (int i = 0; i < 2; ++i) {
                                        const int c = nt * 8 + 2 * (lane & 3) + i;
                                        acc[q][nt][2 * h + i] *= bt[(c >> 3) * 32 + (c & 7) * 4];
                                    }
                            }
                        } else {
                            if (r < P.n + P.na) {
                                // FIELDS: the K + 1 + V dual rows do not fit in shared memory; they go to this CTA's rows
                                // of the global staging buffer, which phase F reads back after the barrier
                                double* ao = (FIELDS ? P.fstage + (int)(blockIdx.x * P.na * TN) : auxs) + (r - P.n) * TN +
                                             2 * (lane & 3);
#pragma unroll
                                for (int nt = 0; nt < NT; ++nt) {
                                    ao[nt * 8] = acc[q][nt][2 * h];
                                    ao[nt * 8 + 1] = acc[q][nt][2 * h + 1];
                                }
                            }
#pragma unroll
                            for (int nt = 0; nt < NT; ++nt) { acc[q][nt][2 * h] = 0.0; acc[q][nt][2 * h + 1] = 0.0; }
                        }
                    }
                double part[2 * NT];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        part[2 * nt + i] = ((acc[0][nt][i] + acc[0][nt][2 + i]) + acc[1][nt][i]) + acc[1][nt][2 + i];
                pt_reduce_scatter<2 * NT>(part, lane);
#pragma unroll
                for (int v = 0; v < QV; ++v) {
                    const int o = pt_reduce_scatter_index<2 * NT>(v, lane);
                    if (o >= 0) qrow[(o >> 1) * 8 + 2 * (lane & 3) + (o & 1)] += part[v];
                }
            }
            __syncthreads();

            // ---------------- phase F: per-point finalize (DESIGN.md §3), one consumer thread per point ----------------
            const int ft = tid - PT_CONS0 * 32;
            if (ft < TN) {
                const long long pj = tile * TN + ft;
                if (pj < P.m) {
                    double q = 0.0;
#pragma unroll
                    for (int w = 0; w < 8; ++w) q += qred[w * TN + ft];     // fixed order: deterministic
                    if constexpr (FIELDS)
                        kb_finalize_point<DIM, double, true>(P, pj, q, P.fstage + (int)(blockIdx.x * P.na * TN) + ft, TN);
                    else
                        kb_finalize_point<DIM, double>(P, pj, q, auxs + ft, TN);
                }
            }
            __syncthreads();      // qred / auxs / scratch are re-used by the next tile
        }
    }
}

static size_t solve_smem_pt() {     // sized for the 64-point tile (the 48-point variant needs less)
    return (size_t)PT_STAGES * (KB_BM * KB_BK + KB_BK * KB_TN) * sizeof(double) + 8 * KB_TN * sizeof(double) +
           KB_MAXAUX * KB_TN * sizeof(double) + 2 * PT_STAGES * sizeof(uint64_t) + 64;
}
size_t kbk_solve_pt_scratch_doubles(int n, int grid) {
    return (size_t)grid * ((n + KB_BK - 1) / KB_BK) * (KB_BK * KB_TN);
}


// Tile widths in points (NT = width / 8 n-tiles). The fields kernels run 32- and 16-point tiles only: with 64-point tiles
// the global staging of the dual rows costs the 64-point kernel its last registers (ptxas spills), so the widest fields
// tile is NT = 4 (KB_TN_FIELDS in api.cu).
using PtWidths = KbList<16, 32, 64>;

cudaError_t kbk_solve_init() {
    const int sm = (int)solve_smem_pt();
    return KbDims::for_each([&](auto D) {
        return KbModels::for_each([&](auto M) {
            return PtWidths::for_each([&](auto TN) {
                KB_CUDA_OK(cudaFuncSetAttribute(solve_kernel_pt<D, M, TN / 8, false>,
                                                cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
                if constexpr (TN == 64) return cudaSuccess;
                else return cudaFuncSetAttribute(solve_kernel_pt<D, M, TN / 8, true>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, sm);
            });
        });
    });
}

cudaError_t kbk_solve_pt(int dim, const SolvePtParams& p, int grid, int tile_points, cudaStream_t st) {
    const size_t sm = solve_smem_pt();
    return KbDims::dispatch(dim, [&](auto D) {
        return KbModels::dispatch(p.vg.model, [&](auto M) {
            return PtWidths::dispatch(tile_points, [&](auto TN) {
                if (!p.nf) solve_kernel_pt<D, M, TN / 8, false><<<grid, PT_THREADS, sm, st>>>(p);
                else if constexpr (TN == 64) return cudaErrorInvalidValue;
                else solve_kernel_pt<D, M, TN / 8, true><<<grid, PT_THREADS, sm, st>>>(p);
                return cudaGetLastError();
            });
        });
    });
}
