// solve_tf32.cu — K3 for dtype = KB200_F32: the same covariance-form contraction q_j = ||W c_j||^2
// (DESIGN.md §3) on the Hopper tensor cores: wgmma.mma_async m64n128k8 .tf32 with fp32 accumulators in
// registers. fp32 accuracy comes from the 3xTF32 split  W = Wh + Wl, c = ch + cl (each part exactly
// representable in TF32):  W c ~= Wh ch + Wh cl + Wl ch  accumulated in fp32 (tolerance for fp32 is 1e-2).
//
// Orientation: D[point][row of W], M = 64 points per CTA tile, N = 256 W rows per row block, split between two
// consumer warpgroups (128 rows = 64 fp32 accumulators per thread each). Each thread squares-and-adds its own
// accumulators; the four lanes sharing a point and the two warpgroups are summed once per point tile.
//   A operand (64 points)  : RHS tile, K-major, from the per-CTA scratch ring (generated once per point tile
//                            by the generator warps, fp32 sqrt/exp on fp64 coordinate differences)
//   B operand (256 W rows) : W tile, K-major, packed by pack_tf32_kernel
//   both in the no-swizzle K-major core-matrix layout: 8-row x 16-byte core matrices, k-chunks 128 B apart (LBO),
//   8-row groups 512 B apart (SBO); one stage = 16 k = 2 wgmma k-steps.
// Roles (480 threads): warps 0-7 = two consumer warpgroups (wgmma + epilogue + per-point finalize), warp 8 lane 0 =
// bulk-copy producer (cp.async.bulk + mbarrier), warps 9-14 = RHS generators (three threads per point).
#include "common.cuh"
#include "kernels.h"

#define TF_STAGES 4
#define TF_CONS_THREADS 256                 // warps 0-7: two consumer warpgroups
#define TF_GEN_THREADS 192                  // warps 9-14: three generator threads per prediction point
#define TF_THREADS (TF_CONS_THREADS + 32 + TF_GEN_THREADS)
#define TF_TM 64                   // points per CTA tile (wgmma M)
#define TF_BN KB_BM                // W rows per row block = 256 (two wgmma N = 128 halves)
#define TF_BK KB_BK                // k per stage = 16
#define TF_W_BYTES (TF_BN * TF_BK * 4 * 2)     // hi + lo = 32 KB
#define TF_C_BYTES (TF_TM * TF_BK * 4 * 2)     // hi + lo = 8 KB
#define TF_STAGE_BYTES (TF_W_BYTES + TF_C_BYTES)

__device__ __forceinline__ float tf32_round(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ uint64_t tf_desc(uint32_t smem_addr) { return kb_wgmma_desc(smem_addr, 128u, 512u); }

// d[64 points x 128 W rows] (+)= A[64 x 8] B[128 x 8]^T; scale_d = 0 overwrites d
__device__ __forceinline__ void tf_mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "setp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
                 "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, "
                 "%43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(scale_d) : "memory");
}

// ---- pack: W (fp64, row-major lower triangle) + dual rows -> TF32 hi/lo tiles in wgmma layout -------
// tile (row block I, k stage t): 8192 floats = [hi 4096][lo 4096];
//   element (r, k) of a part at float offset (r/8)*128 + (k/4)*32 + (r%8)*4 + (k%4)
__global__ void __launch_bounds__(256) pack_tf32_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                         const double* __restrict__ Uz, PackMap pm,
                                                         float* __restrict__ out) {
    int I = blockIdx.y, kt = blockIdx.x;
    if (kt >= pm.ktiles[I]) return;
    float* o = out + ((size_t)pm.tile_off[I] + kt) * (TF_W_BYTES / 4);
    for (int e = threadIdx.x; e < TF_BN * TF_BK; e += 256) {
        int rg = e >> 7, kc = (e >> 5) & 3, rr = (e >> 2) & 7, kk = e & 3;
        int r = I * TF_BN + rg * 8 + rr;
        int k = kt * TF_BK + kc * 4 + kk;
        double v = 0.0;
        if (r < n) { if (k <= r) v = W[(size_t)r * ld + k]; }
        else if (r < n + na) { if (k < n) v = Uz[(size_t)(r - n) * n_pad + k]; }
        float hi = tf32_round((float)v);
        float lo = tf32_round((float)(v - (double)hi));
        o[e] = hi;
        o[TF_BN * TF_BK + e] = lo;
    }
}

template <int DIM, int MODEL>
__device__ __forceinline__ float tf_cov_rhs(const VgParams& v, double dd) {
    // exact hit on the fp64 distance (|d| <= eps, ok.py:665-672); the variogram itself in fp32
    if (v.exact && dd <= v.eps) return (float)v.c0;
    float d = (float)dd;
    float c0 = (float)v.c0, p0 = (float)v.p0, p1 = (float)v.p1, p2 = (float)v.p2;
    float g;
    if (MODEL == KB200_VG_LINEAR) g = p0 * d + p1;
    else if (MODEL == KB200_VG_POWER) g = p0 * powf(d, p1) + p2;
    else if (MODEL == KB200_VG_GAUSSIAN) { float r = p1 * (4.0f / 7.0f); g = p0 * (1.0f - expf(-(d * d) / (r * r))) + p2; }
    else if (MODEL == KB200_VG_EXPONENTIAL) g = p0 * (1.0f - expf(-d / (p1 / 3.0f))) + p2;
    else if (MODEL == KB200_VG_SPHERICAL) {
        if (d <= p1) { float q = d / p1; g = p0 * (1.5f * q - 0.5f * q * q * q) + p2; } else g = p0 + p2;
    } else if (MODEL == KB200_VG_TABLE) g = (float)kb_gamma<KB200_VG_TABLE>(v, dd);     // tabulated callable (fp64 table)
    else { float q = d / (p1 / 3.0f); g = p0 * (1.0f - (1.0f - q) * expf(-q)) + p2; }
    return c0 - g;
}

template <int DIM, int MODEL>
__global__ void __launch_bounds__(TF_THREADS, 1) solve_kernel_tf32(const __grid_constant__ SolvePtParams P) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* stage_base = smem_raw;                                            // TF_STAGES * 40 KB
    float* auxs = reinterpret_cast<float*>(smem_raw + (size_t)TF_STAGES * TF_STAGE_BYTES);   // KB_MAXAUX * 64
    double* qpart = reinterpret_cast<double*>(auxs + KB_MAXAUX * TF_TM);            // 2 warpgroups x 64 points
    uint64_t* full = reinterpret_cast<uint64_t*>(qpart + 2 * TF_TM);                // TF_STAGES
    uint64_t* empty = full + TF_STAGES;                                              // TF_STAGES
    uint64_t* gfull = empty + TF_STAGES;                                             // 2
    uint64_t* gempty = gfull + 2;                                                    // 2

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nk = (P.n + TF_BK - 1) / TF_BK;
    const size_t sbuf = (size_t)nk * TF_C_BYTES;                                     // one RHS column block
    unsigned char* scratch = reinterpret_cast<unsigned char*>(P.scratch) + (size_t)blockIdx.x * 2 * sbuf;
    const unsigned char* gt = reinterpret_cast<const unsigned char*>(P.tiles);
    const long long ntiles = (P.m + TF_TM - 1) / TF_TM;

    if (tid == 0) {
        for (int s = 0; s < TF_STAGES; ++s) { kb_mbar_init(&full[s], 1); kb_mbar_init(&empty[s], 2); }
        for (int b = 0; b < 2; ++b) { kb_mbar_init(&gfull[b], TF_GEN_THREADS); kb_mbar_init(&gempty[b], 1); }
        kb_fence_mbar_init();
    }
    __syncthreads();

    // The generators work ONE POINT TILE AHEAD of the tensor pipe into the other half of a double-buffered scratch
    // ring (gfull / gempty mbarriers), as in solve_i8.cu.
    if (warp >= 9) {
        const int gt_ = tid - 9 * 32;
        const int pl = gt_ & (TF_TM - 1);
        const int ks = gt_ / TF_TM;                        // 0..2
        uint32_t it = 0;
        for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const int b = (int)(it & 1);
            kb_mbar_wait(&gempty[b], ((it >> 1) & 1) ^ 1);
            unsigned char* sc = scratch + (size_t)b * sbuf;
            const long long pj = tile * TF_TM + pl;
            const bool pvalid = pj < P.m;
            double px = 0.0, py = 0.0, pz = 0.0;
            if (pvalid) kb_load_point<DIM>(P.ps, P.an, pj, px, py, pz);
            for (int t = ks; t < nk; t += TF_GEN_THREADS / TF_TM) {
                float* ct = reinterpret_cast<float*>(sc + (size_t)t * TF_C_BYTES);
#pragma unroll
                for (int kc = 0; kc < 4; ++kc) {
                    float hi[4], lo[4];
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const int k = t * TF_BK + kc * 4 + kk;
                        float c = 0.0f;
                        if (pvalid && k < P.n) {
                            double dd = kb_dist<DIM>(__ldg(P.ax + k), __ldg(P.ay + k), KB_HASZ(DIM) ? __ldg(P.az + k) : 0.0,
                                                     px, py, pz);
                            c = tf_cov_rhs<DIM, MODEL>(P.vg, dd);
                        }
                        hi[kk] = tf32_round(c);
                        lo[kk] = tf32_round(c - hi[kk]);
                    }
                    const int off = (pl >> 3) * 128 + kc * 32 + (pl & 7) * 4;      // floats
                    *reinterpret_cast<float4*>(ct + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
                    *reinterpret_cast<float4*>(ct + TF_TM * TF_BK + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
                }
            }
            kb_fence_publish_async();
            kb_mbar_arrive(&gfull[b]);
        }
    } else if (warp == 8) {
        if (lane == 0) {
            const uint64_t pol_w = kb_policy_evict_last(), pol_c = kb_policy_evict_first();
            uint32_t gg = 0, it = 0;
            for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
                const int b = (int)(it & 1);
                const unsigned char* sc = scratch + (size_t)b * sbuf;
                kb_mbar_wait(&gfull[b], (it >> 1) & 1);
                long long tau = 0;
                for (int I = 0; I < P.nrb; ++I) {
                    const int kt = P.pm.ktiles[I];
                    for (int t = 0; t < kt; ++t, ++tau, ++gg) {
                        const int s = gg % TF_STAGES;
                        kb_mbar_wait(&empty[s], (uint32_t)(((gg / TF_STAGES) & 1) ^ 1));
                        kb_mbar_expect_tx(&full[s], TF_STAGE_BYTES);
                        unsigned char* sb = stage_base + (size_t)s * TF_STAGE_BYTES;
                        kb_bulk_g2s_hint(sb, gt + (size_t)tau * TF_W_BYTES, TF_W_BYTES, &full[s], pol_w);
                        kb_bulk_g2s_hint(sb + TF_W_BYTES, sc + (size_t)t * TF_C_BYTES, TF_C_BYTES, &full[s], pol_c);
                    }
                }
            }
        }
    } else {
        // consumers: warpgroup h owns W rows [128 h, 128 h + 128) of every row block. Accumulator element
        // i = 4 j + 2 hh + e of thread (warp w of the group, lane) is point 16 w + lane / 4 + 8 hh, row
        // 128 h + 8 j + 2 (lane % 4) + e.
        const int h = warp >> 2, wtid = tid & 127;
        const int p0 = (warp & 3) * 16 + (lane >> 2);       // points p0 and p0 + 8
        const int c0 = h * (TF_BN / 2) + 2 * (lane & 3);
        const uint32_t hoff = (uint32_t)h * (TF_BN / 2 / 8) * 512u;
        uint32_t gg = 0, it = 0;
        for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            double q[2] = {0.0, 0.0};
            for (int I = 0; I < P.nrb; ++I) {
                const int kt = P.pm.ktiles[I];
                float acc[64];
                for (int t = 0; t < kt; ++t, ++gg) {
                    const int s = gg % TF_STAGES;
                    kb_mbar_wait(&full[s], (uint32_t)((gg / TF_STAGES) & 1));
                    kb_wgmma_fence();
                    const uint32_t wb = kb_smem_u32(stage_base + (size_t)s * TF_STAGE_BYTES);
                    const uint32_t w_hi = wb + hoff, w_lo = wb + TF_W_BYTES / 2 + hoff;
                    const uint32_t c_hi = wb + TF_W_BYTES, c_lo = c_hi + TF_C_BYTES / 2;
#pragma unroll
                    for (int kstep = 0; kstep < TF_BK / 8; ++kstep) {
                        const uint32_t ko = (uint32_t)kstep * 256u;          // 2 k-chunks of 128 B
                        tf_mma(acc, tf_desc(c_hi + ko), tf_desc(w_hi + ko), (t == 0 && kstep == 0) ? 0u : 1u);
                        tf_mma(acc, tf_desc(c_hi + ko), tf_desc(w_lo + ko), 1u);
                        tf_mma(acc, tf_desc(c_lo + ko), tf_desc(w_hi + ko), 1u);
                    }
                    kb_wgmma_commit();
                    kb_wgmma_wait<1>();                  // the previous stage has been read: hand it back
                    if (t > 0 && wtid == 0) kb_mbar_arrive(&empty[(gg - 1) % TF_STAGES]);
                }
                kb_wgmma_wait<0>();
                if (wtid == 0) kb_mbar_arrive(&empty[(gg - 1) % TF_STAGES]);
#pragma unroll
                for (int i = 0; i < 64; ++i) kb_reg_fence(acc[i]);
                const int rb = I * TF_BN + c0;
                if (I * TF_BN + (h + 1) * (TF_BN / 2) <= P.n) {
#pragma unroll
                    for (int i = 0; i < 64; ++i) { const double x = (double)acc[i]; q[(i >> 1) & 1] += x * x; }
                } else {
#pragma unroll
                    for (int i = 0; i < 64; ++i) {
                        const int r = rb + 8 * (i >> 2) + (i & 1), hh = (i >> 1) & 1;
                        const float x = acc[i];
                        if (r < P.n) q[hh] += (double)x * (double)x;
                        else if (r < P.n + P.na) auxs[(r - P.n) * TF_TM + p0 + 8 * hh] = x;
                    }
                }
            }
            // the four lanes of a point hold interleaved columns; then the two warpgroups
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                q[hh] += __shfl_xor_sync(0xffffffffu, q[hh], 1);
                q[hh] += __shfl_xor_sync(0xffffffffu, q[hh], 2);
                if ((lane & 3) == 0) qpart[h * TF_TM + p0 + 8 * hh] = q[hh];
            }
            kb_named_sync(1, TF_CONS_THREADS);
            // ---------------- phase F: finalize (DESIGN.md §3), thread = point ----------------
            if (tid < TF_TM) {
                const long long pj = tile * TF_TM + tid;
                if (pj < P.m) kb_finalize_point<DIM, float>(P, pj, qpart[tid] + qpart[TF_TM + tid], auxs + tid, TF_TM);
            }
            kb_named_sync(1, TF_CONS_THREADS);
            if (tid == 0) kb_mbar_arrive(&gempty[(int)(it & 1)]);      // this tile's scratch half may be rewritten
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------
static size_t tf32_smem() {
    return (size_t)TF_STAGES * TF_STAGE_BYTES + (size_t)KB_MAXAUX * TF_TM * sizeof(float) + 2 * TF_TM * sizeof(double) +
           (2 * TF_STAGES + 4) * sizeof(uint64_t) + 64;
}

size_t kbk_solve_tf32_scratch_bytes(int n, int grid) {
    return (size_t)grid * 2 * ((n + TF_BK - 1) / TF_BK) * TF_C_BYTES;      // double-buffered
}
int kbk_solve_tf32_tile_points() { return TF_TM; }

cudaError_t kbk_solve_tf32_init() {
    return KbDims::for_each([&](auto D) {
        return KbModels::for_each([&](auto M) {
            return cudaFuncSetAttribute(solve_kernel_tf32<D, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tf32_smem());
        });
    });
}

cudaError_t kbk_solve_tf32(int dim, const SolvePtParams& p, int grid, cudaStream_t st) {
    return KbDims::dispatch(dim, [&](auto D) {
        return KbModels::dispatch(p.vg.model, [&](auto M) {
            solve_kernel_tf32<D, M><<<grid, TF_THREADS, tf32_smem(), st>>>(p);
            return cudaGetLastError();
        });
    });
}

cudaError_t kbk_pack_tf32(const double* W, int ld, int n, int n_pad, int na, const double* Uz, const PackMap& pm,
                          void* out, cudaStream_t st) {
    pack_tf32_kernel<<<kb_pack_grid(pm), 256, 0, st>>>(W, ld, n, n_pad, na, Uz, pm, (float*)out);
    return cudaGetLastError();
}
