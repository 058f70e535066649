// solve_wgmma.cu — K3 on the Hopper warpgroup tensor cores (wgmma.mma_async): the covariance-form contraction
// q_j = ||W c_j||^2 (DESIGN.md §3) as one pipeline with two arithmetics plugged into it.
//
// The pipeline (solve_wgmma below). Orientation: D[point][W row], M = 64 points per CTA tile, N = BN W rows per row
// block, split between two consumer warpgroups (BN / 2 rows each). Operands are in the no-swizzle K-major core-matrix
// layout: 8-row x 16-byte core matrices, k-chunks 128 B apart (LBO), 8-row groups SBO apart.
// Roles (480 threads): warps 0-7 = two consumer warpgroups (wgmma, row-block epilogue, per-point finalize), warp 8
// lane 0 = bulk-copy producer (cp.async.bulk + mbarrier: the W tile, evict_last, and the RHS tile, evict_first, of each
// stage), warps 9-14 = RHS generators (three threads per point, interleaved k-stages: the sqrt/exp chains are
// latency-bound). The generators work one point tile AHEAD of the tensor pipe: they write the RHS column block of tile
// i+1 into the other half of a double-buffered per-CTA scratch ring while the MMAs of tile i run (the pipes they use
// do not compete); gfull / gempty mbarriers hand the halves over. Each thread squares-and-adds its own rows; the four
// lanes sharing a point and the two warpgroups are summed once per point tile, then one thread per point finalizes.
//
// The arithmetics (Tf32Arith, I8Arith) supply what differs: tile sizes and stage count, the RHS writer, the MMAs of
// one stage and the row-block epilogue.
//   dtype = KB200_F32: wgmma m64n128k8 .tf32 with fp32 accumulators. fp32 accuracy comes from the 3xTF32 split
//     W = Wh + Wl, c = ch + cl (each part exactly representable in TF32):  W c ~= Wh ch + Wh cl + Wl ch  accumulated
//     in fp32 (tolerance for fp32 is 1e-2). BN = 256 (128 rows = 64 fp32 accumulators per thread), one stage = 16 k
//     = 2 wgmma k-steps, SBO = 512 B. The variogram model is a template argument.
//   dtype = KB200_F64X / F64X5 / F64X4: fp64-class accuracy on the INT8 path (wgmma .s32.s8.s8, exact int32
//     accumulation). Error-free slicing (the "Ozaki scheme"): every row of W and every RHS column is scaled by a power
//     of two into (-1, 1) and cut into S signed slices of 6+7+...+7 bits (S = 6: 41 bits, 5: 34 bits, 4: 27 bits),
//          x = 2^e * sum_s slice_s * 2^(-6-7s),   |slice_s| <= 64,
//     so that  W_rk c_k = 2^(ew_r + ec_j) * sum_{s,t} w_s c_t 2^(-12-7(s+t)).  All slice products with the same
//     d = s + t are summed EXACTLY in one int32 accumulator (|sum| <= n * (d+1) * 64^2 < 2^31 for n <= 32512); pairs
//     with d >= S are dropped (relative 2^-(7S+6) per term). The S accumulators are combined exactly in int64 in the
//     epilogue and converted to fp64 once. S = 6 agrees with the fp64 DMMA kernel to ~1e-10 (tests); fewer slices trade
//     bits for MMAs (S(S+1)/2 per k-stage: 21 / 15 / 10) and operand bytes; dtype='float64' keeps the DMMA kernel as
//     the default. BN = 48 / 64 / 64 for S = 6 / 5 / 4 (S * BN / 4 int32 accumulators per thread stay in registers),
//     one stage = 32 k = one MMA k-step, SBO = 256 B. The variogram model is a run-time switch (phase G is < 10 % of
//     the kernel), so that the slice count and the dimension are the only template parameters.
#include "common.cuh"
#include "kernels.h"

#define WG_CONS_THREADS 256                // warps 0-7: two consumer warpgroups
#define WG_GEN_THREADS 192                 // warps 9-14: three generator threads per prediction point
#define WG_THREADS (WG_CONS_THREADS + 32 + WG_GEN_THREADS)

// ---- warpgroup MMA (wgmma, sm_90a) -------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major, no swizzle ("interleave" layout): 8-row x 16-byte core matrices,
// lbo = byte stride between the two k-adjacent core matrices one instruction reads, sbo = byte stride between
// 8-row groups. Bits 0-13 start address >> 4, 16-29 lbo >> 4, 32-45 sbo >> 4, layout type (62-63) 0.
__device__ __forceinline__ uint64_t kb_wgmma_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | ((uint64_t)((lbo >> 4) & 0x3fffu) << 16) |
           ((uint64_t)((sbo >> 4) & 0x3fffu) << 32);
}
__device__ __forceinline__ void kb_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void kb_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void kb_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" :: "n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator register across a wgmma wait
__device__ __forceinline__ void kb_reg_fence(float& r) { asm volatile("" : "+f"(r) :: "memory"); }
__device__ __forceinline__ void kb_reg_fence(uint32_t& r) { asm volatile("" : "+r"(r) :: "memory"); }
// named barrier over the first `threads` threads of the block (id 0 is __syncthreads)
__device__ __forceinline__ void kb_named_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;\n" :: "r"(id), "r"(threads) : "memory");
}

// ==== float32: 3xTF32 =============================================================================================
struct Tf32Cfg {
    static constexpr int STAGES = 4;
    static constexpr int BN = KB_BM;                        // W rows per row block = 256 (two wgmma N = 128 halves)
    static constexpr int BK = KB_BK;                        // k per stage = 16
    static constexpr int W_BYTES = BN * BK * 4 * 2;         // hi + lo = 32 KB
    static constexpr int C_BYTES = KB_WG_TM * BK * 4 * 2;   // hi + lo = 8 KB
    static constexpr int STAGE_BYTES = W_BYTES + C_BYTES;
    static constexpr int SBO = 512;                         // 8-row group stride of the operand tiles
    static constexpr int PEXP_INTS = 0;                     // no per-point exponents
    typedef float aux_t;                                    // dual-row results
};

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
    float* o = out + ((size_t)pm.tile_off[I] + kt) * (Tf32Cfg::W_BYTES / 4);
    for (int e = threadIdx.x; e < Tf32Cfg::BN * Tf32Cfg::BK; e += 256) {
        int rg = e >> 7, kc = (e >> 5) & 3, rr = (e >> 2) & 7, kk = e & 3;
        int r = I * Tf32Cfg::BN + rg * 8 + rr;
        int k = kt * Tf32Cfg::BK + kc * 4 + kk;
        double v = 0.0;
        if (r < n) { if (k <= r) v = W[(size_t)r * ld + k]; }
        else if (r < n + na) { if (k < n) v = Uz[(size_t)(r - n) * n_pad + k]; }
        float hi = tf32_round((float)v);
        float lo = tf32_round((float)(v - (double)hi));
        o[e] = hi;
        o[Tf32Cfg::BN * Tf32Cfg::BK + e] = lo;
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

template <int MODEL>
struct Tf32Arith : Tf32Cfg {
    typedef float acc_t[64];            // 64 points x 128 W rows of one warpgroup
    __device__ __forceinline__ static int nrb(const SolvePtParams& P) { return P.nrb; }
    __device__ __forceinline__ static int ktiles(const SolvePtParams& P, int I, int) { return P.pm.ktiles[I]; }

    // RHS of point pl for k stage t: hi / lo TF32 parts, fp32 variogram on fp64 coordinate differences
    template <int DIM>
    __device__ __forceinline__ static void rhs_stage(const SolvePtParams& P, unsigned char* dst, int t, int pl, bool pvalid,
                                                     double px, double py, double pz, double) {
        float* ct = reinterpret_cast<float*>(dst);
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
            float hi[4], lo[4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const int k = t * BK + kc * 4 + kk;
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
            *reinterpret_cast<float4*>(ct + KB_WG_TM * BK + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
        }
    }

    // sb: the stage (W tile, then RHS tile), hoff: offset of this warpgroup's W rows
    __device__ __forceinline__ static void mma_stage(acc_t& acc, uint32_t sb, uint32_t hoff, bool first) {
        const uint32_t w_hi = sb + hoff, w_lo = sb + W_BYTES / 2 + hoff;
        const uint32_t c_hi = sb + W_BYTES, c_lo = c_hi + C_BYTES / 2;
#pragma unroll
        for (int kstep = 0; kstep < BK / 8; ++kstep) {
            const uint32_t ko = (uint32_t)kstep * 256u;          // 2 k-chunks of 128 B
            tf_mma(acc, tf_desc(c_hi + ko), tf_desc(w_hi + ko), (first && kstep == 0) ? 0u : 1u);
            tf_mma(acc, tf_desc(c_hi + ko), tf_desc(w_lo + ko), 1u);
            tf_mma(acc, tf_desc(c_lo + ko), tf_desc(w_hi + ko), 1u);
        }
    }

    // sum of squares of the W rows, dual rows to auxs; I: row block, p0: the thread's first point
    __device__ __forceinline__ static void epilogue(const SolvePtParams& P, acc_t& acc, int I, int h, int lane, int p0,
                                                    const double (&)[2], double (&q)[2], float* auxs) {
#pragma unroll
        for (int i = 0; i < 64; ++i) kb_reg_fence(acc[i]);
        const int rb = I * BN + (h * (BN / 2) + 2 * (lane & 3));
        if (I * BN + (h + 1) * (BN / 2) <= P.n) {               // W rows only
#pragma unroll
            for (int i = 0; i < 64; ++i) { const double x = (double)acc[i]; q[(i >> 1) & 1] += x * x; }
        } else {
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int r = rb + 8 * (i >> 2) + (i & 1), hh = (i >> 1) & 1;
                const float x = acc[i];
                if (r < P.n) q[hh] += (double)x * (double)x;
                else if (r < P.n + P.na) auxs[(r - P.n) * KB_WG_TM + p0 + 8 * hh] = x;
            }
        }
    }
};

// ==== float64x: int8 slices =======================================================================================
#define I8_BK 32
#define I8_C_SLICE (KB_WG_TM * I8_BK)            // 2 KB

// W rows per row block: BN / 2 is a valid wgmma N; S * BN / 4 accumulators per thread
__host__ __device__ constexpr int i8_bn(int S) { return S == 6 ? 48 : 64; }
template <int S> struct I8Cfg {
    static constexpr int BN = i8_bn(S);
    static constexpr int BK = I8_BK;
    static constexpr int STAGES = 6;
    static constexpr int W_SLICE = BN * I8_BK;
    static constexpr int W_BYTES = S * W_SLICE;
    static constexpr int C_BYTES = S * I8_C_SLICE;
    static constexpr int STAGE_BYTES = W_BYTES + C_BYTES;
    static constexpr int SBO = 256;                         // 8-row group stride of the operand tiles
    static constexpr int PEXP_INTS = 2 * KB_WG_TM;          // exponent of each point's column, per scratch half
    typedef double aux_t;
};

// K-major, no swizzle: LBO (k-chunk stride) = 128 B, SBO (8-row group stride) = 256 B
__device__ __forceinline__ uint64_t i8_desc(uint32_t smem_addr) { return kb_wgmma_desc(smem_addr, 128u, 256u); }
// d[64 points x R*2 W rows] (+)= A[64 x 32] B[R*2 x 32]^T in int32; scale_d = 0 overwrites d
template <int R>
__device__ __forceinline__ void i8_mma(uint32_t (&d)[R], uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(R == 12 || R == 16, "wgmma N = 24 or 32");
    if constexpr (R == 12) {
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "setp.ne.b32 p, %14, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n24k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, %12, %13, p;\n\t}\n"
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11])
                     : "l"(da), "l"(db), "r"(scale_d) : "memory");
    } else {
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "setp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                     : "l"(da), "l"(db), "r"(scale_d) : "memory");
    }
}

// S signed 7-bit digits of y = x * 2^-e (|y| < 1): x = 2^e * sum_s out[s] * 2^(-6-7s) + O(2^(e-7S)), out[s] in [-64, 64].
// One fp64 multiply + one round-to-nearest conversion to a 6+7(S-1)-bit integer, then balanced base-128 digits with
// integer ops (the digit loop used to be 4 fp64 instructions per slice on the pipe the RHS generators are bound by).
template <int S>
__device__ __forceinline__ void i8_slice(double x, int e, signed char (&out)[S]) {
    long long v = __double2ll_rn(scalbn(x, 6 + 7 * (S - 1) - e));      // |v| <= 2^(6+7(S-1))
#pragma unroll
    for (int s = S - 1; s >= 1; --s) {
        const int d = (int)((v + 64) & 127) - 64;                        // balanced digit in [-64, 63]
        out[s] = (signed char)d;
        v = (v - d) >> 7;                                                // exact: v - d is a multiple of 128
    }
    out[0] = (signed char)v;                                             // |v| <= 64
}
// the same with the scale 2^(6+7(S-1)-e) precomputed by the caller (one per prediction point)
template <int S>
__device__ __forceinline__ void i8_slice_scaled(double x, double scale, signed char (&out)[S]) {
    if (S <= 4) {                                                        // 27 bits + sign: 32-bit integer digits
        int v = __double2int_rn(x * scale);
#pragma unroll
        for (int s = S - 1; s >= 1; --s) {
            const int d = ((v + 64) & 127) - 64;
            out[s] = (signed char)d;
            v = (v - d) >> 7;
        }
        out[0] = (signed char)v;
    } else {
        long long v = __double2ll_rn(x * scale);
#pragma unroll
        for (int s = S - 1; s >= 1; --s) {
            const int d = (int)((v + 64) & 127) - 64;
            out[s] = (signed char)d;
            v = (v - d) >> 7;
        }
        out[0] = (signed char)v;
    }
}
// byte offset of element (r, k) inside one slice tile with `rows` rows (k in [0, 32))
__device__ __forceinline__ int i8_off(int r, int k) { return (r >> 3) * 256 + (k >> 4) * 128 + (r & 7) * 16 + (k & 15); }

__host__ __device__ __forceinline__ int i8_ktiles(int J, int n, int nk, int BN) {
    return ((J + 1) * BN > n) ? nk : min(nk, ((J + 1) * BN + I8_BK - 1) / I8_BK);
}

// ---- pack ---------------------------------------------------------------------------------------------
// rowscale[r] = 2^(ew_r - 12) with ew_r = exponent such that max_k |row_r[k]| * 2^-ew_r < 1
__global__ void __launch_bounds__(256) i8_rowscale_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                           const double* __restrict__ Uz, int nrows,
                                                           int* __restrict__ rowexp, double* __restrict__ rowscale) {
    int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    double m = 0.0;
    if (row < n) { for (int k = lane; k <= row; k += 32) m = fmax(m, fabs(W[(size_t)row * ld + k])); }
    else if (row < n + na) { for (int k = lane; k < n; k += 32) m = fmax(m, fabs(Uz[(size_t)(row - n) * n_pad + k])); }
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) {
        int e = 0;
        if (m > 0.0) { (void)frexp(m, &e); }        // m = f * 2^e, f in [0.5, 1)
        rowexp[row] = e;
        rowscale[row] = scalbn(1.0, e - 12);
    }
}

// tile (row block J, k stage t): S slices x (BN rows x 32 k) int8 in the wgmma operand layout
template <int S>
__global__ void __launch_bounds__(256) i8_pack_kernel(const double* __restrict__ W, int ld, int n, int n_pad, int na,
                                                       const double* __restrict__ Uz, const int* __restrict__ rowexp,
                                                       int nk, const long long* __restrict__ tile_off,
                                                       signed char* __restrict__ out) {
    typedef I8Cfg<S> C;
    const int J = blockIdx.y, t = blockIdx.x;
    if (t >= i8_ktiles(J, n, nk, C::BN)) return;
    signed char* o = out + (size_t)(tile_off[J] + t) * C::W_BYTES;
    for (int e = threadIdx.x; e < C::BN * I8_BK; e += 256) {
        const int rl = e >> 5, kl = e & 31;
        const int r = J * C::BN + rl, k = t * I8_BK + kl;
        double v = 0.0;
        if (r < n) { if (k <= r) v = W[(size_t)r * ld + k]; }
        else if (r < n + na) { if (k < n) v = Uz[(size_t)(r - n) * n_pad + k]; }
        signed char sl[S];
        i8_slice<S>(v, (r < n + na) ? rowexp[r] : 0, sl);
        const int off = i8_off(rl, kl);
#pragma unroll
        for (int s = 0; s < S; ++s) o[s * C::W_SLICE + off] = sl[s];
    }
}

// shifted covariance with the model as a run-time switch (uniform across the grid)
__device__ __forceinline__ double i8_cov_rhs(const VgParams& v, double d) {
    switch (v.model) {
        case KB200_VG_LINEAR: return kb_cov_rhs<KB200_VG_LINEAR>(v, d);
        case KB200_VG_POWER: return kb_cov_rhs<KB200_VG_POWER>(v, d);
        case KB200_VG_GAUSSIAN: return kb_cov_rhs<KB200_VG_GAUSSIAN>(v, d);
        case KB200_VG_EXPONENTIAL: return kb_cov_rhs<KB200_VG_EXPONENTIAL>(v, d);
        case KB200_VG_SPHERICAL: return kb_cov_rhs<KB200_VG_SPHERICAL>(v, d);
        case KB200_VG_TABLE: return kb_cov_rhs<KB200_VG_TABLE>(v, d);
        default: return kb_cov_rhs<KB200_VG_HOLE_EFFECT>(v, d);
    }
}

template <int S>
struct I8Arith : I8Cfg<S> {
    typedef I8Cfg<S> C;
    static constexpr int NH = C::BN / 2;                 // W rows per consumer warpgroup
    static constexpr int R = NH / 2;                     // int32 accumulators per thread and slice sum
    typedef uint32_t acc_t[S][R];                        // one accumulator set per slice-pair sum d = s + t
    __device__ __forceinline__ static int nrb(const SolvePtParams& P) { return (P.n + P.na + C::BN - 1) / C::BN; }
    __device__ __forceinline__ static int ktiles(const SolvePtParams& P, int J, int nk) { return i8_ktiles(J, P.n, nk, C::BN); }

    // exponent ec of this point's column: cmax * 2^-ec < 1. |c| <= c0 for the bounded models (gamma <= sill); for
    // linear / power / tabulated models a first pass finds the maximum.
    template <int DIM>
    __device__ __forceinline__ static int column_exponent(const SolvePtParams& P, int model, bool pvalid, double px,
                                                          double py, double pz) {
        double cmax = fabs(P.vg.c0);
        if (model == KB200_VG_LINEAR || model == KB200_VG_POWER || model == KB200_VG_TABLE) {
            if (pvalid)
                for (int k = 0; k < P.n; ++k) {
                    double d = kb_dist<DIM>(__ldg(P.ax + k), __ldg(P.ay + k), KB_HASZ(DIM) ? __ldg(P.az + k) : 0.0, px, py, pz);
                    cmax = fmax(cmax, fabs(i8_cov_rhs(P.vg, d)));
                }
        }
        int ec;
        (void)frexp(cmax * 1.0000001, &ec);
        return ec;
    }
    // the generator's slicing scale 2^(6+7(S-1)-ec) of a column
    __device__ __forceinline__ static double column_scale(int ec) { return scalbn(1.0, 6 + 7 * (S - 1) - ec); }

    // RHS of point pl for k stage t: S int8 slices per value
    template <int DIM>
    __device__ __forceinline__ static void rhs_stage(const SolvePtParams& P, unsigned char* ct, int t, int pl, bool pvalid,
                                                     double px, double py, double pz, double cscale) {
#pragma unroll 1
        for (int kc = 0; kc < 2; ++kc) {           // two 16-byte k-chunks per stage
            signed char sl[16][S];
#pragma unroll
            for (int kk = 0; kk < 16; ++kk) {
                const int k = t * I8_BK + kc * 16 + kk;
                double c = 0.0;
                if (pvalid && k < P.n) {
                    double d = kb_dist<DIM>(__ldg(P.ax + k), __ldg(P.ay + k), KB_HASZ(DIM) ? __ldg(P.az + k) : 0.0, px, py, pz);
                    c = i8_cov_rhs(P.vg, d);
                }
                i8_slice_scaled<S>(c, cscale, sl[kk]);
            }
            const int off = (pl >> 3) * 256 + kc * 128 + (pl & 7) * 16;
#pragma unroll
            for (int s = 0; s < S; ++s) {
                uint32_t w[4];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    w[q] = (uint32_t)(uint8_t)sl[4 * q][s] | ((uint32_t)(uint8_t)sl[4 * q + 1][s] << 8) |
                           ((uint32_t)(uint8_t)sl[4 * q + 2][s] << 16) | ((uint32_t)(uint8_t)sl[4 * q + 3][s] << 24);
                *reinterpret_cast<uint4*>(ct + s * I8_C_SLICE + off) = make_uint4(w[0], w[1], w[2], w[3]);
            }
        }
    }

    // as Tf32Arith::mma_stage; the S(S+1)/2 slice pairs with s + t < S
    __device__ __forceinline__ static void mma_stage(acc_t& acc, uint32_t sb, uint32_t hoff, bool first) {
        const uint32_t w = sb + hoff, c = sb + C::W_BYTES;
#pragma unroll
        for (int d = 0; d < S; ++d) {
#pragma unroll
            for (int sw = 0; sw <= d; ++sw) {
                const int sc = d - sw;                                     // slice of c
                i8_mma(acc[d], i8_desc(c + sc * I8_C_SLICE), i8_desc(w + sw * C::W_SLICE), (first && sw == 0) ? 0u : 1u);
            }
        }
    }

    // as Tf32Arith::epilogue after the exact recombination; pscale: the scales of points p0 and p0 + 8
    __device__ __forceinline__ static void epilogue(const SolvePtParams& P, acc_t& acc, int J, int h, int lane, int p0,
                                                    const double (&pscale)[2], double (&q)[2], double* auxs) {
#pragma unroll
        for (int d = 0; d < S; ++d)
#pragma unroll
            for (int i = 0; i < R; ++i) kb_reg_fence(acc[d][i]);
        const int rb = J * C::BN + h * NH + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const int r = rb + 8 * (i >> 2) + (i & 1), hh = (i >> 1) & 1;
            if (r < P.n + P.na) {
                // exact recombination: V = sum_d acc_d * 2^(7 (S-1-d)) fits in int64 (|acc_d| < 2^30, d = 0 has
                // one slice pair: < 2^27 * 2^35)
                long long V = 0;
#pragma unroll
                for (int d = 0; d < S; ++d) V = V * 128 + (long long)(int)acc[d][i];
                const double x = (double)V * (__ldg(P.rowscale + r) * pscale[hh]);
                if (r < P.n) q[hh] += x * x;
                else auxs[(r - P.n) * KB_WG_TM + p0 + 8 * hh] = x;
            }
        }
    }
    // 2^(ec - 7(S-1)): with the row scale 2^(ew - 12), the weight of the int64 recombination
    __device__ __forceinline__ static double point_scale(int ec) { return scalbn(1.0, ec - 7 * (S - 1)); }
};

// ==== the pipeline ================================================================================================
template <int DIM, class A>
__device__ __forceinline__ void solve_wgmma(const SolvePtParams& P) {
    constexpr int TM = KB_WG_TM;
    constexpr int NH = A::BN / 2;                                                      // W rows per consumer warpgroup
    typedef typename A::aux_t aux_t;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* stage_base = smem_raw;                                              // STAGES * STAGE_BYTES
    aux_t* auxs = reinterpret_cast<aux_t*>(smem_raw + (size_t)A::STAGES * A::STAGE_BYTES);   // KB_MAXAUX * 64
    double* qpart = reinterpret_cast<double*>(auxs + KB_MAXAUX * TM);                 // 2 warpgroups x 64 points
    int* pexp = reinterpret_cast<int*>(qpart + 2 * TM);                                // PEXP_INTS point exponents
    uint64_t* full = reinterpret_cast<uint64_t*>(pexp + A::PEXP_INTS);                 // STAGES
    uint64_t* empty = full + A::STAGES;                                                // STAGES
    uint64_t* gfull = empty + A::STAGES;                                               // 2
    uint64_t* gempty = gfull + 2;                                                      // 2

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nk = (P.n + A::BK - 1) / A::BK;
    const int nrb = A::nrb(P);
    const size_t sbuf = (size_t)nk * A::C_BYTES;                                       // one RHS column block
    unsigned char* scratch = reinterpret_cast<unsigned char*>(P.scratch) + (size_t)blockIdx.x * 2 * sbuf;
    const unsigned char* gt = reinterpret_cast<const unsigned char*>(P.tiles);
    const long long ntiles = (P.m + TM - 1) / TM;
    const int model = P.vg.model;

    if (tid == 0) {
        for (int s = 0; s < A::STAGES; ++s) { kb_mbar_init(&full[s], 1); kb_mbar_init(&empty[s], 2); }
        for (int b = 0; b < 2; ++b) { kb_mbar_init(&gfull[b], WG_GEN_THREADS); kb_mbar_init(&gempty[b], 1); }
        kb_fence_mbar_init();
    }
    __syncthreads();

    if (warp >= 9) {
        // ---------------- generators: RHS column block of the next tile -> scratch half b ----------------
        const int pl = (tid - 9 * 32) & (TM - 1);          // 0..63: point within the tile
        const int ks = (tid - 9 * 32) / TM;                // 0..2: k-stage residue handled by this thread
        uint32_t it = 0;
        for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const int b = (int)(it & 1);
            kb_mbar_wait(&gempty[b], ((it >> 1) & 1) ^ 1);         // the tile that used this buffer is finished
            unsigned char* sc = scratch + (size_t)b * sbuf;
            const long long pj = tile * TM + pl;
            const bool pvalid = pj < P.m;
            double px = 0.0, py = 0.0, pz = 0.0;
            if (pvalid) kb_load_point<DIM>(P.ps, P.an, pj, px, py, pz);
            double cscale = 0.0;
            if constexpr (A::PEXP_INTS > 0) {
                const int ec = A::template column_exponent<DIM>(P, model, pvalid, px, py, pz);
                if (ks == 0) pexp[b * TM + pl] = ec;
                cscale = A::column_scale(ec);
            }
            for (int t = ks; t < nk; t += WG_GEN_THREADS / TM)
                A::template rhs_stage<DIM>(P, sc + (size_t)t * A::C_BYTES, t, pl, pvalid, px, py, pz, cscale);
            kb_fence_publish_async();      // the bulk copies of this CTA read the ring
            kb_mbar_arrive(&gfull[b]);
        }
    } else if (warp == 8) {
        // ---------------- producer: W tiles + RHS tiles -> smem ring ----------------
        if (lane == 0) {
            const uint64_t pol_w = kb_policy_evict_last(), pol_c = kb_policy_evict_first();
            uint32_t gg = 0, it = 0;
            for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
                const int b = (int)(it & 1);
                const unsigned char* sc = scratch + (size_t)b * sbuf;
                kb_mbar_wait(&gfull[b], (it >> 1) & 1);
                long long tau = 0;
                for (int J = 0; J < nrb; ++J) {
                    const int kt = A::ktiles(P, J, nk);
                    for (int t = 0; t < kt; ++t, ++tau, ++gg) {
                        const int s = gg % A::STAGES;
                        kb_mbar_wait(&empty[s], (uint32_t)(((gg / A::STAGES) & 1) ^ 1));
                        kb_mbar_expect_tx(&full[s], A::STAGE_BYTES);
                        unsigned char* sb = stage_base + (size_t)s * A::STAGE_BYTES;
                        kb_bulk_g2s_hint(sb, gt + (size_t)tau * A::W_BYTES, A::W_BYTES, &full[s], pol_w);
                        kb_bulk_g2s_hint(sb + A::W_BYTES, sc + (size_t)t * A::C_BYTES, A::C_BYTES, &full[s], pol_c);
                    }
                }
            }
        }
    } else {
        // ---------------- consumers: warpgroup h owns W rows [NH h, NH h + NH) of every row block ----------------
        // accumulator element i = 4 j + 2 hh + e of (warp w of the group, lane): point 16 w + lane / 4 + 8 hh,
        // row NH h + 8 j + 2 (lane % 4) + e
        const int h = warp >> 2, wtid = tid & 127;
        const int p0 = (warp & 3) * 16 + (lane >> 2);       // points p0 and p0 + 8
        const uint32_t hoff = (uint32_t)h * (NH / 8) * A::SBO;
        uint32_t gg = 0, it = 0;
        for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const int b = (int)(it & 1);
            double pscale[2];
            if constexpr (A::PEXP_INTS > 0) {
                kb_mbar_wait(&gfull[b], (it >> 1) & 1);            // acquire the generators' pexp[b]
                for (int hh = 0; hh < 2; ++hh) pscale[hh] = A::point_scale(pexp[b * TM + p0 + 8 * hh]);
            }
            double q[2] = {0.0, 0.0};
            for (int J = 0; J < nrb; ++J) {
                const int kt = A::ktiles(P, J, nk);
                typename A::acc_t acc;
                for (int t = 0; t < kt; ++t, ++gg) {
                    const int s = gg % A::STAGES;
                    kb_mbar_wait(&full[s], (uint32_t)((gg / A::STAGES) & 1));
                    kb_wgmma_fence();
                    const uint32_t sb = kb_smem_u32(stage_base + (size_t)s * A::STAGE_BYTES);
                    A::mma_stage(acc, sb, hoff, t == 0);
                    kb_wgmma_commit();
                    kb_wgmma_wait<1>();                  // the previous stage has been read: hand it back
                    if (t > 0 && wtid == 0) kb_mbar_arrive(&empty[(gg - 1) % A::STAGES]);
                }
                kb_wgmma_wait<0>();
                if (wtid == 0) kb_mbar_arrive(&empty[(gg - 1) % A::STAGES]);
                A::epilogue(P, acc, J, h, lane, p0, pscale, q, auxs);
            }
            // the four lanes of a point hold interleaved rows; then the two warpgroups
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                q[hh] += __shfl_xor_sync(0xffffffffu, q[hh], 1);
                q[hh] += __shfl_xor_sync(0xffffffffu, q[hh], 2);
                if ((lane & 3) == 0) qpart[h * TM + p0 + 8 * hh] = q[hh];
            }
            kb_named_sync(1, WG_CONS_THREADS);
            // ---------------- phase F: finalize (DESIGN.md §3), thread = point ----------------
            if (tid < TM) {
                const long long pj = tile * TM + tid;
                if (pj < P.m) kb_finalize_point<DIM, aux_t>(P, pj, qpart[tid] + qpart[TM + tid], auxs + tid, TM);
            }
            kb_named_sync(1, WG_CONS_THREADS);
            if (tid == 0) kb_mbar_arrive(&gempty[b]);       // scratch half b (and pexp[b]) may be rewritten
        }
    }
}

template <int DIM, int MODEL>
__global__ void __launch_bounds__(WG_THREADS, 1) solve_kernel_tf32(const __grid_constant__ SolvePtParams P) {
    solve_wgmma<DIM, Tf32Arith<MODEL>>(P);
}
template <int S, int DIM>
__global__ void __launch_bounds__(WG_THREADS, 1) solve_kernel_i8(const __grid_constant__ SolvePtParams P) {
    solve_wgmma<DIM, I8Arith<S>>(P);
}

// ---- host side ---------------------------------------------------------------------------------------
template <class C> static size_t wg_smem() {
    return (size_t)C::STAGES * C::STAGE_BYTES + (size_t)KB_MAXAUX * KB_WG_TM * sizeof(typename C::aux_t) +
           2 * KB_WG_TM * sizeof(double) + C::PEXP_INTS * sizeof(int) + (2 * C::STAGES + 4) * sizeof(uint64_t) + 64;
}
template <class C> static size_t wg_scratch_bytes(int n, int grid) {
    return (size_t)grid * 2 * ((n + C::BK - 1) / C::BK) * C::C_BYTES;     // double-buffered
}

size_t kbk_solve_wgmma_scratch_bytes(int slices, int n, int grid) {
    size_t bytes = wg_scratch_bytes<Tf32Cfg>(n, grid);
    KbSlices::dispatch(slices, [&](auto S) { bytes = wg_scratch_bytes<I8Cfg<S>>(n, grid); return cudaSuccess; });
    return bytes;
}

cudaError_t kbk_solve_wgmma_init() {
    auto set = [](auto kernel, size_t smem) {
        return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    };
    return KbDims::for_each([&](auto D) {
        KB_CUDA_OK(KbModels::for_each([&](auto M) { return set(solve_kernel_tf32<D, M>, wg_smem<Tf32Cfg>()); }));
        return KbSlices::for_each([&](auto S) { return set(solve_kernel_i8<S, D>, wg_smem<I8Cfg<S>>()); });
    });
}

cudaError_t kbk_solve_wgmma(int slices, int dim, const SolvePtParams& p, int grid, cudaStream_t st) {
    auto launch = [&](auto kernel, size_t smem) {
        kernel<<<grid, WG_THREADS, smem, st>>>(p);
        return cudaGetLastError();
    };
    if (slices == 0)
        return KbDims::dispatch(dim, [&](auto D) {
            return KbModels::dispatch(p.vg.model, [&](auto M) { return launch(solve_kernel_tf32<D, M>, wg_smem<Tf32Cfg>()); });
        });
    if (p.vg.model < KB200_VG_LINEAR || p.vg.model > KB200_VG_TABLE) return cudaErrorInvalidValue;
    return KbSlices::dispatch(slices, [&](auto S) {
        return KbDims::dispatch(dim, [&](auto D) { return launch(solve_kernel_i8<S, D>, wg_smem<I8Cfg<S>>()); });
    });
}

// ---- pack entry points -------------------------------------------------------------------------------
cudaError_t kbk_pack_tf32(const double* W, int ld, int n, int n_pad, int na, const double* Uz, const PackMap& pm,
                          void* out, cudaStream_t st) {
    pack_tf32_kernel<<<kb_pack_grid(pm), 256, 0, st>>>(W, ld, n, n_pad, na, Uz, pm, (float*)out);
    return cudaGetLastError();
}

bool kbk_i8_valid_slices(int S) { return KbSlices::dispatch(S, [](auto) { return cudaSuccess; }) == cudaSuccess; }
int kbk_i8_nrb(int S, int n, int na) { return (n + na + i8_bn(S) - 1) / i8_bn(S); }
int kbk_i8_rows(int S, int n, int na) { return kbk_i8_nrb(S, n, na) * i8_bn(S); }
long long kbk_i8_total_tiles(int S, int n, int na, long long* tile_off /* [nrb+1] or null */) {
    int nk = (n + I8_BK - 1) / I8_BK, nrb = kbk_i8_nrb(S, n, na);
    long long off = 0;
    for (int J = 0; J < nrb; ++J) { if (tile_off) tile_off[J] = off; off += i8_ktiles(J, n, nk, i8_bn(S)); }
    if (tile_off) tile_off[nrb] = off;
    return off;
}
size_t kbk_i8_tile_bytes(int S) { return (size_t)S * i8_bn(S) * I8_BK; }

// W (+ dual rows) -> row scales + int8 slice tiles. tile_off_dev: device copy of the per-row-block tile offsets.
cudaError_t kbk_pack_i8(int S, const double* W, int ld, int n, int n_pad, int na, const double* Uz,
                        int* rowexp, double* rowscale, const long long* tile_off_dev, void* out, cudaStream_t st) {
    int nrb = kbk_i8_nrb(S, n, na), nk = (n + I8_BK - 1) / I8_BK;
    int nrows = nrb * i8_bn(S);
    i8_rowscale_kernel<<<(nrows + 7) / 8, 256, 0, st>>>(W, ld, n, n_pad, na, Uz, nrows, rowexp, rowscale);
    return KbSlices::dispatch(S, [&](auto SL) {
        i8_pack_kernel<SL><<<dim3(nk, nrb), 256, 0, st>>>(W, ld, n, n_pad, na, Uz, rowexp, nk, tile_off_dev, (signed char*)out);
        return cudaGetLastError();
    });
}
