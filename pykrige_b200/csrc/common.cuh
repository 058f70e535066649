// common.cuh — shared device helpers for libkrige_b200 (sm_90a).
//
// Semantics follow the reference (cited per function); the code is written from
// scratch for the GPU.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/krige_b200.h"

#define KB_WARP 32

// ---- tile geometry of the fused solve kernel (see DESIGN.md §4) -------------
#define KB_BM 256      // rows of W per CTA tile
#define KB_TN 64       // prediction points per CTA tile
#define KB_BK 16       // k extent of one staged tile
#define KB_NB 64       // Cholesky / triangular-inverse block size
#define KB_MAXAUX (KB200_MAX_DRIFT + 2)   // dual rows: U (K+1 columns) + zeta
#define KB_MAXRB 128   // max row blocks (n_pad/KB_BM + 1) -> n up to ~32k

struct VgParams {
    int model;
    double p0, p1, p2;   // stored (psill-form) parameters, variogram_models.py:25-81
    double inv_a;        // host-computed reciprocal of the model's distance scale: 1/(range/3) (exponential, hole-effect),
                         // 1/(4 range/7)^2 (gaussian), 1/range (spherical): one fp64 division less per evaluation
    double c0;           // covariance shift (see DESIGN.md §3): cov(d) = c0 - gamma(d)
    double eps;          // exact-hit cutoff, ok.py:177
    int exact;           // ok.py:671-672
    // KB200_VG_TABLE: (value, slope per node) pairs at sqrt-spaced nodes, see kb200_set_variogram_table
    const double2* tab;
    double tab_inv_h;    // (n_nodes - 1) / sqrt(dmax)
    int tab_n;
};

// Affine anisotropy map (core.py:120-193): adj = Mt (p - c) + c.
// Explicit _rn intrinsics: data points and prediction points must go through the
// *identical* instruction sequence so that coincident inputs give d == 0 exactly
// (exact-hit semantics, ok.py:665-672) regardless of how nvcc contracts FMAs.
struct Aniso {
    double m[9];
    double c[3];
};

// DIM = 2, 3: euclidean coordinates.  DIM = KB_GEO (4): coordinates_type='geographic' (ok.py:292-306):
// (x, y) = (lon, lat) in degrees, no anisotropy; on the device a point is its unit vector on the sphere
// (the same conversion the reference uses for its kd-tree, ok.py:936-956) and distances are great-circle
// degrees (core.py:36-97: atan2(|u x v|, u . v), which is that formula written with unit vectors).
#define KB_GEO 4
#define KB_HASZ(DIM) ((DIM) >= 3)

template <int DIM>
__device__ __forceinline__ void kb_adjust(const Aniso& a, double x, double y, double z,
                                          double& ox, double& oy, double& oz) {
    if (DIM == KB_GEO) {
        const double rad = 0.017453292519943295;     // pi / 180
        double slon, clon, slat, clat;
        sincos(x * rad, &slon, &clon);
        sincos(y * rad, &slat, &clat);
        ox = clon * clat; oy = slon * clat; oz = slat;
        return;
    }
    double dx = __dsub_rn(x, a.c[0]);
    double dy = __dsub_rn(y, a.c[1]);
    if (DIM == 2) {
        double rx = __dadd_rn(__dmul_rn(a.m[0], dx), __dmul_rn(a.m[1], dy));
        double ry = __dadd_rn(__dmul_rn(a.m[2], dx), __dmul_rn(a.m[3], dy));
        ox = __dadd_rn(rx, a.c[0]);
        oy = __dadd_rn(ry, a.c[1]);
        oz = 0.0;
    } else {
        double dz = __dsub_rn(z, a.c[2]);
        double rx = __dadd_rn(__dadd_rn(__dmul_rn(a.m[0], dx), __dmul_rn(a.m[1], dy)), __dmul_rn(a.m[2], dz));
        double ry = __dadd_rn(__dadd_rn(__dmul_rn(a.m[3], dx), __dmul_rn(a.m[4], dy)), __dmul_rn(a.m[5], dz));
        double rz = __dadd_rn(__dadd_rn(__dmul_rn(a.m[6], dx), __dmul_rn(a.m[7], dy)), __dmul_rn(a.m[8], dz));
        ox = __dadd_rn(rx, a.c[0]);
        oy = __dadd_rn(ry, a.c[1]);
        oz = __dadd_rn(rz, a.c[2]);
    }
}

// exp(x) for x <= 0 (the variogram models only evaluate decaying exponentials): k = rint(x log2 e), r = x - k ln 2
// (Cody-Waite with the two fdlibm constants), exp(r) by the degree-13 Taylor polynomial on |r| <= ln 2 / 2 (truncation
// 4e-18; Horner form: a few ulp), scaling by 2^k through the exponent field. About half the instructions of exp():
// no overflow / NaN / denormal handling (x < -708 returns 0; the arguments are finite distances over a range), and the
// evaluation is on the critical path of the moving window (2016 per point) and of every RHS generator.
// exp(0) is exactly 1, so gamma(0) stays exactly the nugget.
__device__ __forceinline__ double kb_exp_neg(double x) {
    const double kd = rint(x * 1.4426950408889634);
    double r = fma(kd, -6.93147180369123816490e-01, x);
    r = fma(kd, -1.90821492927058770002e-10, r);
    double p = 1.6059043836821613e-10;            // 1/13!
    p = fma(p, r, 2.08767569878681e-09);          // 1/12!
    p = fma(p, r, 2.505210838544172e-08);         // 1/11!
    p = fma(p, r, 2.755731922398589e-07);         // 1/10!
    p = fma(p, r, 2.7557319223985893e-06);        // 1/9!
    p = fma(p, r, 2.48015873015873e-05);          // 1/8!
    p = fma(p, r, 1.984126984126984e-04);         // 1/7!
    p = fma(p, r, 1.388888888888889e-03);         // 1/6!
    p = fma(p, r, 8.333333333333333e-03);         // 1/5!
    p = fma(p, r, 4.1666666666666664e-02);        // 1/4!
    p = fma(p, r, 1.6666666666666666e-01);        // 1/3!
    p = fma(p, r, 0.5);
    p = fma(p, r, 1.0);
    p = fma(p, r, 1.0);
    const int k = (int)kd;                         // in [-1022, 0] for x >= -708
    const double v = __hiloint2double(__double2hiint(p) + (k << 20), __double2loint(p));
    return x < -708.0 ? 0.0 : v;
}

// gamma(d) for the six built-in models, variogram_models.py:25-81 (same closed
// forms; docs/source/variogram_models.rst:8-44), and the tabulated model for custom callables.
template <int MODEL>
__device__ __forceinline__ double kb_gamma(const VgParams& v, double d) {
    if (MODEL == KB200_VG_LINEAR) {
        return v.p0 * d + v.p1;                                       // slope*d + nugget
    } else if (MODEL == KB200_VG_POWER) {
        return v.p0 * pow(d, v.p1) + v.p2;                            // scale*d^exponent + nugget
    } else if (MODEL == KB200_VG_GAUSSIAN) {
        return v.p0 * (1.0 - kb_exp_neg(-(d * d) * v.inv_a)) + v.p2;
    } else if (MODEL == KB200_VG_EXPONENTIAL) {
        return v.p0 * (1.0 - kb_exp_neg(-d * v.inv_a)) + v.p2;
    } else if (MODEL == KB200_VG_SPHERICAL) {
        if (d <= v.p1) {
            double q = d * v.inv_a;
            return v.p0 * (1.5 * q - 0.5 * q * q * q) + v.p2;
        }
        return v.p0 + v.p2;
    } else if (MODEL == KB200_VG_TABLE) {
        // tabulated callable: cubic Hermite in u = sqrt(d) * (n-1)/sqrt(dmax); one 32-byte read per evaluation
        const double u = sqrt(d) * v.tab_inv_h;
        int i = (int)u;
        i = i > v.tab_n - 2 ? v.tab_n - 2 : i;
        const double t = u - (double)i;
        const double2 a = __ldg(v.tab + i), b = __ldg(v.tab + i + 1);
        const double t2 = t * t, t3 = t2 * t;
        return (2.0 * t3 - 3.0 * t2 + 1.0) * a.x + (t3 - 2.0 * t2 + t) * a.y
             + (3.0 * t2 - 2.0 * t3) * b.x + (t3 - t2) * b.y;
    } else {  // hole-effect
        double q = d * v.inv_a;
        return v.p0 * (1.0 - (1.0 - q) * kb_exp_neg(-q)) + v.p2;
    }
}

// Shifted covariance of a (data, prediction point) pair: the RHS entry.
//   reference: b = -gamma(d), b = 0 on an exact hit when exact_values (ok.py:669-672)
//   here:      c = c0 + b  (DESIGN.md §3)
template <int MODEL>
__device__ __forceinline__ double kb_cov_rhs(const VgParams& v, double d) {
    if (v.exact && fabs(d) <= v.eps) return v.c0;
    return v.c0 - kb_gamma<MODEL>(v, d);
}

template <int DIM>
__device__ __forceinline__ double kb_dist(double ax, double ay, double az,
                                          double bx, double by, double bz) {
    if (DIM == KB_GEO) {
        // great-circle distance in degrees between unit vectors; coincident points give exactly 0
        double cx = __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by));
        double cy = __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz));
        double cz = __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));
        double s = sqrt(cx * cx + cy * cy + cz * cz);
        double c = ax * bx + ay * by + az * bz;
        return atan2(s, c) * 57.29577951308232;      // 180 / pi
    }
    double dx = ax - bx, dy = ay - by;
    double s = dx * dx + dy * dy;
    if (DIM == 3) { double dz = az - bz; s += dz * dz; }
    return sqrt(s);
}

// Where prediction points come from: explicit arrays or a rectangular grid
// (2-D: x fastest, ok.py:864-866; 3-D: (z,y,x) 'ij' order, x fastest, ok3d.py:863-866).
struct PointSource {
    int grid;                 // 0 = explicit arrays, 1 = grid axes
    const double* px; const double* py; const double* pz;   // explicit (original coords)
    const double* gx; const double* gy; const double* gz;   // axes
    long long nx, ny, nz;
    long long first;          // offset of point 0 of this launch in the flattened grid / arrays
};

template <int DIM>
__device__ __forceinline__ void kb_load_point_raw(const PointSource& ps, long long p,
                                                  double& rx, double& ry, double& rz) {
    rz = 0.0;
    long long q = p + ps.first;
    if (ps.grid) {
        long long ix = q % ps.nx;
        long long r = q / ps.nx;
        long long iy = r % ps.ny;
        rx = ps.gx[ix];
        ry = ps.gy[iy];
        if (DIM == 3) { long long iz = r / ps.ny; rz = ps.gz[iz]; }
    } else {
        rx = ps.px[q];
        ry = ps.py[q];
        if (DIM == 3) rz = ps.pz[q];
    }
}

template <int DIM>
__device__ __forceinline__ void kb_load_point(const PointSource& ps, const Aniso& an, long long p,
                                              double& x, double& y, double& z) {
    double rx, ry, rz;
    kb_load_point_raw<DIM>(ps, p, rx, ry, rz);
    kb_adjust<DIM>(an, rx, ry, rz, x, y, z);
}

// ---- mma.sync m8n8k4 f64 (DMMA): the fp64 tensor path on sm_90a -------------
// A 8x4 row: lane holds A[lane>>2][lane&3]; B 4x8 col: lane holds B[lane&3][lane>>2];
// C 8x8: lane holds C[lane>>2][2*(lane&3) + {0,1}].
__device__ __forceinline__ void kb_dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// ---- L2 cache policies for the bulk copies of the solve kernels ----------------------------------------------
// The factor tile stream (W) is read by every CTA for every point tile: keep what L2 holds of it (evict_last; DESIGN.md §2
// has the measurement on H100, where W outgrows L2 above N ~ 3500). The per-CTA
// RHS scratch ring is private, far larger than L2 in total (one ring per SM, n x tile bytes each) and dead after one
// tile: evict_first, so that it does not push W out.
__device__ __forceinline__ uint64_t kb_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t kb_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(p));
    return p;
}
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP) with an L2 cache policy
__device__ __forceinline__ void kb_bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n"
                 :: "r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes),
                    "r"((uint32_t)__cvta_generic_to_shared(bar)), "l"(policy) : "memory");
}

// ---- warpgroup MMA (wgmma, sm_90a) helpers for the tensor-core solve kernels ---------------------------------
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

#define KB_CUDA_OK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) return _e; } while (0)
