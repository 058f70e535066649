// pinv.cu — pseudo_inv=True: the kriging matrix is inverted with a pseudo-inverse
// (`P_INV[pseudo_inv_type](a)`, core.py:33; ok.py:660-661, uk.py:932-933, ok3d.py:634-635, uk3d.py:749-750),
// which averages redundant points instead of failing on the singular system.
//
// Device algorithm: the bordered matrix A = [[-Gamma, F], [F^T, 0]] (gamma form, zero diagonal, raw drift
// columns — exactly the reference's `a`, so the truncation acts on the same spectrum) is decomposed by a
// one-sided (Hestenes) Jacobi SVD: B = A V with V a product of plane rotations, iterated until the columns
// of B are mutually orthogonal; then A = (B S^-1) S V^T and
//     A^+ = sum_{s_p > cutoff} v_p b_p^T / s_p^2,   cutoff = nt * eps * s_max   (scipy.linalg.pinv's default).
// pinv and pinvh are the same operator for a symmetric matrix; both map to this path.
// The prediction then runs on the quadratic-form variant of the solve kernel (gform = 2):
//     sigma^2 = -b^T A^+ b,  z = Z^T (A^+ b)[:n],  b = [-gamma(d); f(p)]   (ok.py:674-681).
#include <vector>
#include "common.cuh"
#include "kernels.h"

#define PJ_T 256

// 1-D bulk copies through the TMA engine (common.cuh; SASS UBLKCP): a single CTA per SM cannot keep enough plain
// loads in flight to stream its columns at HBM speed.
__device__ __forceinline__ void pj_bulk_s2g(void* dst, const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n"
                 :: "l"(dst), "r"(kb_smem_u32(src)), "r"(bytes) : "memory");
}

// Bt (row p = column p of B) := A, Vt := I. C: assembled with c0 = 0 (lower triangle valid, zero
// diagonal); Fz: drift columns 0..K-1 then ones (column K), each n_pad long.
__global__ void pinv_build_kernel(int n, int K1, int nt, int ld, const double* __restrict__ C, int ldc,
                                  const double* __restrict__ Fz, int n_pad,
                                  double* __restrict__ Bt, double* __restrict__ Vt) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y;
    if (j >= ld || i >= nt) return;
    double v = 0.0;
    if (j < nt) {
        if (i < n && j < n) v = i == j ? 0.0 : (i > j ? C[(size_t)i * ldc + j] : C[(size_t)j * ldc + i]);
        else if (i < n) v = Fz[(size_t)(j - n) * n_pad + i];
        else if (j < n) v = Fz[(size_t)(i - n) * n_pad + j];
    }
    Bt[(size_t)i * ld + j] = v;
    Vt[(size_t)i * ld + j] = (i == j) ? 1.0 : 0.0;
}

__device__ __forceinline__ void pj_reduce3(double& a, double& b, double& g, double* red) {
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
        g += __shfl_xor_sync(0xffffffffu, g, o);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { red[w] = a; red[8 + w] = b; red[16 + w] = g; }
    __syncthreads();
    a = b = g = 0.0;
    for (int q = 0; q < PJ_T / 32; ++q) { a += red[q]; b += red[8 + q]; g += red[16 + q]; }   // same order in every thread
}

// One round of the round-robin ordering over column BLOCKS: the columns are cut into blocks of NC/2; a CTA
// takes a pair of blocks (NC columns), stages them in shared memory and runs one full inner tournament on
// them: NC-1 steps of NC/2 disjoint column pairs, each pair owned by a group of 8/(NC/2) warps (exact
// one-sided rotations: three dot products and one plane rotation per pair, all from shared memory). The
// columns are written back once; the accumulated NC x NC rotation is then applied to the same columns of V
// in one streaming pass. Per pair of columns this moves 8 nt / (NC - 1) doubles instead of 8 nt (NC = 2 is
// the plain one-sided Jacobi). mb = number of blocks (even, or 1).
template <int NC>
__global__ void __launch_bounds__(PJ_T) pinv_jacobi_round_kernel(int nt, int ld, double* __restrict__ Bt,
                                                                 double* __restrict__ Vt, int r, int mb,
                                                                 double tol, double thr2, int* __restrict__ counter) {
    extern __shared__ __align__(128) double pj_sm[];      // NC columns of B, stride nts
    constexpr int HB = NC / 2;             // columns per block = pairs per inner step
    constexpr int WPP = (PJ_T / 32) / HB;  // warps per pair
    constexpr int GS = 32 * WPP;           // threads per pair
    __shared__ double part[HB][WPP][3];
    __shared__ double M[NC][NC];           // rows_new = M rows_old (accumulated rotations)
    __shared__ int scol[NC];
    __shared__ int any_rot;
    __shared__ __align__(8) uint64_t bar;
    const int k = blockIdx.x, tid = threadIdx.x;
    const int grp = tid / GS, lg = tid % GS, wig = lg >> 5, lane = tid & 31;
    if (tid < NC) {
        int I, J;
        if (mb == 1) { I = 0; J = 0; }
        else if (k == 0) { I = mb - 1; J = r; }
        else { I = (r + k) % (mb - 1); J = (r - k + (mb - 1)) % (mb - 1); }
        const int c = (tid < HB ? I * HB + tid : J * HB + (tid - HB));
        scol[tid] = (c < nt && !(mb == 1 && tid >= HB)) ? c : -1;
    }
    if (tid < NC * NC) M[tid / NC][tid % NC] = (tid / NC == tid % NC) ? 1.0 : 0.0;
    if (tid == 0) {
        any_rot = 0;
        kb_mbar_init(&bar, 1);
        kb_fence_mbar_init();
    }
    __syncthreads();
    const int nts = (nt + 1) & ~1;                       // column stride in shared memory (16-byte multiple)
    const uint32_t cb = (uint32_t)nts * 8u;              // bytes per column copy (<= ld * 8: rows are padded to 8)
    if (tid == 0) {
        uint32_t total = 0;
        for (int a = 0; a < NC; ++a) if (scol[a] >= 0) total += cb;
        kb_mbar_expect_tx(&bar, total);
        for (int a = 0; a < NC; ++a)
            if (scol[a] >= 0) kb_bulk_g2s(pj_sm + (size_t)a * nts, Bt + (size_t)scol[a] * ld, cb, &bar);
    }
    kb_mbar_wait(&bar, 0);
    for (int step = 0; step < NC - 1; ++step) {
        // inner round robin on NC players: group 0 pairs (NC-1, step), group g pairs ((step+g), (step-g)) mod NC-1
        int a, c;
        if (NC == 2) { a = 0; c = 1; }
        else if (grp == 0) { a = NC - 1; c = step; }
        else { a = (step + grp) % (NC - 1); c = (step - grp + (NC - 1)) % (NC - 1); }
        if (a > c) { const int t = a; a = c; c = t; }
        const bool valid = scol[a] >= 0 && scol[c] >= 0;
        double* xa = pj_sm + (size_t)a * nts;
        double* xc = pj_sm + (size_t)c * nts;
        double al = 0.0, be = 0.0, ga = 0.0;
        if (valid)
            for (int i = lg; i < nt; i += GS) {
                const double x = xa[i], y = xc[i];
                al += x * x; be += y * y; ga += x * y;
            }
        for (int o = 16; o > 0; o >>= 1) {
            al += __shfl_xor_sync(0xffffffffu, al, o);
            be += __shfl_xor_sync(0xffffffffu, be, o);
            ga += __shfl_xor_sync(0xffffffffu, ga, o);
        }
        if (lane == 0) { part[grp][wig][0] = al; part[grp][wig][1] = be; part[grp][wig][2] = ga; }
        __syncthreads();
        al = be = ga = 0.0;
#pragma unroll
        for (int w = 0; w < WPP; ++w) { al += part[grp][w][0]; be += part[grp][w][1]; ga += part[grp][w][2]; }
        const double ab = al * be;
        if (valid && ab > 1e-280 && fabs(ga) > tol * sqrt(ab)) {                  // uniform within the group
            const double zeta = (be - al) / (2.0 * ga);
            const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
            for (int i = lg; i < nt; i += GS) {
                const double x = xa[i], y = xc[i];
                xa[i] = cs * x - sn * y;
                xc[i] = sn * x + cs * y;
            }
            if (lg < NC) {
                const double x = M[a][lg], y = M[c][lg];
                M[a][lg] = cs * x - sn * y;
                M[c][lg] = sn * x + cs * y;
            }
            if (lg == 0) {
                any_rot = 1;
                if (al >= thr2 && be >= thr2) atomicAdd(counter, 1);              // only live columns count
            }
        }
        __syncthreads();                   // the next step pairs the columns differently
    }
    if (!any_rot) return;
    // rotated columns: generic-proxy writes to shared memory -> bulk stores (async proxy)
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();
    if (tid == 0) {
        for (int a = 0; a < NC; ++a)
            if (scol[a] >= 0) pj_bulk_s2g(Bt + (size_t)scol[a] * ld, pj_sm + (size_t)a * nts, cb);
        asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
    }
    // V: rows_new = M rows_old, streamed; UV elements per thread and trip keep >= 16 loads in flight
    constexpr int UV = NC >= 16 ? 1 : 16 / NC;
    for (int i0 = tid; i0 < nt; i0 += PJ_T * UV) {
        double v[UV][NC];
#pragma unroll
        for (int u = 0; u < UV; ++u) {
            const int i = i0 + u * PJ_T;
#pragma unroll
            for (int a = 0; a < NC; ++a) v[u][a] = (i < nt && scol[a] >= 0) ? Vt[(size_t)scol[a] * ld + i] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < UV; ++u) {
            const int i = i0 + u * PJ_T;
            if (i < nt) {
#pragma unroll
                for (int a = 0; a < NC; ++a) {
                    double acc = 0.0;
#pragma unroll
                    for (int c = 0; c < NC; ++c) acc = fma(M[a][c], v[u][c], acc);
                    if (scol[a] >= 0) Vt[(size_t)scol[a] * ld + i] = acc;
                }
            }
        }
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory");   // the stores have left shared memory and landed
}

// s2[p] = ||b_p||^2
__global__ void __launch_bounds__(PJ_T) pinv_sigma_kernel(int nt, int ld, const double* __restrict__ Bt,
                                                          double* __restrict__ s2) {
    __shared__ double red[24];
    const double* bp = Bt + (size_t)blockIdx.x * ld;
    double a = 0.0, b = 0.0, g = 0.0;
    for (int i = threadIdx.x; i < nt; i += PJ_T) { const double x = bp[i]; a += x * x; }
    pj_reduce3(a, b, g, red);
    if (threadIdx.x == 0) s2[blockIdx.x] = a;
}

// G[i][j] = sum_p dinv[p] Vt[p][i] Bt[p][j]   (64 x 64 tile per CTA, 4 x 4 per thread)
__global__ void __launch_bounds__(256) pinv_gemm_kernel(int nt, int ld, const double* __restrict__ Vt,
                                                        const double* __restrict__ Bt, const double* __restrict__ dinv,
                                                        double* __restrict__ G) {
    __shared__ double As[16][64], Bs[16][64];
    const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int p0 = 0; p0 < nt; p0 += 16) {
        for (int e = threadIdx.x; e < 16 * 64; e += 256) {
            const int pp = e >> 6, c = e & 63, p = p0 + pp;
            double va = 0.0, vb = 0.0;
            if (p < nt) {
                const double d = dinv[p];
                if (d != 0.0) {
                    if (i0 + c < nt) va = d * Vt[(size_t)p * ld + i0 + c];
                    if (j0 + c < nt) vb = Bt[(size_t)p * ld + j0 + c];
                }
            }
            As[pp][c] = va; Bs[pp][c] = vb;
        }
        __syncthreads();
#pragma unroll
        for (int pp = 0; pp < 16; ++pp) {
            double av[4], bv[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) { av[a] = As[pp][ty * 4 + a]; bv[a] = Bs[pp][tx * 4 + a]; }
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] += av[a] * bv[b];
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int i = i0 + ty * 4 + a, j = j0 + tx * 4 + b;
            if (i < nt && j < ld) G[(size_t)i * ld + j] = j < nt ? acc[a][b] : 0.0;
        }
}

// A^+ is symmetric; remove the rounding asymmetry of the product: G := (G + G^T)/2 (lower -> both).
__global__ void pinv_sym_kernel(int nt, int ld, double* __restrict__ G) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y;
    if (i < nt && j < i) {
        const double v = 0.5 * (G[(size_t)i * ld + j] + G[(size_t)j * ld + i]);
        G[(size_t)i * ld + j] = v;
        G[(size_t)j * ld + i] = v;
    }
}

// Split A^+ = [[G11, G12], [G21, G22]] into what the solve kernel consumes (one warp per row r of A^+):
//   r <  n : Cout row r = G11[r][:] (n_pad x ldc layout of the fallback path); Uz row K1 entry r = (G11 Z)[r]
//   r >= n : Uz row (r-n) = G21[r-n][:n]; consts[a*K1 + b] = G22; consts[K1*K1 + a] = (G21 Z)[a]
__global__ void __launch_bounds__(256) pinv_split_kernel(int n, int K1, int nt, int ld, const double* __restrict__ G,
                                                         const double* __restrict__ values,
                                                         double* __restrict__ Cout, int ldc, int n_pad,
                                                         double* __restrict__ Uz, double* __restrict__ consts) {
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= nt) return;
    const double* g = G + (size_t)r * ld;
    double dot = 0.0;
    for (int k = lane; k < n; k += 32) {
        const double v = g[k];
        dot += v * values[k];
        if (r < n) Cout[(size_t)r * ldc + k] = v;
        else Uz[(size_t)(r - n) * n_pad + k] = v;
    }
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (r < n) {
        for (int k = n + lane; k < ldc; k += 32) Cout[(size_t)r * ldc + k] = 0.0;
        if (lane == 0) Uz[(size_t)K1 * n_pad + r] = dot;
    } else {
        const int a = r - n;
        for (int k = n + lane; k < n_pad; k += 32) Uz[(size_t)a * n_pad + k] = 0.0;
        if (lane < K1) consts[a * K1 + lane] = g[n + lane];
        if (lane == 0) consts[K1 * K1 + a] = dot;
    }
}

__global__ void pinv_pad_kernel(int n, int K1, int n_pad, int ldc, double* __restrict__ Cout, double* __restrict__ Uz) {
    // rows n..n_pad-1 of Cout and the tail of Uz row K1 are zero
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = n + blockIdx.y;
    if (i < n_pad && j < ldc) Cout[(size_t)i * ldc + j] = 0.0;
    if (blockIdx.y == 0 && j >= n && j < n_pad) Uz[(size_t)K1 * n_pad + j] = 0.0;
}

int kbk_pinv_max_nt() { return (227 * 1024 - 4096) / 16 - 1; }
size_t kbk_pinv_workspace_doubles(int nt) {
    const size_t ld = ((size_t)nt + 7) / 8 * 8;
    return 3 * (size_t)nt * ld + 2 * (size_t)nt + 64;
}

cudaError_t kbk_pinv_init() {
    const int mx = 227 * 1024 - 4096;
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(pinv_jacobi_round_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(pinv_jacobi_round_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(pinv_jacobi_round_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx)) != cudaSuccess) return e;
    return cudaFuncSetAttribute(pinv_jacobi_round_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
}

// Runs the whole pseudo-inverse. C (n_pad x ldc): assembled with c0 = 0; on return it holds G11.
// work: kbk_pinv_workspace_doubles(nt) doubles. counter: device int. Returns the number of sweeps in
// *sweeps (negative: not converged), the live rank in *rank.
cudaError_t kbk_pinv(int n, int K1, int n_pad, double* C, int ldc, const double* Fz, const double* values,
                     double* Uz, double* consts, double* work, int* counter, cudaStream_t st,
                     int* launches, int* sweeps, int* rank) {
    const int nt = n + K1;
    const int ld = (nt + 7) / 8 * 8;
    double* Bt = work;
    double* Vt = Bt + (size_t)nt * ld;
    double* G = Vt + (size_t)nt * ld;
    double* s2 = G + (size_t)nt * ld;
    double* dinv = s2 + nt;
    pinv_build_kernel<<<dim3((ld + 255) / 256, nt), 256, 0, st>>>(n, K1, nt, ld, C, ldc, Fz, n_pad, Bt, Vt);
    ++*launches;
    // live threshold for the convergence count: columns below nt*eps*||A||_F are null space
    pinv_sigma_kernel<<<nt, PJ_T, 0, st>>>(nt, ld, Bt, s2);
    ++*launches;
    std::vector<double> hs(nt);
    cudaError_t e = cudaMemcpyAsync(hs.data(), s2, (size_t)nt * 8, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    double fro2 = 0.0;
    for (double v : hs) fro2 += v;
    const double epsm = 2.220446049250313e-16;
    const double thr2 = (nt * epsm) * (nt * epsm) * fro2;
    const double tol = nt * epsm > 1e-15 ? nt * epsm : 1e-15;     // dgesvj-style orthogonality threshold
    // columns per CTA: as many as fit in shared memory (16 / 8 / 4 / 2)
    const size_t smax = 227 * 1024 - 4096;
    int nc = 16;
    const size_t nts_h = ((size_t)nt + 1) & ~(size_t)1;  // column stride in shared memory
    while (nc > 2 && (size_t)nc * nts_h * sizeof(double) > smax) nc /= 2;
    const int hb = nc / 2;
    int mb = (nt + hb - 1) / hb;                        // column blocks
    if (mb > 1) mb = (mb + 1) / 2 * 2;                  // even number of players (the last may be a dummy)
    const int rounds = mb > 1 ? mb - 1 : 1, ctas = mb > 1 ? mb / 2 : 1;
    const size_t sm = (size_t)nc * nts_h * sizeof(double);
    *sweeps = -1;
    for (int sweep = 0; sweep < 40 && nt > 1; ++sweep) {
        if ((e = cudaMemsetAsync(counter, 0, sizeof(int), st)) != cudaSuccess) return e;
        for (int r = 0; r < rounds; ++r) {
            if (nc == 16) pinv_jacobi_round_kernel<16><<<ctas, PJ_T, sm, st>>>(nt, ld, Bt, Vt, r, mb, tol, thr2, counter);
            else if (nc == 8) pinv_jacobi_round_kernel<8><<<ctas, PJ_T, sm, st>>>(nt, ld, Bt, Vt, r, mb, tol, thr2, counter);
            else if (nc == 4) pinv_jacobi_round_kernel<4><<<ctas, PJ_T, sm, st>>>(nt, ld, Bt, Vt, r, mb, tol, thr2, counter);
            else pinv_jacobi_round_kernel<2><<<ctas, PJ_T, sm, st>>>(nt, ld, Bt, Vt, r, mb, tol, thr2, counter);
        }
        *launches += rounds;
        int rot = 0;
        if ((e = cudaMemcpyAsync(&rot, counter, sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
        if (rot == 0) { *sweeps = sweep + 1; break; }
    }
    if (nt == 1) *sweeps = 0;
    pinv_sigma_kernel<<<nt, PJ_T, 0, st>>>(nt, ld, Bt, s2);
    ++*launches;
    if ((e = cudaMemcpyAsync(hs.data(), s2, (size_t)nt * 8, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    double smax2 = 0.0;
    for (double v : hs) smax2 = v > smax2 ? v : smax2;
    const double cut = nt * epsm * sqrt(smax2);          // scipy.linalg.pinv: rtol = max(M, N) * eps
    int live = 0;
    for (double& v : hs) {
        if (sqrt(v) > cut && v > 0.0) { v = 1.0 / v; ++live; } else v = 0.0;
    }
    *rank = live;
    if ((e = cudaMemcpyAsync(dinv, hs.data(), (size_t)nt * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
    pinv_gemm_kernel<<<dim3((ld + 63) / 64, (nt + 63) / 64), 256, 0, st>>>(nt, ld, Vt, Bt, dinv, G);
    pinv_sym_kernel<<<dim3((nt + 255) / 256, nt), 256, 0, st>>>(nt, ld, G);
    pinv_pad_kernel<<<dim3((ldc + 255) / 256, n_pad - n > 0 ? n_pad - n : 1), 256, 0, st>>>(n, K1, n_pad, ldc, C, Uz);
    pinv_split_kernel<<<(nt + 7) / 8, 256, 0, st>>>(n, K1, nt, ld, G, values, C, ldc, n_pad, Uz, consts);
    *launches += 4;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;     // hs is a host temporary of the H2D above
    return cudaGetLastError();
}
