// variogram.cu — constructor-side kernels (SURVEY.md §8f next-2):
//   * experimental semivariogram: all N(N-1)/2 data pairs binned into nlags equal-width lags
//     (core.py:432-505: pdist + per-bin means; 5e9 pairs at N = 1e5, 80 GB as a pair list)
//   * sequential cross-validation residuals of core.py:759-836 (`_find_statistics`: point i kriged from
//     points [0, i), an O(N^4) loop in the reference) read off ONE Cholesky factor in O(N) — see
//     stats_kernel below.
#include "common.cuh"
#include "kernels.h"

#define EV_T 256          // threads per CTA = rows i of a pair tile
#define EV_J 64           // columns j of a pair tile (staged in shared memory)

// Tile t of the lower block triangle: row block bi (EV_T rows), column block bj (EV_J columns),
// bj*EV_J <= bi*EV_T + EV_T-1  ->  (EV_T/EV_J)*(bi+1) column blocks per row block.
__device__ __forceinline__ void ev_tile(long long t, int& bi, int& bj) {
    const long long R = EV_T / EV_J;
    // tiles before row block b: R * b(b+1)/2
    long long b = (long long)floor((sqrt(1.0 + 8.0 * (double)t / (double)R) - 1.0) * 0.5);
    if (b < 0) b = 0;
    while (R * b * (b + 1) / 2 > t) --b;
    while (R * (b + 1) * (b + 2) / 2 <= t) ++b;
    bi = (int)b;
    bj = (int)(t - R * b * (b + 1) / 2);
}

static long long ev_ntiles(int n) {
    long long nb = (n + EV_T - 1) / EV_T;
    return (long long)(EV_T / EV_J) * nb * (nb + 1) / 2;
}

// Euclidean pair distance in scipy pdist's operation order (s = dx*dx; s += dy*dy; ...; sqrt), with no
// FMA contraction, so that d — and with it dmin, dmax, the bin edges and every bin assignment — is the
// bit pattern the reference sees. Geographic: great-circle degrees between unit vectors (common.cuh).
template <int DIM>
__device__ __forceinline__ double ev_dist(double ax, double ay, double az, double bx, double by, double bz) {
    if (DIM == KB_GEO) return kb_dist<KB_GEO>(ax, ay, az, bx, by, bz);
    double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by);
    double s = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
    if (DIM == 3) { double dz = __dsub_rn(az, bz); s = __dadd_rn(s, __dmul_rn(dz, dz)); }
    return __dsqrt_rn(s);
}

template <int DIM>
__device__ __forceinline__ void ev_load(int n, int i, const double* __restrict__ x, const double* __restrict__ y,
                                        const double* __restrict__ z, double& ox, double& oy, double& oz) {
    ox = oy = oz = 0.0;
    if (i >= n) return;
    if (DIM == KB_GEO) { Aniso a{}; kb_adjust<KB_GEO>(a, x[i], y[i], 0.0, ox, oy, oz); return; }
    ox = x[i]; oy = y[i];
    if (DIM == 3) oz = z[i];
}

// pass 1: smallest and largest pair distance, one (min, max) per CTA
template <int DIM>
__global__ void __launch_bounds__(EV_T) ev_minmax_kernel(int n, const double* __restrict__ x, const double* __restrict__ y,
                                                         const double* __restrict__ z, long long ntiles,
                                                         double* __restrict__ bmin, double* __restrict__ bmax) {
    __shared__ double sx[EV_J], sy[EV_J], sz[EV_J];
    __shared__ double rmin[EV_T / 32], rmax[EV_T / 32];
    const int tid = threadIdx.x;
    double lo = INFINITY, hi = -INFINITY;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int bi, bj;
        ev_tile(t, bi, bj);
        const int i = bi * EV_T + tid, j0 = bj * EV_J;
        __syncthreads();
        if (tid < EV_J) ev_load<DIM>(n, j0 + tid, x, y, z, sx[tid], sy[tid], sz[tid]);
        double xi, yi, zi;
        ev_load<DIM>(n, i, x, y, z, xi, yi, zi);
        __syncthreads();
        const int jend = min(EV_J, min(n, i) - j0);        // pairs j < i only
        if (i < n)
            for (int q = 0; q < jend; ++q) {
                double d = ev_dist<DIM>(xi, yi, zi, sx[q], sy[q], sz[q]);
                lo = fmin(lo, d); hi = fmax(hi, d);
            }
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((tid & 31) == 0) { rmin[tid >> 5] = lo; rmax[tid >> 5] = hi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < EV_T / 32; ++w) { lo = fmin(lo, rmin[w]); hi = fmax(hi, rmax[w]); }
        bmin[blockIdx.x] = lo; bmax[blockIdx.x] = hi;
    }
}

// pass 2: per-lag pair count, sum of d and sum of 0.5 (v_i - v_j)^2. PRIV: every thread owns a private
// set of bins in shared memory (no atomics, fixed summation order -> deterministic); otherwise
// (nlags too large for that) one set of bins per CTA with shared-memory atomics.
// edges[k] = dmin + k*dd (k < nlags), edges[nlags] = dmax + 0.001, computed by the host exactly as
// core.py:471-476; a pair belongs to lag k iff edges[k] <= d < edges[k+1] (core.py:497-499).
// part: [gridDim.x][3][nlags] = (count, sum d, sum g) per CTA.
template <int DIM, bool PRIV>
__global__ void __launch_bounds__(EV_T) ev_bin_kernel(int n, const double* __restrict__ x, const double* __restrict__ y,
                                                      const double* __restrict__ z, const double* __restrict__ v,
                                                      long long ntiles, int nlags, const double* __restrict__ edges,
                                                      double inv_dd, double* __restrict__ part) {
    extern __shared__ double ev_sm[];
    double* se = ev_sm;                               // nlags + 1 edges
    double* sx = se + nlags + 1;
    double* sy = sx + EV_J;
    double* sz = sy + EV_J;
    double* sv = sz + EV_J;
    const int nb = PRIV ? nlags * EV_T : nlags;
    double* bd = sv + EV_J;                           // sum d
    double* bg = bd + nb;                             // sum g
    double* bc = bg + nb;                             // counts (exact in fp64 up to 2^53)
    const int tid = threadIdx.x;
    for (int e = tid; e <= nlags; e += EV_T) se[e] = edges[e];
    for (int e = tid; e < 3 * nb; e += EV_T) bd[e] = 0.0;
    const double e0 = edges[0];
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int bi, bj;
        ev_tile(t, bi, bj);
        const int i = bi * EV_T + tid, j0 = bj * EV_J;
        __syncthreads();
        if (tid < EV_J) {
            ev_load<DIM>(n, j0 + tid, x, y, z, sx[tid], sy[tid], sz[tid]);
            sv[tid] = (j0 + tid < n) ? v[j0 + tid] : 0.0;
        }
        double xi, yi, zi;
        ev_load<DIM>(n, i, x, y, z, xi, yi, zi);
        const double vi = i < n ? v[i] : 0.0;
        __syncthreads();
        const int jend = min(EV_J, min(n, i) - j0);
        if (i < n)
            for (int q = 0; q < jend; ++q) {
                const double d = ev_dist<DIM>(xi, yi, zi, sx[q], sy[q], sz[q]);
                const double dv = __dsub_rn(vi, sv[q]);
                const double g = __dmul_rn(0.5, __dmul_rn(dv, dv));
                int k = (int)((d - e0) * inv_dd);
                k = max(0, min(nlags - 1, k));
                while (k > 0 && d < se[k]) --k;
                while (k < nlags - 1 && d >= se[k + 1]) ++k;
                if (d >= se[k] && d < se[k + 1]) {
                    if (PRIV) {
                        const int o = k * EV_T + tid;
                        bd[o] += d; bg[o] += g; bc[o] += 1.0;
                    } else {
                        atomicAdd(&bd[k], d); atomicAdd(&bg[k], g); atomicAdd(&bc[k], 1.0);
                    }
                }
            }
    }
    __syncthreads();
    double* out = part + (size_t)blockIdx.x * 3 * nlags;
    for (int e = tid; e < 3 * nlags; e += EV_T) {
        const int q = e / nlags, k = e - q * nlags;       // q: 0 count, 1 sum d, 2 sum g
        const double* src = q == 0 ? bc : (q == 1 ? bd : bg);
        double s = 0.0;
        if (PRIV) for (int w = 0; w < EV_T; ++w) s += src[k * EV_T + w];
        else s = src[k];
        out[q * nlags + k] = s;
    }
}

// fixed-order sum of the per-CTA partials: out[3][nlags]
__global__ void ev_reduce_kernel(int nblk, int nlags, const double* __restrict__ part, double* __restrict__ out) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * nlags) return;
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += part[(size_t)b * 3 * nlags + e];
    out[e] = s;
}

size_t kbk_ev_smem(int nlags, int priv) {
    size_t nb = priv ? (size_t)nlags * EV_T : (size_t)nlags;
    return ((size_t)nlags + 1 + 4 * EV_J + 3 * nb) * sizeof(double);
}
int kbk_ev_priv_max_lags() { return (int)((227 * 1024 - (4 * EV_J + 2) * 8) / ((3 * EV_T + 1) * 8)); }

cudaError_t kbk_ev_init() {
    return KbDims::for_each([](auto D) {
        KB_CUDA_OK(cudaFuncSetAttribute(ev_bin_kernel<D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        return cudaFuncSetAttribute(ev_bin_kernel<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    });
}

int kbk_ev_grid(int n, int num_sms) {
    long long nt = ev_ntiles(n);
    return (int)(nt < num_sms ? nt : num_sms);
}

cudaError_t kbk_ev_minmax(int dim, int n, const double* x, const double* y, const double* z, int grid,
                          double* bmin, double* bmax, cudaStream_t st) {
    return KbDims::dispatch(dim, [&](auto D) {
        ev_minmax_kernel<D><<<grid, EV_T, 0, st>>>(n, x, y, z, ev_ntiles(n), bmin, bmax);
        return cudaGetLastError();
    });
}

cudaError_t kbk_ev_bin(int dim, int n, const double* x, const double* y, const double* z, const double* v,
                       int nlags, const double* edges, double inv_dd, int grid, double* part, double* out,
                       cudaStream_t st) {
    const long long nt = ev_ntiles(n);
    const int priv = nlags <= kbk_ev_priv_max_lags();
    const size_t sm = kbk_ev_smem(nlags, priv);
    KB_CUDA_OK(KbDims::dispatch(dim, [&](auto D) {
        return KbBools::dispatch(priv, [&](auto PRIV) {
            ev_bin_kernel<D, bool(PRIV)><<<grid, EV_T, sm, st>>>(n, x, y, z, v, nt, nlags, edges, inv_dd, part);
            return cudaGetLastError();
        });
    }));
    ev_reduce_kernel<<<(3 * nlags + 127) / 128, 128, 0, st>>>(grid, nlags, part, out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Cross-validation residuals (core.py:759-836). The reference kriges data point i from points [0, i)
// with the ordinary-kriging system of core.py:732-752, for every i: N solves of growing size. With
// C = c0 - gamma = L L^T (the factor the execute path already holds), the leading i x i block of L is the
// factor of the first i points, row i of L is L_i^-1 c_i, and u = L^-1 1, zeta = L^-1 Z restricted to
// [0, i) are the forward solves of that sub-problem. Eliminating the unbiasedness row gives
//     s_i = sum_{j<i} u_j^2,  t_i = sum_{j<i} u_j zeta_j,
//     sigma_i^2 = L_ii^2 (1 + u_i^2 / s_i),     delta_i = Z_i - zhat_i = L_ii (zeta_i - u_i t_i / s_i),
// i.e. every residual comes from diag(L), u, zeta and two prefix sums.
// dup[i] != 0 marks a point within 1e-10 of an earlier one: the reference forces an exact hit there
// (core.py:729-731,748-749), gets sigma^2 = 0 and drops the point (core.py:818-819).
template <int DIM>
__global__ void stats_dup_kernel(int n, const double* __restrict__ ax, const double* __restrict__ ay,
                                 const double* __restrict__ az, int* __restrict__ dup) {
    // blockIdx.x: 256 rows i; blockIdx.y: one 256-column chunk of the candidates j < i (dup[] starts at 0)
    __shared__ double sx[256], sy[256], sz[256];
    const int i = blockIdx.x * 256 + threadIdx.x;
    const int j0 = blockIdx.y * 256;
    if (j0 > blockIdx.x * 256 + 255) return;            // chunk entirely above the diagonal (block-uniform)
    const double xi = i < n ? ax[i] : 0.0, yi = i < n ? ay[i] : 0.0, zi = i < n ? az[i] : 0.0;
    const int j = j0 + threadIdx.x;
    sx[threadIdx.x] = j < n ? ax[j] : 0.0; sy[threadIdx.x] = j < n ? ay[j] : 0.0; sz[threadIdx.x] = j < n ? az[j] : 0.0;
    __syncthreads();
    int hit = 0;
    const int je = min(256, min(n, i) - j0);
    for (int q = 0; q < je; ++q)
        if (fabs(kb_dist<DIM>(xi, yi, zi, sx[q], sy[q], sz[q])) <= 1e-10) hit = 1;
    if (i < n && hit) atomicOr(&dup[i], 1);
}

__global__ void __launch_bounds__(1024) stats_kernel(int n, const double* __restrict__ L, int ld,
                                                     const double* __restrict__ u, const double* __restrict__ zeta,
                                                     const int* __restrict__ dup,
                                                     double* __restrict__ delta, double* __restrict__ sigma) {
    __shared__ double ss[1024], st[1024];
    const int tid = threadIdx.x;
    const int chunk = (n + 1023) / 1024;
    const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
    double s = 0.0, t = 0.0;
    for (int i = i0; i < i1; ++i) { s += u[i] * u[i]; t += u[i] * zeta[i]; }
    ss[tid] = s; st[tid] = t;
    __syncthreads();
    if (tid == 0) {                                   // exclusive scan in a fixed order (1024 terms)
        double a = 0.0, b = 0.0;
        for (int w = 0; w < 1024; ++w) { double x = ss[w], y = st[w]; ss[w] = a; st[w] = b; a += x; b += y; }
    }
    __syncthreads();
    s = ss[tid]; t = st[tid];
    for (int i = i0; i < i1; ++i) {
        const double ui = u[i], zi = zeta[i], lii = L[(size_t)i * ld + i];
        double dl = 0.0, sg = 0.0;
        if (i > 0 && !dup[i]) {
            const double var = lii * lii * (1.0 + ui * ui / s);
            dl = lii * (zi - ui * t / s);
            sg = sqrt(var);
        }
        delta[i] = dl; sigma[i] = sg;
        s += ui * ui; t += ui * zi;
    }
}

cudaError_t kbk_statistics(int dim, int n, const double* ax, const double* ay, const double* az,
                           const double* L, int ld, const double* u, const double* zeta, int* dup,
                           double* delta, double* sigma, cudaStream_t st) {
    const int gb = (n + 255) / 256;
    const dim3 g(gb, gb);
    KB_CUDA_OK(cudaMemsetAsync(dup, 0, (size_t)n * sizeof(int), st));
    KB_CUDA_OK(KbDims::dispatch(dim, [&](auto D) {
        stats_dup_kernel<D><<<g, 256, 0, st>>>(n, ax, ay, az, dup);
        return cudaGetLastError();
    }));
    stats_kernel<<<1, 1024, 0, st>>>(n, L, ld, u, zeta, dup, delta, sigma);
    return cudaGetLastError();
}
