// kernels.h — internal launcher interface between api.cu and the kernel files.
#pragma once
#include "common.cuh"

struct DriftScale {            // f' = (f - shift) * scale  (change of drift basis)
    double shift[KB200_MAX_DRIFT + 1];
    double scale[KB200_MAX_DRIFT + 1];
};

// Tile stream layout of the packed inverse factor: row block I owns ktiles[I]
// consecutive tiles of KB_BM x KB_BK values starting at tile index tile_off[I].
struct PackMap {
    int nrb;
    int ktiles[KB_MAXRB];
    long long tile_off[KB_MAXRB];
};

// Drift terms evaluated at the prediction points by the solve kernels themselves (kb200_set_device_drift):
// point-logarithmic wells (uk.py:955-966) and the external-Z raster with the reference's bilinear sampler
// (uk.py:512-628, 967-971). They are the FIRST n_dev of the n_hd host-described drift columns.
struct DeviceDrift {
    int n_wells;               // point_log terms: (adjusted x, adjusted y, strength) triples
    int ext;                   // 1: one external_Z term
    int ext_nx, ext_ny;
    int ext_sorted;            // both raster axes non-decreasing -> binary search; else the reference's linear rule
    const double* wells;       // [n_wells][3]
    const double* ext_x; const double* ext_y; const double* ext_z;   // axes and raster [ny][nx]
};

// K3 v3 (persistent point-tile kernel): solve + finalize in one launch
struct SolvePtParams {
    VgParams vg;
    Aniso an;
    PointSource ps;
    int n, na, nrb, n_rl, n_hd;
    const double* ax; const double* ay; const double* az;
    const void* tiles;
    PackMap pm;
    DriftScale ds;
    const double* consts;
    DeviceDrift dd; int n_dev; // device-evaluated drift columns (n_dev = dd.n_wells + dd.ext <= n_hd)
    const double* drift_pts; long long drift_stride, drift_first;   // host-supplied columns: the remaining n_hd - n_dev
    long long m;
    int gform;                // 1: tiles hold the symmetric inverse (quadratic form q = c^T G c), 0: W = chol(C)^-1
    const double* rowscale;   // int8-slice path only: 2^(ew_r - 12) per packed row
    double* scratch;          // [grid][ceil(n/16)][16*64]  RHS column blocks in fragment order
    double* z_out; double* ss_out;
};

#ifdef __CUDACC__
// index of the first node >= v and of the last node <= v (the node selection of uk.py:556-559)
__device__ __forceinline__ void kb_ext_nodes(const double* __restrict__ ax, int n, int sorted, double v, int& i1, int& i2) {
    if (sorted) {
        int lo = 0, hi = n;                      // lower_bound: first index with ax >= v
        while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(ax + mid) < v) lo = mid + 1; else hi = mid; }
        i2 = lo < n ? lo : n - 1;
        lo = 0; hi = n;                          // upper_bound - 1: last index with ax <= v
        while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(ax + mid) <= v) lo = mid + 1; else hi = mid; }
        i1 = lo > 0 ? lo - 1 : 0;
    } else {
        i2 = n - 1; i1 = 0;
        for (int i = 0; i < n; ++i) if (__ldg(ax + i) >= v) { i2 = i; break; }
        for (int i = n - 1; i >= 0; --i) if (__ldg(ax + i) <= v) { i1 = i; break; }
    }
}

// bilinear sample of the external-Z raster at the ORIGINAL coordinates (x, y): uk.py:560-628 incl. the
// on-node / on-grid-line cases
__device__ __forceinline__ double kb_ext_sample(const DeviceDrift& dd, double x, double y) {
    int x1, x2, y1, y2;
    kb_ext_nodes(dd.ext_x, dd.ext_nx, dd.ext_sorted, x, x1, x2);
    kb_ext_nodes(dd.ext_y, dd.ext_ny, dd.ext_sorted, y, y1, y2);
    const double xa = __ldg(dd.ext_x + x1), xb = __ldg(dd.ext_x + x2);
    const double ya = __ldg(dd.ext_y + y1), yb = __ldg(dd.ext_y + y2);
    const double z11 = __ldg(dd.ext_z + (size_t)y1 * dd.ext_nx + x1);
    const double z22 = __ldg(dd.ext_z + (size_t)y2 * dd.ext_nx + x2);
    if (y1 == y2) {
        if (x1 == x2) return z11;
        return (z11 * (xb - x) + z22 * (x - xa)) / (xb - xa);
    }
    if (x1 == x2) return (z11 * (yb - y) + z22 * (y - ya)) / (yb - ya);
    const double z12 = __ldg(dd.ext_z + (size_t)y1 * dd.ext_nx + x2);
    const double z21 = __ldg(dd.ext_z + (size_t)y2 * dd.ext_nx + x1);
    return (z11 * (xb - x) * (yb - y) + z12 * (x - xa) * (yb - y) + z21 * (xb - x) * (y - ya)
            + z22 * (x - xa) * (y - ya)) / ((xb - xa) * (yb - ya));
}

// Phase F of the three solve kernels (DESIGN.md §3): drift values f of prediction point pj (regional-linear from the
// adjusted coordinates, uk.py:949-954 / uk3d.py:767-773; point_log + external_Z on the device; the rest from the
// host-supplied columns), the (K+1)x(K+1) drift solve, and the two outputs. aux[a * astride] = dual-row dot
// products of this point (rows 0..K: U^T c, row K+1: zeta . c), q = ||W c||^2 (or the quadratic form).
template <int DIM, typename AuxT>
__device__ __forceinline__ void kb_finalize_point(const SolvePtParams& P, long long pj, double q,
                                                  const AuxT* aux, int astride) {
    const int K = P.n_rl + P.n_hd, K1 = K + 1;
    double r[KB200_MAX_DRIFT + 1];
    double f[KB200_MAX_DRIFT + 1];
    if (P.n_rl > 0 || P.n_dev > 0) {
        double rx, ry, rz, x, y, z;
        kb_load_point_raw<DIM>(P.ps, pj, rx, ry, rz);
        kb_adjust<DIM>(P.an, rx, ry, rz, x, y, z);
        if (P.n_rl > 0) {
            f[0] = (x - P.ds.shift[0]) * P.ds.scale[0];
            f[1] = (y - P.ds.shift[1]) * P.ds.scale[1];
            if (DIM == 3) f[2] = (z - P.ds.shift[2]) * P.ds.scale[2];
        }
        int c = P.n_rl;
        for (int w = 0; w < P.dd.n_wells; ++w, ++c) {
            const double wx = __ldg(P.dd.wells + 3 * w), wy = __ldg(P.dd.wells + 3 * w + 1);
            const double dx = x - wx, dy = y - wy;
            double ld = log(sqrt(dx * dx + dy * dy));
            if (isinf(ld)) ld = -100.0;                               // uk.py:960-961
            f[c] = (-__ldg(P.dd.wells + 3 * w + 2) * ld - P.ds.shift[c]) * P.ds.scale[c];
        }
        if (P.dd.ext) { f[c] = (kb_ext_sample(P.dd, rx, ry) - P.ds.shift[c]) * P.ds.scale[c]; ++c; }
    }
    for (int c = P.n_dev; c < P.n_hd; ++c) {
        double v = P.drift_pts[(size_t)(c - P.n_dev) * P.drift_stride + P.drift_first + pj];
        f[P.n_rl + c] = (v - P.ds.shift[P.n_rl + c]) * P.ds.scale[P.n_rl + c];
    }
    f[K] = 1.0;
    const double zc = (double)aux[K1 * astride];
    const double* Sinv = P.consts;
    const double* phi = P.consts + K1 * K1;
    if (P.gform == 2) {
        // pseudo-inverse form (pinv.cu): b = [c; f], sigma^2 = -b^T A^+ b, z = w1.c + w2.f with
        // q = c^T G11 c, aux rows = G21 c, consts = G22 | w2
        double acc = q, zz = zc;
        for (int a = 0; a < K1; ++a) {
            double gf = 0.0;
            for (int b = 0; b < K1; ++b) gf += Sinv[a * K1 + b] * f[b];
            acc += f[a] * (2.0 * (double)aux[a * astride] + gf);
            zz += phi[a] * f[a];
        }
        P.ss_out[pj] = -acc;
        P.z_out[pj] = zz;
        return;
    }
    for (int a = 0; a < K1; ++a) r[a] = (double)aux[a * astride] - f[a];
    double rmu = 0.0, muphi = 0.0;
    for (int a = 0; a < K1; ++a) {
        double mu = 0.0;
        for (int b = 0; b < K1; ++b) mu += Sinv[a * K1 + b] * r[b];
        rmu += r[a] * mu;
        muphi += mu * phi[a];
    }
    P.ss_out[pj] = P.vg.c0 - q + rmu;
    P.z_out[pj] = zc - muphi;
}
#endif

cudaError_t kbk_adjust_data(int dim, const Aniso& an, int n, const double* x, const double* y, const double* z,
                            double* ax, double* ay, double* az, cudaStream_t st);
cudaError_t kbk_assemble(int dim, const VgParams& vg, int n, int n_pad, int ld,
                         const double* ax, const double* ay, const double* az, double* C, cudaStream_t st);
cudaError_t kbk_cholesky(double* C, double* W, double* Lstage, int ld, int n_pad, int* flag, double dtol, cudaStream_t st,
                         cudaStream_t hi, cudaEvent_t* ev, int n_ev, int* launches);   // Lstage: (n_pad/64) x 4096 doubles of scratch;
                                                                                       // hi: high-priority side stream; ev: >= 2*ceil(n_pad/256)+1 events
cudaError_t kbk_trtri(const double* L, double* W, double* T1, int ld, int n_pad, cudaStream_t st, int* launches);
cudaError_t kbk_dual(const double* W, int ld, int n, int n_pad, int n_rl, int n_hd,
                     const double* ax, const double* ay, const double* az, const DriftScale& ds,
                     const double* hd, const double* values,
                     double* Fz, double* Hz, double* Uz, double* consts, int* flag, cudaStream_t st, int* launches);
cudaError_t kbk_pack(int dtype, const double* W, int ld, int n, int n_pad, int na, const double* Uz,
                     const PackMap& pm, void* out, cudaStream_t st);

// in-place inverse of the (symmetric, possibly indefinite) matrix whose lower triangle is in C: blocked Gauss-Jordan with
// partial pivoting (cooperative panel kernel + DMMA rank-64 updates); force_scalar = 1 selects the column-at-a-time form
size_t      kbk_general_inverse_workspace_bytes(int n_pad);
cudaError_t kbk_general_inverse(double* C, int ld, int n, int n_pad, void* work, int* flag, double ptol,
                                cudaStream_t st, int* launches, int force_scalar);
cudaError_t kbk_dual_gform(const double* G, int ld, int n, int n_pad, int n_rl, int n_hd,
                           const double* ax, const double* ay, const double* az, const DriftScale& ds,
                           const double* hd, const double* values,
                           double* Fz, double* Uz, double* consts, int* flag, cudaStream_t st, int* launches);
cudaError_t kbk_pack_gform(const double* G, int ld, int n, int n_pad, int na, const double* Uz,
                           const PackMap& pm, void* out, cudaStream_t st);
cudaError_t kbk_factor_init();
cudaError_t kbk_solve_init();   // opt-in shared memory attributes
cudaError_t kbk_solve_pt(int dim, const SolvePtParams& p, int grid, int tile_points /* 64 | 32 | 16 */, cudaStream_t st);
size_t      kbk_solve_pt_scratch_doubles(int n, int grid);

// fp32 path (solve_tf32.cu): wgmma .tf32, 3xTF32 split, fp32 accumulators in registers
cudaError_t kbk_solve_tf32_init();
cudaError_t kbk_solve_tf32(int dim, const SolvePtParams& p, int grid, cudaStream_t st);
cudaError_t kbk_pack_tf32(const double* W, int ld, int n, int n_pad, int na, const double* Uz, const PackMap& pm,
                          void* out, cudaStream_t st);
size_t      kbk_solve_tf32_scratch_bytes(int n, int grid);
int         kbk_solve_tf32_tile_points();

// fp64-class path on the INT8 tensor cores (solve_i8.cu): error-free slicing into S = 4 | 5 | 6 slices + exact int32
// accumulation
bool        kbk_i8_valid_slices(int S);
cudaError_t kbk_solve_i8_init();
cudaError_t kbk_solve_i8(int S, int dim, const SolvePtParams& p, int grid, cudaStream_t st);
cudaError_t kbk_pack_i8(int S, const double* W, int ld, int n, int n_pad, int na, const double* Uz,
                        int* rowexp, double* rowscale, const long long* tile_off_dev, void* out, cudaStream_t st);
int         kbk_i8_nrb(int S, int n, int na);
int         kbk_i8_rows(int S, int n, int na);
long long   kbk_i8_total_tiles(int S, int n, int na, long long* tile_off);
size_t      kbk_i8_tile_bytes(int S);
size_t      kbk_solve_i8_scratch_bytes(int S, int n, int grid);
int         kbk_solve_i8_tile_points();

// moving window (knn.cu)
struct KnnParams {
    VgParams vg;
    Aniso an;
    PointSource ps;
    int dim, n, k;
    const double* ax; const double* ay; const double* az; const double* values;  // adjusted data, cell-sorted
    const int* sorig;          // original index of each sorted point (deterministic tie-break)
    // uniform cell grid over the adjusted data
    int gx, gy, gz;
    int r0;                    // start radius of the cell search (from the mean point density)
    double ox, oy, oz, inv_cell, cell;
    const int* cell_start;     // [ncells+1]
    long long m;
    double* z_out; double* ss_out;
    int* flag;                 // singular local system
};
cudaError_t kbk_knn_build(int dim, int n, const double* ax, const double* ay, const double* az, const double* values,
                          KnnParams& kp, double* sx, double* sy, double* sz, double* sv, int* sorig,
                          int* cell_of, int* cell_start, int* cursor, int ncells, cudaStream_t st, int* launches);
cudaError_t kbk_knn_solve(const KnnParams& p, int chol, cudaStream_t st);
size_t      kbk_knn_smem_per_warp(int k, int chol, int hasz);

// variogram.cu: constructor-side kernels (experimental variogram binning, cross-validation residuals)
cudaError_t kbk_ev_init();
int         kbk_ev_grid(int n, int num_sms);
size_t      kbk_ev_smem(int nlags, int priv);
int         kbk_ev_priv_max_lags();
cudaError_t kbk_ev_minmax(int dim, int n, const double* x, const double* y, const double* z, int grid,
                          double* bmin, double* bmax, cudaStream_t st);
cudaError_t kbk_ev_bin(int dim, int n, const double* x, const double* y, const double* z, const double* v,
                       int nlags, const double* edges, double inv_dd, int grid, double* part, double* out,
                       cudaStream_t st);
cudaError_t kbk_statistics(int dim, int n, const double* ax, const double* ay, const double* az,
                           const double* L, int ld, const double* u, const double* zeta, int* dup,
                           double* delta, double* sigma, cudaStream_t st);

// pinv.cu: pseudo_inv=True (one-sided Jacobi SVD of the bordered kriging matrix)
cudaError_t kbk_build_fz(int n, int n_pad, int n_rl, int n_hd, const double* ax, const double* ay, const double* az,
                         const DriftScale& ds, const double* hd, const double* values, double* Fz, cudaStream_t st);
cudaError_t kbk_pinv_init();
int         kbk_pinv_max_nt();
size_t      kbk_pinv_workspace_doubles(int nt);
cudaError_t kbk_pinv(int n, int K1, int n_pad, double* C, int ldc, const double* Fz, const double* values,
                     double* Uz, double* consts, double* work, int* counter, cudaStream_t st,
                     int* launches, int* sweeps, int* rank);
