// knn.cu — moving-window kriging (n_closest_points = k).
//
// Reference semantics (ok.py:722-758, 929-986; native twin cok.pyx:98-193):
//   per prediction point: the k nearest data points (cKDTree.query(k, eps=0.0): exact, sorted by
//   distance), local system a = A_full[idx+{n}, idx+{n}] (zero diagonal, ones border), b = -gamma(d)
//   (0 on exact hits), x = solve(a, b) (dgesv), z = x[:k].Z[idx], sigma2 = -x.b.
// The reference gathers the local block from the full N x N matrix (80 GB at N = 1e5, SURVEY F4);
// here the block is assembled on the fly from the neighbour coordinates.
//
// K4 (search): uniform cell grid over the adjusted data (counting sort by cell); one warp per
//     prediction point grows a block of cells until the k-th candidate lies inside the visited
//     region, then a warp bitonic sort yields the k nearest in ascending distance (ties by index).
// K5 (solve): same warp assembles the k x k shifted covariance block C = c0 - gamma (diag c0) in
//     shared memory and runs LU with partial pivoting (two right-hand sides c and 1); the ordinary
//     kriging weights follow from the bordered-system identities (DESIGN.md §5).
#include "common.cuh"
#include "kernels.h"
#include <cfloat>
#include <algorithm>

#define KN_CAP 512          // candidate buffer (per warp)
#define KN_SELECT_DOUBLES 272   // selection scratch: 256 histogram ints + 256 slot ints + 32 boundary ints

__global__ void knn_count_kernel(int dim, int n, const double* __restrict__ ax, const double* __restrict__ ay,
                                 const double* __restrict__ az, KnnParams kp, int* __restrict__ cell_of,
                                 int* __restrict__ counts) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int cx = min(kp.gx - 1, max(0, (int)floor((ax[i] - kp.ox) * kp.inv_cell)));
    int cy = min(kp.gy - 1, max(0, (int)floor((ay[i] - kp.oy) * kp.inv_cell)));
    int cz = dim >= 3 ? min(kp.gz - 1, max(0, (int)floor((az[i] - kp.oz) * kp.inv_cell))) : 0;
    int c = (cz * kp.gy + cy) * kp.gx + cx;
    cell_of[i] = c;
    atomicAdd(&counts[c], 1);
}

// exclusive scan of counts[0..ncells) into start[0..ncells], single block
__global__ void __launch_bounds__(1024) knn_scan_kernel(int ncells, const int* __restrict__ counts, int* __restrict__ start) {
    __shared__ int part[1024];
    int tid = threadIdx.x;
    int per = (ncells + 1023) / 1024;
    int b = tid * per, e = min(ncells, b + per);
    int s = 0;
    for (int i = b; i < e; ++i) s += counts[i];
    part[tid] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        int v = tid >= o ? part[tid - o] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    int run = tid ? part[tid - 1] : 0;
    for (int i = b; i < e; ++i) { start[i] = run; run += counts[i]; }
    if (tid == 1023) start[ncells] = part[1023];
}

// counting-sort scatter. The position inside a cell depends on atomics, but the neighbour ORDER used
// by the solve is fixed by the final sort (distance, then original index), so results are deterministic.
__global__ void knn_scatter_kernel(int n, const int* __restrict__ cell_of, const int* __restrict__ start,
                                   int* __restrict__ cursor, const double* __restrict__ ax,
                                   const double* __restrict__ ay, const double* __restrict__ az,
                                   const double* __restrict__ val, double* __restrict__ sx, double* __restrict__ sy,
                                   double* __restrict__ sz, double* __restrict__ sv, int* __restrict__ sorig) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = cell_of[i];
    int pos = start[c] + atomicAdd(&cursor[c], 1);
    sx[pos] = ax[i]; sy[pos] = ay[i]; sz[pos] = az[i]; sv[pos] = val[i]; sorig[pos] = i;
}

// The counting-sort scatter leaves the points of a cell in the order the atomics happened to run; one thread per
// cell re-orders its run by original index (cells hold ~2 points: insertion sort), so that the candidate walk -
// and with it the order of the neighbours in the local system - is the same on every launch and every device.
__global__ void knn_cellsort_kernel(int ncells, const int* __restrict__ start, double* __restrict__ sx,
                                    double* __restrict__ sy, double* __restrict__ sz, double* __restrict__ sv,
                                    int* __restrict__ sorig) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncells) return;
    const int b = start[c], e = start[c + 1];
    for (int i = b + 1; i < e; ++i) {
        const int oi = sorig[i];
        const double x = sx[i], y = sy[i], z = sz[i], v = sv[i];
        int j = i - 1;
        while (j >= b && sorig[j] > oi) {
            sorig[j + 1] = sorig[j]; sx[j + 1] = sx[j]; sy[j + 1] = sy[j]; sz[j + 1] = sz[j]; sv[j + 1] = sv[j];
            --j;
        }
        sorig[j + 1] = oi; sx[j + 1] = x; sy[j + 1] = y; sz[j + 1] = z; sv[j + 1] = v;
    }
}

// ---- warp helpers -----------------------------------------------------------
__device__ __forceinline__ bool cand_less(double da, int ia, double db, int ib) {
    return da < db || (da == db && ia < ib);
}

// ascending bitonic sort of (d2[], id[]) of length `len` (power of two) by one warp
__device__ __forceinline__ void warp_bitonic(double* d2, int* id, const int* __restrict__ sorig, int len, int lane) {
    for (int size = 2; size <= len; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = lane; t < (len >> 1); t += 32) {
                int lo = 2 * t - (t & (stride - 1));
                int hi = lo + stride;
                bool up = ((lo & size) == 0);
                double dl = d2[lo], dh = d2[hi];
                int il = id[lo], ih = id[hi];
                int ol = 0, oh = 0;
                if (dl == dh) {        // ties are rare: only then fetch the original indices (deterministic order)
                    ol = il >= 0 ? sorig[il] : 0x7fffffff;
                    oh = ih >= 0 ? sorig[ih] : 0x7fffffff;
                }
                bool sw = up ? cand_less(dh, oh, dl, ol) : cand_less(dl, ol, dh, oh);
                if (sw) { d2[lo] = dh; d2[hi] = dl; id[lo] = ih; id[hi] = il; }
            }
            __syncwarp();
        }
    }
}

// CHOL = true : packed lower-triangular Cholesky of the local covariance block (no pivoting, half the
//               updates, 20 KB of shared memory per point at k = 64 -> more points in flight); needs k <= 128.
//               A non-positive pivot (variogram not valid in this dimension) sets *flag = 2 and the host
//               re-runs the launch with CHOL = false.
// CHOL = false: LU with partial pivoting on the full k x k block (dgesv semantics, cok.pyx:165-174).
// MODE 1 (LOO): leave-one-out of station q = ps.first + p (ps holds the raw station coordinates): the candidate with
//              original index q is never counted. It lands at d^2 == 0 exactly (data and query go through the same
//              adjust sequence), so only there is its index looked up.
// MODE 2 (LGO): leave-group-out: the query is station q as in MODE 1, and every candidate of q's group is never counted
//              (sgroup: groups in the cell-sorted order, qgroup: in the original order).
template <int DIM, int MODEL, bool CHOL, int MODE>
__device__ __forceinline__ void knn_solve_body(const KnnParams& P, int warps_per_cta, int per_warp_doubles,
                                               const int* __restrict__ sgroup, const int* __restrict__ qgroup) {
    constexpr bool LOO = MODE == 1;
    extern __shared__ __align__(16) double ksm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp >= warps_per_cta) return;
    const long long p = (long long)blockIdx.x * warps_per_cta + warp;
    if (p >= P.m) return;
    const int k = P.k;
    const int S = k | 1;                       // odd row stride: conflict-free column walks
    double* base = ksm + (size_t)warp * per_warp_doubles;
    double* A = base;                          // k * S  (aliased by the candidate buffers during the search)
    const int kp = CHOL ? ((k + 7) & ~7) : k;        // padded system size of the tiled Cholesky
    const int naug = (2 + P.nv + 7) >> 3;            // augmented tile rows: [c ; 1 ; Z_0 .. Z_{nv-1}]
    // tiled Cholesky: nt (nt + 1) / 2 lower tiles + naug * nt augmented tiles + 1 tile for the diagonal inverse, 64 doubles
    // each — keep in step with kbk_knn_smem_per_warp
    size_t a_doubles = CHOL ? ((size_t)(kp / 8) * (kp / 8 + 1) / 2 + (size_t)naug * (kp / 8) + 1) * 64 : (size_t)k * S;
    size_t cand_doubles = KN_CAP + KN_CAP / 2 + KN_SELECT_DOUBLES;   // d2[CAP] doubles + id[CAP] ints + selection scratch
    size_t off = a_doubles > cand_doubles ? a_doubles : cand_doubles;
    // per-neighbour arrays behind the matrix: the tiled Cholesky needs rc, nx, ny, (nz,) nv only (its right-hand sides
    // live in the augmented tile row) - one array fewer in 2-D lets a ninth point fit into an SM's shared memory;
    // the LU path keeps all seven. Keep in step with kbk_knn_smem_per_warp.
    double* rc = base + off;                   // rhs c (LU: becomes C^-1 c)
    double* tailp = rc + kp;
    double* r1 = rc; double* cv = rc;          // LU only: rhs 1 (becomes C^-1 1), c kept for sigma^2
    if (!CHOL) { r1 = tailp; cv = tailp + kp; tailp += 2 * kp; }
    double* nx = tailp; double* ny = nx + kp; tailp = ny + kp;
    double* nz = nx;                           // 2-D: never read (kb_dist<2> ignores z)
    if (KB_HASZ(DIM)) { nz = tailp; tailp += kp; }
    double* ni = tailp;                        // cell-sorted index of each neighbour: field v's value is P.values[v n + i]
    double* cd2 = base;
    int* cid = reinterpret_cast<int*>(base + KN_CAP);

    double qx, qy, qz;
    kb_load_point<DIM>(P.ps, P.an, p, qx, qy, qz);
    const int qg = MODE == 2 ? qgroup[P.ps.first + p] : 0;

    // ---------------- K4: exact k nearest ----------------
    const int cqx = min(P.gx - 1, max(0, (int)floor((qx - P.ox) * P.inv_cell)));
    const int cqy = min(P.gy - 1, max(0, (int)floor((qy - P.oy) * P.inv_cell)));
    const int cqz = KB_HASZ(DIM) ? min(P.gz - 1, max(0, (int)floor((qz - P.oz) * P.inv_cell))) : 0;
    int cnt = 0;
    int r = P.r0;                                      // start radius (cells) from the mean point density
    auto compact = [&](int keep) {
        int len = 1; while (len < cnt) len <<= 1;
        for (int t = cnt + lane; t < len; t += 32) { cd2[t] = DBL_MAX; cid[t] = -1; }
        __syncwarp();
        warp_bitonic(cd2, cid, P.sorig, len, lane);
        cnt = min(cnt, keep);
    };
    for (;;) {
        const int x0 = max(0, cqx - r), x1 = min(P.gx - 1, cqx + r);
        const int y0 = max(0, cqy - r), y1 = min(P.gy - 1, cqy + r);
        const int z0 = KB_HASZ(DIM) ? max(0, cqz - r) : 0, z1 = KB_HASZ(DIM) ? min(P.gz - 1, cqz + r) : 0;
        cnt = 0;
        const int nyr = y1 - y0 + 1;
        const int nrows = nyr * (z1 - z0 + 1);
        // every cell row of the block is one contiguous run of the cell-sorted points: 32 rows at a time,
        // one lane per row fetches the run bounds (one round of independent loads), then the warp walks the
        // concatenated runs with a flat index so that the coordinate loads of all candidates are independent
        for (int row0 = 0; row0 < nrows; row0 += 32) {
            const int rr = row0 + lane;
            int rb = 0, rlen = 0;
            if (rr < nrows) {
                const int cy = y0 + rr % nyr, cz = z0 + rr / nyr;
                const int rowbase = (cz * P.gy + cy) * P.gx;
                rb = P.cell_start[rowbase + x0];
                rlen = P.cell_start[rowbase + x1 + 1] - rb;
            }
            int incl = rlen;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const int pre = incl - rlen;
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            for (int f0 = 0; f0 < total; f0 += 32) {
                const int f = f0 + lane;
                bool ok = f < total;
                int j = 0;
#pragma unroll
                for (int st = 16; st > 0; st >>= 1) {
                    const int cand = j + st;                               // <= 31
                    const int pc = __shfl_sync(0xffffffffu, pre, cand);
                    if (pc <= f) j = cand;
                }
                const int bj = __shfl_sync(0xffffffffu, rb, j);
                const int pj = __shfl_sync(0xffffffffu, pre, j);
                double d2 = 0.0;
                int i = 0;
                if (ok) {
                    i = bj + (f - pj);
                    double dx = P.ax[i] - qx, dy = P.ay[i] - qy;
                    d2 = dx * dx + dy * dy;
                    if (KB_HASZ(DIM)) { double dz = P.az[i] - qz; d2 += dz * dz; }
                    if (LOO && d2 == 0.0 && P.sorig[i] == P.ps.first + p) ok = false;
                    if (MODE == 2 && sgroup[i] == qg) ok = false;
                }
                unsigned msk = __ballot_sync(0xffffffffu, ok);
                int pos = cnt + __popc(msk & ((1u << lane) - 1u));
                if (ok) { cd2[pos] = d2; cid[pos] = i; }
                cnt += __popc(msk);
                __syncwarp();
                if (cnt > KN_CAP - 32) compact(k);
            }
        }
        // distance from the query to the nearest face of the visited block that still has cells behind it
        double dout = DBL_MAX;
        if (x0 > 0) dout = fmin(dout, qx - (P.ox + x0 * P.cell));
        if (x1 < P.gx - 1) dout = fmin(dout, (P.ox + (x1 + 1) * P.cell) - qx);
        if (y0 > 0) dout = fmin(dout, qy - (P.oy + y0 * P.cell));
        if (y1 < P.gy - 1) dout = fmin(dout, (P.oy + (y1 + 1) * P.cell) - qy);
        if (KB_HASZ(DIM)) {
            if (z0 > 0) dout = fmin(dout, qz - (P.oz + z0 * P.cell));
            if (z1 < P.gz - 1) dout = fmin(dout, (P.oz + (z1 + 1) * P.cell) - qz);
        }
        if (dout == DBL_MAX) break;                    // whole grid visited
        int inside = 0;
        if (dout > 0.0) {
            double lim = dout * dout;
            for (int t = lane; t < cnt; t += 32) inside += (cd2[t] <= lim) ? 1 : 0;
            for (int o = 16; o > 0; o >>= 1) inside += __shfl_xor_sync(0xffffffffu, inside, o);
        }
        if (inside >= k) break;
        r += (r < 2) ? 1 : (r >> 1);                   // not enough inside the inscribed sphere: larger block, start over
    }
    // ---- the k nearest of the cnt candidates, WITHOUT sorting them ----
    // d^2 of points scattered in the plane/space is close to uniform in area/volume, so 256 linear buckets over
    // [0, max d^2] put ~1 candidate into the bucket that holds the k-th smallest: everything in lower buckets is
    // selected, the boundary bucket is ranked exactly by (d^2, original index) - the rule of the sort it replaces.
    // The neighbours keep the order of the candidate walk (cells are ordered by original index: deterministic).
    // A boundary bucket with more than 32 entries (lattices, duplicates) falls back to the full sort.
    double dk2;                                        // d^2 of the k-th neighbour
    {
        int* hist = reinterpret_cast<int*>(base + KN_CAP + KN_CAP / 2);   // 256 ints behind the candidate buffers
        int* sel = hist + 256;                         // k (<= 256) selected candidate slots, then the boundary list (32)
        double dmax = 0.0;
        for (int t = lane; t < cnt; t += 32) dmax = fmax(dmax, cd2[t]);
        for (int o = 16; o > 0; o >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
        const double bs = dmax > 0.0 ? 255.999 / dmax : 0.0;
        for (int t = lane; t < 256; t += 32) hist[t] = 0;
        __syncwarp();
        for (int t = lane; t < cnt; t += 32) atomicAdd(&hist[(int)(cd2[t] * bs)], 1);
        __syncwarp();
        // bucket of the k-th smallest: lane owns buckets 8 lane .. 8 lane + 7
        int hloc[8], run = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) { hloc[q] = hist[lane * 8 + q]; run += hloc[q]; }
        int incl = run;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        int before = incl - run;                       // candidates in the buckets of lower lanes
        int bstar = -1, below = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (bstar < 0 && before + hloc[q] >= k && before < k) { bstar = lane * 8 + q; below = before; }
            before += hloc[q];
        }
        const unsigned who = __ballot_sync(0xffffffffu, bstar >= 0);
        const int src = __ffs(who) - 1;                // exactly one lane found it (cnt >= k)
        bstar = __shfl_sync(0xffffffffu, bstar, src);
        below = __shfl_sync(0xffffffffu, below, src);
        const int nbound = hist[bstar];                // entries of the boundary bucket
        const int need = k - below;                    // how many of them are neighbours
        if (nbound > 32 || cnt < k) {
            compact(k);                                // degenerate distribution: exact full sort (ascending)
            dk2 = cd2[k - 1];
        } else {
            // pass 1: the boundary candidates into a list; pass 2 ranks them; pass 3 compacts the selection in walk order
            int nb_seen = 0;
            for (int t0 = 0; t0 < cnt; t0 += 32) {
                const int t = t0 + lane;
                const bool isb = t < cnt && (int)(cd2[t] * bs) == bstar;
                const unsigned m = __ballot_sync(0xffffffffu, isb);
                if (isb) sel[k + nb_seen + __popc(m & ((1u << lane) - 1u))] = t;
                nb_seen += __popc(m);
            }
            __syncwarp();
            // lane j < nbound: rank of boundary candidate j by (d^2, original index)
            bool take = false;
            double myd = 0.0; int myo = 0, myt = -1;
            if (lane < nbound) { myt = sel[k + lane]; myd = cd2[myt]; myo = P.sorig[cid[myt]]; }
            int rank = 0;
            for (int j = 0; j < nbound; ++j) {
                const double dj = __shfl_sync(0xffffffffu, myd, j);
                const int oj = __shfl_sync(0xffffffffu, myo, j);
                if (lane < nbound && j != lane && cand_less(dj, oj, myd, myo)) ++rank;
            }
            take = lane < nbound && rank < need;
            // threshold = the largest selected boundary d^2 (or the largest d^2 below the bucket when need == 0)
            double thr = take ? myd : -1.0;
            for (int o = 16; o > 0; o >>= 1) thr = fmax(thr, __shfl_xor_sync(0xffffffffu, thr, o));
            // mark the taken boundary candidates in the hist area (reuse: 1 flag per candidate slot is too large, so a
            // 32-bit mask over the boundary list positions is broadcast instead)
            const unsigned takemask = __ballot_sync(0xffffffffu, take);
            int nsel = 0;
            double dmaxsel = thr;
            for (int t0 = 0; t0 < cnt; t0 += 32) {
                const int t = t0 + lane;
                bool pick = false;
                if (t < cnt) {
                    const int b = (int)(cd2[t] * bs);
                    if (b < bstar) { pick = true; dmaxsel = fmax(dmaxsel, cd2[t]); }
                    else if (b == bstar) {
                        for (int j = 0; j < nbound; ++j) if (((takemask >> j) & 1u) && sel[k + j] == t) pick = true;
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, pick);
                if (pick) sel[nsel + __popc(m & ((1u << lane) - 1u))] = t;
                nsel += __popc(m);
            }
            for (int o = 16; o > 0; o >>= 1) dmaxsel = fmax(dmaxsel, __shfl_xor_sync(0xffffffffu, dmaxsel, o));
            dk2 = dmaxsel;
            __syncwarp();
            // gather the selection to the front of the candidate arrays (slots are increasing: reads of slot s >= t
            // happen before writes of slot t only if staged through registers)
            for (int c0 = 0; c0 < k; c0 += 128) {      // 128 slots per round: reads of a round never see its own writes
                double gd[4]; int gi[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = c0 + lane + 32 * u;
                    if (t < k) { const int sidx = sel[t]; gd[u] = cd2[sidx]; gi[u] = cid[sidx]; }
                }
                __syncwarp();
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = c0 + lane + 32 * u;
                    if (t < k) { cd2[t] = gd[u]; cid[t] = gi[u]; }
                }
                __syncwarp();
            }
            __syncwarp();
        }
    }
    // neighbours -> per-warp arrays (these live outside the region the candidate buffers alias)
    VgParams vg = P.vg;
    if (MODEL == KB200_VG_LINEAR || MODEL == KB200_VG_POWER || MODEL == KB200_VG_TABLE) {
        // unbounded (or unknown: tabulated) models: local shift c0 = gamma(2 d_k) >= gamma of any neighbour pair (DESIGN.md §5)
        double dk = sqrt(dk2);
        if (DIM == KB_GEO) dk = 2.0 * asin(fmin(1.0, 0.5 * dk)) * 57.29577951308232;   // chord -> degrees
        double g = kb_gamma<MODEL>(vg, 2.0 * dk);
        vg.c0 = g > 0.0 ? g : 1.0;
    }
    for (int t = lane; t < k; t += 32) {
        int i = cid[t];
        nx[t] = P.ax[i]; ny[t] = P.ay[i]; ni[t] = (double)i;
        if (KB_HASZ(DIM)) nz[t] = P.az[i];
        // euclidean: the search distance is the kriging distance; geographic: neighbours were ranked by chord
        // length (ok.py:936-960), the kriging distance is the great-circle distance (ok.py:962-969)
        const double dq = DIM == KB_GEO ? kb_dist<DIM>(nx[t], ny[t], nz[t], qx, qy, qz) : sqrt(cd2[t]);
        double c = kb_cov_rhs<MODEL>(vg, dq);
        rc[t] = c;
        if (!CHOL) { cv[t] = c; r1[t] = 1.0; }
    }
    for (int t = k + lane; t < kp; t += 32) {          // identity padding of the blocked system
        nx[t] = 0.0; ny[t] = 0.0; ni[t] = -1.0; rc[t] = 0.0;
        if (KB_HASZ(DIM)) nz[t] = 0.0;
        if (!CHOL) { cv[t] = 0.0; r1[t] = 0.0; }
    }
    __syncwarp();                                      // candidates consumed: A may be overwritten now

    if (CHOL) {
        // ---------------- K5 (Cholesky): augmented 8x8-tiled factorisation on the fp64 tensor pipe ----------------
        // The k x k block C = c0 - gamma (identity-padded to kp = 8 * nt) is stored as lower-triangular 8x8 tiles in
        // MMA-operand order: element (r, q) of a tile at (q >> 2) * 32 + r * 4 + (q & 3), so that the A/B fragment of
        // mma.m8n8k4 (lane <-> (r = lane >> 2, q = 4 k4 + (lane & 3))) is one conflict-free LDS.64 at k4 * 32 + lane and
        // the C fragment one LDS.128. Three extra rows [c ; 1 ; Z] form an augmented tile row: after the right-looking
        // factorisation they hold y_c = L^-1 c, y_1 = L^-1 1, y_Z = L^-1 Z, and the bordered system of ok.py:738-756
        // follows from dot products alone (no back substitution):
        //     mu = (y_1.y_c - 1) / (y_1.y_1),  z = y_c.y_Z - mu y_1.y_Z,  sigma^2 = c0 - (y_c.y_c - mu y_1.y_c) - mu.
        // Per 8-column step: potf2 + inverse of the diagonal tile in registers (warp shuffles inside groups of 8 lanes),
        // panel tiles X <- X Winv^T and trailing tiles C_ij -= L_ip L_jp^T as DMMAs (2 per tile).
        // With value fields the augmented rows continue [c ; 1 ; Z_0 ; Z_1 ; ...] over naug tile rows nt .. nt + naug - 1;
        // every row goes through the same per-row arithmetic, so field v's y_Z does not depend on nv.
        const int nt = kp >> 3;                       // tile rows of the covariance block; tile rows >= nt = the augmented rows
#define KN_T(i, j) (A + ((i) < nt ? (size_t)(i) * ((i) + 1) / 2 + (j) : (size_t)nt * (nt + 1) / 2 + (size_t)((i) - nt) * nt + (j)) * 64)
        double* Wt = A + ((size_t)nt * (nt + 1) / 2 + (size_t)naug * nt) * 64;   // inverse of the current diagonal tile
        const int fr = lane >> 2, fq = lane & 3;
        // assembly: lane <-> (row fr, columns fq and 4 + fq) of every tile; two tiles (four independent sqrt/exp chains)
        // per iteration: the evaluation is latency-bound with 8 warps per SM
        for (int ti = 0; ti < nt; ++ti) {
            const int i = ti * 8 + fr;
            const double xi = nx[i], yi = ny[i], zi = KB_HASZ(DIM) ? nz[i] : 0.0;
            for (int tj = 0; tj <= ti; tj += 2) {
                double v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int tjj = tj + (u >> 1);
                    const int j = tjj * 8 + (u & 1) * 4 + fq;
                    double val = 0.0;
                    if (tjj <= ti) {
                        if (i == j) val = (i < k) ? vg.c0 : 1.0;
                        else if (j < i && i < k) {
                            double d = kb_dist<DIM>(xi, yi, zi, nx[j], ny[j], KB_HASZ(DIM) ? nz[j] : 0.0);
                            val = vg.c0 - kb_gamma<MODEL>(vg, d);
                        }
                    }
                    v[u] = val;
                }
                double* T = KN_T(ti, tj);
                T[lane] = v[0]; T[32 + lane] = v[1];
                if (tj + 1 <= ti) { T[64 + lane] = v[2]; T[96 + lane] = v[3]; }     // tile (ti, tj + 1) follows (ti, tj)
            }
        }
        for (int ta = 0; ta < naug * nt; ++ta) {      // augmented rows: 0 = c, 1 = ones, 2 + v = Z_v (the rest zero)
            const int ar = (ta / nt) * 8 + fr, tj = ta % nt;
            double* T = KN_T(nt + ta / nt, tj);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int t = tj * 8 + half * 4 + fq;
                double v = 0.0;
                if (ar == 0) v = rc[t];
                else if (ar == 1) v = (t < k) ? 1.0 : 0.0;
                else if (ar < 2 + P.nv && t < k) v = P.values[(size_t)(ar - 2) * P.n + (int)ni[t]];
                T[half * 32 + lane] = v;
            }
        }
        __syncwarp();
        bool notpd = false;
        const double ptol = 3.6e-15 * vg.c0;       // 16 eps: exact duplicates (nugget 0) give a pivot of +-1 ulp, not 0
        const int gr = lane & 7, gg = lane >> 3;   // potf2: row within the tile, redundant group
        for (int ps = 0; ps < nt; ++ps) {
            // ---- diagonal tile: L_pp (rows in registers) and Winv = L_pp^-1 ----
            {
                const double* T = KN_T(ps, ps);
                double d[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) d[q] = T[(q >> 2) * 32 + gr * 4 + (q & 3)];
                double dinv = 1.0;
#pragma unroll
                for (int pc = 0; pc < 8; ++pc) {
                    const double piv = __shfl_sync(0xffffffffu, d[pc], pc, 8);
                    if (!(piv > ptol)) notpd = true;    // at or below the rounding noise of c0 - sum l^2: not PD
                    const double inv = rsqrt(piv);
                    const double l = d[pc] * inv;       // lane pc: sqrt(piv); lanes below: L[r][pc]
                    d[pc] = l;
                    if (gr == pc) dinv = inv;
#pragma unroll
                    for (int c = pc + 1; c < 8; ++c) d[c] = fma(-l, __shfl_sync(0xffffffffu, l, c, 8), d[c]);
                }
                // column gr of the inverse: x[i] = Winv[i][gr]
                double x[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    double sacc = 0.0;
#pragma unroll
                    for (int q = 0; q < i; ++q) sacc = fma(__shfl_sync(0xffffffffu, d[q], i, 8), x[q], sacc);
                    const double di = __shfl_sync(0xffffffffu, dinv, i, 8);
                    x[i] = (i < gr) ? 0.0 : ((i == gr) ? dinv : -sacc * di);
                }
                // group gg writes rows 2 gg and 2 gg + 1 of Winv (operand order)
                const double v0 = gg == 0 ? x[0] : (gg == 1 ? x[2] : (gg == 2 ? x[4] : x[6]));
                const double v1 = gg == 0 ? x[1] : (gg == 1 ? x[3] : (gg == 2 ? x[5] : x[7]));
                Wt[(gr >> 2) * 32 + (2 * gg) * 4 + (gr & 3)] = v0;
                Wt[(gr >> 2) * 32 + (2 * gg + 1) * 4 + (gr & 3)] = v1;
            }
            __syncwarp();
            // ---- panel: X(i, p) <- X Winv^T for the tile rows below (incl. the augmented rows) ----
            {
                const double wb0 = Wt[lane], wb1 = Wt[32 + lane];
                for (int i = ps + 1; i < nt + naug; ++i) {
                    double* T = KN_T(i, ps);
                    const double a0 = T[lane], a1 = T[32 + lane];
                    double c0 = 0.0, c1 = 0.0;
                    kb_dmma(c0, c1, a0, wb0);
                    kb_dmma(c0, c1, a1, wb1);
                    __syncwarp();                   // every lane has read its operands before the tile is overwritten
                    *reinterpret_cast<double2*>(T + (fq >> 1) * 32 + fr * 4 + 2 * (fq & 1)) = make_double2(c0, c1);
                }
            }
            __syncwarp();
            // ---- trailing update: C(i, j) -= L(i, p) L(j, p)^T,  p < j <= i  (augmented rows: j < nt) ----
            // two column tiles per iteration: independent accumulator chains hide the DMMA / LDS latency
            for (int i = ps + 1; i < nt + naug; ++i) {
                const double* Li = KN_T(i, ps);
                const double a0 = -Li[lane], a1 = -Li[32 + lane];
                const int jend = i < nt ? i : nt - 1;
                const int coff = (fq >> 1) * 32 + fr * 4 + 2 * (fq & 1);
                int j = ps + 1;
                for (; j + 1 <= jend; j += 2) {
                    const double* Lj0 = KN_T(j, ps);
                    const double* Lj1 = KN_T(j + 1, ps);
                    double2* Cp0 = reinterpret_cast<double2*>(KN_T(i, j) + coff);
                    double2* Cp1 = reinterpret_cast<double2*>(KN_T(i, j + 1) + coff);
                    double2 ca = *Cp0, cb = *Cp1;
                    const double b00 = Lj0[lane], b01 = Lj0[32 + lane], b10 = Lj1[lane], b11 = Lj1[32 + lane];
                    kb_dmma(ca.x, ca.y, a0, b00);
                    kb_dmma(cb.x, cb.y, a0, b10);
                    kb_dmma(ca.x, ca.y, a1, b01);
                    kb_dmma(cb.x, cb.y, a1, b11);
                    *Cp0 = ca; *Cp1 = cb;
                }
                if (j <= jend) {
                    const double* Lj = KN_T(j, ps);
                    double2* Cp = reinterpret_cast<double2*>(KN_T(i, j) + coff);
                    double2 c = *Cp;
                    kb_dmma(c.x, c.y, a0, Lj[lane]);
                    kb_dmma(c.x, c.y, a1, Lj[32 + lane]);
                    *Cp = c;
                }
            }
            __syncwarp();
        }
        if (notpd) {
            if (lane == 0) {
                atomicMax(P.flag, 2); P.ss_out[p] = 0.0;
                for (int v = 0; v < P.nv; ++v) P.z_out[p + v * P.zstride] = 0.0;
            }
            return;
        }
        // ---- bordered-system identities from the augmented rows ----
        double s11 = 0.0, s1c = 0.0, scc = 0.0;
        for (int t = lane; t < kp; t += 32) {
            const double* T = KN_T(nt, t >> 3) + ((t & 7) >> 2) * 32 + (t & 3);
            const double yc = T[0], y1 = T[4];
            s11 = fma(y1, y1, s11); s1c = fma(y1, yc, s1c); scc = fma(yc, yc, scc);
        }
        for (int o = 16; o > 0; o >>= 1) {
            s11 += __shfl_xor_sync(0xffffffffu, s11, o); s1c += __shfl_xor_sync(0xffffffffu, s1c, o);
            scc += __shfl_xor_sync(0xffffffffu, scc, o);
        }
        const double mu = (s1c - 1.0) / s11;
        if (lane == 0) P.ss_out[p] = vg.c0 - (scc - mu * s1c) - mu;       // ok.py:756 (= -x.b) in covariance form
        for (int v = 0; v < P.nv; ++v) {
            const int ar = 2 + v;                      // augmented row of field v
            double s1z = 0.0, scz = 0.0;
            for (int t = lane; t < kp; t += 32) {
                const double* T = KN_T(nt, t >> 3) + ((t & 7) >> 2) * 32 + (t & 3);
                const double yc = T[0], y1 = T[4], yz = KN_T(nt + (ar >> 3), t >> 3)[((t & 7) >> 2) * 32 + (ar & 7) * 4 + (t & 3)];
                s1z = fma(y1, yz, s1z); scz = fma(yc, yz, scz);
            }
            for (int o = 16; o > 0; o >>= 1) {
                s1z += __shfl_xor_sync(0xffffffffu, s1z, o); scz += __shfl_xor_sync(0xffffffffu, scz, o);
            }
            if (lane == 0) P.z_out[p + v * P.zstride] = scz - mu * s1z;                       // ok.py:755
        }
        return;
#undef KN_T
    } else {
    // ---------------- K5: local system ----------------
    // C[i][j] = c0 - gamma(|x_i - x_j|), C[i][i] = c0   (ok.py:641-644 in covariance form)
    for (int e = lane; e < k * k; e += 32) {
        int i = e / k, j = e - i * k;
        double v;
        if (i == j) v = vg.c0;
        else {
            double d = kb_dist<DIM>(nx[i], ny[i], nz[i], nx[j], ny[j], nz[j]);
            v = vg.c0 - kb_gamma<MODEL>(vg, d);
        }
        A[i * S + j] = v;
    }
    __syncwarp();
    // LU with partial pivoting (dgesv semantics, cok.pyx:165-174), both right-hand sides carried along
    bool singular = false;
    for (int pcol = 0; pcol < k; ++pcol) {
        double best = -1.0; int bi = pcol;
        for (int i = pcol + lane; i < k; i += 32) {
            double v = fabs(A[i * S + pcol]);
            if (v > best) { best = v; bi = i; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            double ob = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (!(best > 0.0)) { singular = true; break; }
        if (bi != pcol) {
            for (int j = lane; j < k; j += 32) {
                double t = A[pcol * S + j]; A[pcol * S + j] = A[bi * S + j]; A[bi * S + j] = t;
            }
            if (lane == 0) {
                double t = rc[pcol]; rc[pcol] = rc[bi]; rc[bi] = t;
                t = r1[pcol]; r1[pcol] = r1[bi]; r1[bi] = t;
            }
            __syncwarp();
        }
        // the multiplier is a true quotient, not a product with the reciprocal: a row equal to the pivot row (coincident
        // stations, nugget 0) then gets l = 1 exactly and cancels to an exact zero row, so the system is found singular
        // (a reciprocal can leave l one ulp off 1 and the contracted update a +-ulp row that passes as a pivot)
        const double piv = A[pcol * S + pcol];
        const double bc = rc[pcol], b1 = r1[pcol];
        for (int i = pcol + 1 + lane; i < k; i += 32) {
            double l = A[i * S + pcol] / piv;
            A[i * S + pcol] = l;
            rc[i] -= l * bc;
            r1[i] -= l * b1;
        }
        __syncwarp();
        // rank-1 update of the trailing block: lanes across columns, rows unrolled by 4
        for (int j0 = pcol + 1; j0 < k; j0 += 32) {
            int j = j0 + lane;
            bool ok = j < k;
            double u = ok ? A[pcol * S + j] : 0.0;
            int i = pcol + 1;
            for (; i + 3 < k; i += 4) {
                double l0 = A[i * S + pcol], l1 = A[(i + 1) * S + pcol], l2 = A[(i + 2) * S + pcol], l3 = A[(i + 3) * S + pcol];
                if (ok) {
                    A[i * S + j] -= l0 * u; A[(i + 1) * S + j] -= l1 * u;
                    A[(i + 2) * S + j] -= l2 * u; A[(i + 3) * S + j] -= l3 * u;
                }
            }
            for (; i < k; ++i) { double l = A[i * S + pcol]; if (ok) A[i * S + j] -= l * u; }
        }
        __syncwarp();
    }
    if (singular) {
        if (lane == 0) {
            atomicMax(P.flag, 1); P.ss_out[p] = 0.0;
            for (int v = 0; v < P.nv; ++v) P.z_out[p + v * P.zstride] = 0.0;
        }
        return;
    }
    // back substitution U x = y for both right-hand sides
    for (int pcol = k - 1; pcol >= 0; --pcol) {
        const double inv = 1.0 / A[pcol * S + pcol];
        const double xc = rc[pcol] * inv, x1 = r1[pcol] * inv;
        __syncwarp();
        if (lane == 0) { rc[pcol] = xc; r1[pcol] = x1; }
        for (int i = lane; i < pcol; i += 32) {
            double u = A[i * S + pcol];
            rc[i] -= u * xc;
            r1[i] -= u * x1;
        }
        __syncwarp();
    }
    }   // CHOL / LU
    // bordered-system identities: mu = (1'C^-1 c - 1)/(1'C^-1 1); lambda = C^-1 c - mu C^-1 1
    double s1 = 0.0, sc = 0.0;
    for (int t = lane; t < k; t += 32) { s1 += r1[t]; sc += rc[t]; }
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); sc += __shfl_xor_sync(0xffffffffu, sc, o); }
    const double mu = (sc - 1.0) / s1;
    double lc = 0.0;
    for (int t = lane; t < k; t += 32) {
        double lam = rc[t] - mu * r1[t];
        lc += lam * cv[t];
    }
    for (int o = 16; o > 0; o >>= 1) lc += __shfl_xor_sync(0xffffffffu, lc, o);
    if (lane == 0) P.ss_out[p] = vg.c0 - lc - mu;       // ok.py:756 (= -x.b) in covariance form
    for (int v = 0; v < P.nv; ++v) {                    // the same weights for every field
        double zz = 0.0;
        for (int t = lane; t < k; t += 32) {
            double lam = rc[t] - mu * r1[t];
            zz += lam * P.values[(size_t)v * P.n + (int)ni[t]];
        }
        for (int o = 16; o > 0; o >>= 1) zz += __shfl_xor_sync(0xffffffffu, zz, o);
        if (lane == 0) P.z_out[p + v * P.zstride] = zz;                       // ok.py:755
    }
}

template <int DIM, int MODEL, bool CHOL, bool LOO = false>
__global__ void __launch_bounds__(320) knn_solve_kernel(const __grid_constant__ KnnParams P, int warps_per_cta,
                                                         int per_warp_doubles) {
    knn_solve_body<DIM, MODEL, CHOL, LOO ? 1 : 0>(P, warps_per_cta, per_warp_doubles, nullptr, nullptr);
}

template <int DIM, int MODEL, bool CHOL>
__global__ void __launch_bounds__(320) knn_lgo_kernel(const __grid_constant__ KnnParams P, int warps_per_cta,
                                                       int per_warp_doubles, const int* __restrict__ sgroup,
                                                       const int* __restrict__ qgroup) {
    knn_solve_body<DIM, MODEL, CHOL, 2>(P, warps_per_cta, per_warp_doubles, sgroup, qgroup);
}

// ---- host side -------------------------------------------------------------
size_t kbk_knn_smem_per_warp(int k, int chol, int hasz, int nv) {
    size_t S = (size_t)(k | 1);
    size_t kp = chol ? (size_t)((k + 7) & ~7) : (size_t)k;
    size_t nt = kp / 8, naug = (size_t)(2 + nv + 7) / 8;
    size_t a = chol ? (nt * (nt + 1) / 2 + naug * nt + 1) * 64 : (size_t)k * S, c = KN_CAP + KN_CAP / 2 + KN_SELECT_DOUBLES;
    const size_t tail = chol ? (hasz ? 5 : 4) : 7;      // rc, nx, ny, (nz,) ni  |  + r1, cv for the LU path
    return ((a > c ? a : c) + tail * kp + 2) * sizeof(double);
}

__global__ void knn_sort_fields_kernel(int n, int nv, const int* __restrict__ sorig, const double* __restrict__ src,
                                       double* __restrict__ dst) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int i = sorig[s];
    for (int v = 0; v < nv; ++v) dst[(size_t)v * n + s] = src[(size_t)v * n + i];
}

cudaError_t kbk_knn_sort_fields(int n, int nv, const int* sorig, const double* src, double* dst, cudaStream_t st) {
    knn_sort_fields_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, nv, sorig, src, dst);
    return cudaGetLastError();
}

cudaError_t kbk_knn_solve(const KnnParams& p, int chol, cudaStream_t st, int mode, const int* sgroup, const int* qgroup) {
    return KbDims::dispatch(p.dim, [&](auto D) {
        return KbModels::dispatch(p.vg.model, [&](auto M) {
            return KbBools::dispatch(chol && p.k <= 128, [&](auto CHOL) {
                return KbList<0, 1, 2>::dispatch(mode, [&](auto MODE) {
                    const size_t per = kbk_knn_smem_per_warp(p.k, CHOL, KB_HASZ(D) ? 1 : 0, p.nv);
                    // as many points in flight per SM as fit (<= 320 threads; 227 KB minus the static 1 KB)
                    const int wpc = (int)std::min<size_t>(10, (size_t)(226 * 1024) / per);
                    if (wpc < 1) return cudaErrorInvalidValue;
                    const size_t smem = per * wpc;
                    auto launch = [&](auto kernel, auto... groups) {
                        KB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        kernel<<<(unsigned)((p.m + wpc - 1) / wpc), wpc * 32, smem, st>>>(p, wpc, (int)(per / sizeof(double)),
                                                                                          groups...);
                        return cudaGetLastError();
                    };
                    if constexpr (MODE == 2) return launch(knn_lgo_kernel<D, M, bool(CHOL)>, sgroup, qgroup);
                    else return launch(knn_solve_kernel<D, M, bool(CHOL), MODE == 1>);
                });
            });
        });
    });
}

__global__ void knn_sort_groups_kernel(int n, const int* __restrict__ sorig, const int* __restrict__ src,
                                       int* __restrict__ dst) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) dst[s] = src[sorig[s]];
}

cudaError_t kbk_knn_sort_groups(int n, const int* sorig, const int* src, int* dst, cudaStream_t st) {
    knn_sort_groups_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, sorig, src, dst);
    return cudaGetLastError();
}

cudaError_t kbk_knn_build(int dim, int n, const double* ax, const double* ay, const double* az, const double* values,
                          KnnParams& kp, double* sx, double* sy, double* sz, double* sv, int* sorig,
                          int* cell_of, int* cell_start, int* cursor, int ncells, cudaStream_t st, int* launches) {
    KB_CUDA_OK(cudaMemsetAsync(cursor, 0, (size_t)(ncells + 1) * sizeof(int), st));
    KB_CUDA_OK(cudaMemsetAsync(cell_start, 0, (size_t)(ncells + 1) * sizeof(int), st));
    int g = (n + 255) / 256;
    // counts go to `cursor` first, the scan writes cell_start, then cursor is re-zeroed for the scatter
    knn_count_kernel<<<g, 256, 0, st>>>(dim, n, ax, ay, az, kp, cell_of, cursor);
    knn_scan_kernel<<<1, 1024, 0, st>>>(ncells, cursor, cell_start);
    KB_CUDA_OK(cudaMemsetAsync(cursor, 0, (size_t)(ncells + 1) * sizeof(int), st));
    knn_scatter_kernel<<<g, 256, 0, st>>>(n, cell_of, cell_start, cursor, ax, ay, az, values, sx, sy, sz, sv, sorig);
    knn_cellsort_kernel<<<(ncells + 255) / 256, 256, 0, st>>>(ncells, cell_start, sx, sy, sz, sv, sorig);
    *launches += 4;
    kp.ax = sx; kp.ay = sy; kp.az = sz; kp.values = sv; kp.sorig = sorig; kp.cell_start = cell_start; kp.nv = 1;
    return cudaGetLastError();
}
