// api.cu — C ABI of libkrige_b200.so (include/krige_b200.h): handle, problem set-up,
// orchestration of the factor kernels (factor.cu), the fused solve (solve.cu) and the
// moving window (knn.cu). Host code only; no torch types, no CPU compute path.
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include <cstring>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <algorithm>
#include <thread>
#include <climits>
#include "kernels.h"

#define KB_VERSION 2000
static const int64_t KB_STAGE_PTS = 1 << 20;   // prediction points per staged output chunk (2 x 8 MB through pinned memory)
#define KB_TILE_COST_32 0.534     // one round of 32-point tiles relative to one round of 64-point tiles (fp64 kernel, N=5000,
#define KB_TILE_COST_16 0.432     // one H100 80GB HBM3 at 700 W: 3.90 / 2.08 / 1.68 ms per round at an uncapped
                                  // 1965-1980 MHz SM clock; scripts/tile_timing.py)
static const int64_t KB_STAGE_MIN = 1 << 18;   // below this the outputs go straight to the caller's buffers
#define KB_TN_FIELDS 32   // widest point tile of the value-fields solve kernels (solve.cu: no spills up to 32 points)

// Prediction points on the device: [first, first + count) of the explicit points or of the flattened grid
struct Src {
    bool grid; int64_t nx, ny, nz;
    const double *a, *b, *c;      // points (px,py,pz) or axes (gx,gy,gz), device pointers
    int64_t first, count;
    const double* d_drift; int64_t drift_stride, drift_first;

    Src sub(int64_t o, int64_t m) const {        // points [o, o + m) of this source
        Src s = *this; s.first += o; s.count = m; s.drift_first += o; return s;
    }
    PointSource point_source() const {
        PointSource ps{};
        ps.grid = grid ? 1 : 0;
        ps.px = a; ps.py = b; ps.pz = c; ps.gx = a; ps.gy = b; ps.gz = c;
        ps.nx = nx; ps.ny = ny; ps.nz = nz; ps.first = first;
        return ps;
    }
};

// tm[] slots, in the order of kb200_last_timings (krige_b200.h) and _cabi.TIMING_KEYS
enum Tm { TM_ASSEMBLE, TM_CHOLESKY, TM_TRTRI, TM_PACK_DUAL, TM_SOLVE, TM_FINALIZE, TM_H2D, TM_D2H, TM_KNN_SEARCH,
          TM_KNN_SOLVE, TM_SOLVE_LAUNCHES, TM_LAUNCHES, TM_COUNT };
// ev[] slots: the phases of kb200_set_problem (kb200_set_problem_knn: upload, then the cell grid build), the window
// of an execute call's solve launches (run_to_host records it for its callers) and its host <-> device copies
enum Ev { EV_UPLOAD, EV_ADJUSTED, EV_ASM, EV_KNN_BUILT = EV_ASM, EV_FACTOR, EV_INVERT, EV_DUAL, EV_PACKED,
          EV_RUN, EV_RUN_END, EV_H2D, EV_H2D_END, EV_D2H_END, EV_COUNT };

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct kb200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;

    // description
    bool described = false, ready = false, knn_ready = false;
    // kb200_set_problem factored the problem on this handle (not kb200_blob_commit): its factor or inverse (wC, wW),
    // dual blocks (wF) and data (wRaw) are in the workspace
    bool local_factor = false;
    int slices = 0;           // int8-slice dtypes: number of slices (6 / 5 / 4), else 0
    int gform = 0;            // 1: general (indefinite) fallback, tiles hold the symmetric inverse
    int geo = 0;              // 1: coordinates_type='geographic' for the next problem description
    int pinv = 0;             // 1: pseudo_inv=True for the next problem description (global path only)
    int pinv_sweeps = 0, pinv_rank = 0;
    int dim = 2, dtype = KB200_F64, n = 0, n_pad = 0, ld = 0, n_rl = 0, n_hd = 0, K1 = 1, na = 2, nrb = 0;
    VgParams vg{};
    Aniso an{};
    DriftScale ds{};
    PackMap pm{};
    std::vector<double> hx, hy, hz, hval, hdrift;
    double bb_lo[3] = {0, 0, 0}, bb_hi[3] = {0, 0, 0};   // adjusted bounding box of the data
    // value fields (kb200_set_values): nf columns of nf_n values, column-major; nf = 0: the problem's own values
    int nf = 0; int64_t nf_n = 0;
    std::vector<double> hfields;
    int aux_cols = KB_MAXAUX;  // columns of each of Fz / Hz / Uz in wF: max(KB_MAXAUX, na)
    int64_t zstride = 0;       // z_out block stride of the fields in the running execute call
    int pin_blocks = 0;        // capacity of each pinned staging buffer, in blocks of KB_STAGE_PTS doubles

    DevBuf blob;              // the factor blob (BlobView)
    size_t off_consts = 0, off_ax = 0, off_ay = 0, off_az = 0, off_tiles = 0, off_rowscale = 0, blob_bytes = 0;

    // factor workspace
    DevBuf wC, wW, wT, wF, wRaw, wFlag;
    // execute workspace
    DevBuf wPts, wOut, wDrift, wScratch, wFstage;
    int num_sms = 132;
    // device-evaluated drift terms (kb200_set_device_drift): configuration + the count used by the described problem
    DeviceDrift dd{};
    DevBuf wWells, wExt;
    int n_dev = 0;
    // pinned staging of the outputs (two chunks in flight) and the stream that drains them
    void* pin[2] = {nullptr, nullptr};
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t evk[2] = {}, evc[2] = {};
    // look-ahead Cholesky: high-priority side stream for the panel chain + ordering events
    cudaStream_t hi_stream = nullptr;
    std::vector<cudaEvent_t> fev;
    // knn workspace
    DevBuf kSorted, kCells, kFields;
    DevBuf wVario;            // constructor-side helpers (experimental variogram, statistics)
    DevBuf wLoo;              // leave-one-out workspace
    DevBuf wLgo, wLgoM;       // leave-group-out: blocks and lists | padded matrices of a large group
    DevBuf wPairs;            // cross-validation under exact_values: the near-pair lists
    DevBuf wTab;              // KB200_VG_TABLE: (value, slope) pairs on the device
    std::vector<double> htab; // ... and on the host (value, slope interleaved), for the covariance shift
    double tab_dmax = 0.0; int tab_n = 0;
    KnnParams kp{};
    int k_ncells = 0;

    cudaEvent_t ev[EV_COUNT] = {};
    double tm[TM_COUNT] = {};
    long long launches = 0, solve_launches = 0;
};

static int fail(kb200_ctx* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    return code;
}
#define CU(h, expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { \
    return fail(h, _e == cudaErrorMemoryAllocation ? KB200_ENOMEM : KB200_ECUDA, \
                std::string(#expr) + ": " + cudaGetErrorString(_e)); } } while (0)

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Every setter changes what the next description means: the described (and any factored) problem is gone
static void drop_problem(kb200_ctx* h) {
    h->described = false; h->ready = false; h->knn_ready = false; h->local_factor = false;
}

// The factor blob, one allocation that multigpu.py ships between processes built from the same commit:
// header | consts (S^-1 | phi_v) | ax | ay | az (adjusted data coordinates) | tiles | rowscale (int8-slice dtypes)
struct BlobView { double *hdr, *consts, *ax, *ay, *az; char* tiles; double* rowscale; };
static BlobView blob_view(const kb200_ctx* h) {
    char* p = h->blob.as<char>();
    auto at = [p](size_t off) { return reinterpret_cast<double*>(p + off); };
    return {at(0), at(h->off_consts), at(h->off_ax), at(h->off_ay), at(h->off_az), p + h->off_tiles, at(h->off_rowscale)};
}

// blob header slots (doubles): magic, c0, drift shift and scale per column, gform
enum HdrSlot { HDR_MAGIC = 0, HDR_C0 = 1, HDR_SHIFT = 2, HDR_SCALE = HDR_SHIFT + KB200_MAX_DRIFT + 1,
               HDR_GFORM = HDR_SCALE + KB200_MAX_DRIFT + 1, HDR_DOUBLES = 64 };
static_assert(HDR_GFORM == 34 && HDR_GFORM < HDR_DOUBLES, "blob header layout");
static const double KB_MAGIC = 20260922.0;

static void write_header(const kb200_ctx* h, double* hdr) {
    std::fill(hdr, hdr + HDR_DOUBLES, 0.0);
    hdr[HDR_MAGIC] = KB_MAGIC; hdr[HDR_C0] = h->vg.c0; hdr[HDR_GFORM] = (double)h->gform;
    for (int c = 0; c <= KB200_MAX_DRIFT; ++c) { hdr[HDR_SHIFT + c] = h->ds.shift[c]; hdr[HDR_SCALE + c] = h->ds.scale[c]; }
}

static bool read_header(kb200_ctx* h, const double* hdr) {
    if (hdr[HDR_MAGIC] != KB_MAGIC) return false;
    h->vg.c0 = hdr[HDR_C0];
    h->gform = (int)hdr[HDR_GFORM];
    for (int c = 0; c <= KB200_MAX_DRIFT; ++c) { h->ds.shift[c] = hdr[HDR_SHIFT + c]; h->ds.scale[c] = hdr[HDR_SCALE + c]; }
    return true;
}

// wRaw: the raw data columns x | y | z | values | n_hd drift columns | nf value fields, n doubles each
enum RawCol { RAW_X, RAW_Y, RAW_Z, RAW_V, RAW_DRIFT };
static double* raw_col(const kb200_ctx* h, int c) { return h->wRaw.as<double>() + (size_t)c * h->n; }
// the values the problem kriges: its own, or the nf value fields of kb200_set_values
static double* kriged_values(const kb200_ctx* h) { return raw_col(h, h->nf ? RAW_DRIFT + h->n_hd : RAW_V); }

// wF: Fz | Hz | Uz, aux_cols columns of n_pad each
enum AuxBlock { AUX_F, AUX_H, AUX_U };
static double* aux_block(const kb200_ctx* h, int i) {
    return h->wF.as<double>() + (size_t)i * h->aux_cols * h->n_pad;
}

extern "C" int kb200_version(void) { return KB_VERSION; }

extern "C" int kb200_create(kb200_handle* out, int device) {
    if (!out) return KB200_EBADARG;
    *out = nullptr;
    int cnt = 0;
    cudaError_t e = cudaGetDeviceCount(&cnt);
    if (e != cudaSuccess || cnt == 0) return KB200_ECUDA;   // no CPU fallback by design
    kb200_ctx* h = new kb200_ctx();
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= cnt) { delete h; return KB200_EBADARG; }
    h->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete h; return KB200_ECUDA; }
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return KB200_ECUDA; }
    h->own_stream = true;
    for (auto& ev : h->ev) if (cudaEventCreate(&ev) != cudaSuccess) { delete h; return KB200_ECUDA; }
    if (kbk_factor_init() != cudaSuccess || kbk_solve_init() != cudaSuccess || kbk_solve_wgmma_init() != cudaSuccess ||
        kbk_ev_init() != cudaSuccess || kbk_pinv_init() != cudaSuccess) { delete h; return KB200_ECUDA; }
    if (cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || h->num_sms < 1) h->num_sms = 132;
    *out = h;
    return KB200_OK;
}

extern "C" void kb200_destroy(kb200_handle h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    for (DevBuf* b : {&h->blob, &h->wC, &h->wW, &h->wT, &h->wF, &h->wRaw, &h->wFlag,
                      &h->wPts, &h->wOut, &h->wDrift, &h->wScratch, &h->wFstage, &h->kSorted, &h->kCells, &h->kFields, &h->wVario, &h->wTab,
                      &h->wLoo, &h->wLgo, &h->wLgoM, &h->wPairs, &h->wWells, &h->wExt}) b->release();
    for (int i = 0; i < 2; ++i) {
        if (h->pin[i]) cudaFreeHost(h->pin[i]);
        if (h->evk[i]) cudaEventDestroy(h->evk[i]);
        if (h->evc[i]) cudaEventDestroy(h->evc[i]);
    }
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->hi_stream) cudaStreamDestroy(h->hi_stream);
    for (auto& e : h->fev) cudaEventDestroy(e);
    for (auto& ev : h->ev) if (ev) cudaEventDestroy(ev);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" const char* kb200_last_error(kb200_handle h) { return h ? h->err.c_str() : "null handle"; }

extern "C" int kb200_set_stream(kb200_handle h, void* s) {
    if (!h) return KB200_EBADARG;
    if (h->own_stream && h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
    h->stream = reinterpret_cast<cudaStream_t>(s);
    h->own_stream = false;
    return KB200_OK;
}

extern "C" int kb200_set_coordinates(kb200_handle h, int coordinates_type) {
    if (!h) return KB200_EBADARG;
    if (coordinates_type != KB200_EUCLIDEAN && coordinates_type != KB200_GEOGRAPHIC)
        return fail(h, KB200_EBADARG, "coordinates_type must be KB200_EUCLIDEAN or KB200_GEOGRAPHIC");
    h->geo = coordinates_type == KB200_GEOGRAPHIC ? 1 : 0;
    drop_problem(h);
    return KB200_OK;
}

extern "C" int kb200_set_pseudo_inverse(kb200_handle h, int enable) {
    if (!h) return KB200_EBADARG;
    h->pinv = enable ? 1 : 0;
    drop_problem(h);
    return KB200_OK;
}

extern "C" int kb200_set_values(kb200_handle h, int n_fields, int64_t n, const double* values) {
    if (!h) return KB200_EBADARG;
    drop_problem(h);
    h->nf = 0; h->nf_n = 0; h->hfields.clear();
    if (n_fields == 0) return KB200_OK;
    if (n_fields < 0 || n_fields > KB200_MAX_FIELDS)
        return fail(h, KB200_EBADARG, "n_fields must be in [0, " + std::to_string(KB200_MAX_FIELDS) + "]");
    if (n < 1 || n > (1LL << 30) || !values) return fail(h, KB200_EBADARG, "values: n >= 1 rows and a non-NULL array");
    const size_t cnt = (size_t)n * n_fields;
    for (size_t i = 0; i < cnt; ++i)
        if (!std::isfinite(values[i]))
            return fail(h, KB200_EBADARG, "values must be finite (field " + std::to_string(i / n) + ", row " +
                        std::to_string(i % n) + ")");
    h->hfields.assign(values, values + cnt);
    h->nf = n_fields; h->nf_n = n;
    return KB200_OK;
}

extern "C" void kb200_reset_counters(kb200_handle h) {
    if (!h) return;
    h->launches = 0; h->solve_launches = 0;
    for (double& t : h->tm) t = 0.0;
}

extern "C" int kb200_last_timings(kb200_handle h, double* ms, int n) {
    if (!h || !ms) return KB200_EBADARG;
    h->tm[TM_SOLVE_LAUNCHES] = (double)h->solve_launches;
    h->tm[TM_LAUNCHES] = (double)h->launches;
    int m = std::min(n, (int)TM_COUNT);
    for (int i = 0; i < m; ++i) ms[i] = h->tm[i];
    return m;
}

// gamma on the host (only to choose the covariance shift c0)
static double host_gamma(const kb200_ctx* h, const VgParams& v, double d) {
    switch (v.model) {
        case KB200_VG_LINEAR: return v.p0 * d + v.p1;
        case KB200_VG_POWER: return v.p0 * std::pow(d, v.p1) + v.p2;
        case KB200_VG_TABLE: {
            // same cubic Hermite as kb_gamma<KB200_VG_TABLE>; the largest tabulated value up to d, so that the
            // shift also covers non-monotone callables
            if (h->tab_n < 2) return 1.0;
            const double inv_h = (h->tab_n - 1) / std::sqrt(h->tab_dmax);
            int last = (int)std::min<double>(h->tab_n - 1, std::ceil(std::sqrt(std::max(d, 0.0)) * inv_h));
            double g = h->htab[0];
            for (int i = 0; i <= last; ++i) g = std::max(g, h->htab[2 * (size_t)i]);
            return g;
        }
        default: return v.p0 + v.p2;
    }
}

extern "C" int kb200_set_variogram_table(kb200_handle h, int64_t n_nodes, double dmax, const double* gamma_nodes) {
    if (!h) return KB200_EBADARG;
    if (n_nodes < 16 || n_nodes > (1LL << 26) || !gamma_nodes || !(dmax > 0.0) || !std::isfinite(dmax))
        return fail(h, KB200_EBADARG, "variogram table: 16 <= n_nodes <= 2^26, dmax > 0");
    const int n = (int)n_nodes;
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(gamma_nodes[i])) return fail(h, KB200_EBADARG, "variogram table: the callable must be finite on [0, dmax] (node " + std::to_string(i) + ")");
    drop_problem(h);
    // slopes per unit node index: centred differences, second-order one-sided at the two ends
    h->htab.resize(2 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        double m;
        if (i == 0) m = -1.5 * gamma_nodes[0] + 2.0 * gamma_nodes[1] - 0.5 * gamma_nodes[2];
        else if (i == n - 1) m = 1.5 * gamma_nodes[n - 1] - 2.0 * gamma_nodes[n - 2] + 0.5 * gamma_nodes[n - 3];
        else m = 0.5 * (gamma_nodes[i + 1] - gamma_nodes[i - 1]);
        h->htab[2 * (size_t)i] = gamma_nodes[i];
        h->htab[2 * (size_t)i + 1] = m;
    }
    h->tab_n = n; h->tab_dmax = dmax;
    cudaSetDevice(h->device);
    CU(h, h->wTab.reserve(h->htab.size() * sizeof(double)));
    CU(h, cudaMemcpyAsync(h->wTab.p, h->htab.data(), h->htab.size() * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return KB200_OK;
}

// [lo, hi] grown by the device coordinates of n points: adjusted with the handle's anisotropy (h->an), or the unit
// vectors of geographic lon/lat
static void extend_box(const kb200_ctx* h, int dim, int64_t n, const double* x, const double* y, const double* z,
                       double* lo, double* hi) {
    for (int64_t i = 0; i < n; ++i) {
        if (h->geo) {
            const double rad = 0.017453292519943295;
            double u[3] = {std::cos(x[i] * rad) * std::cos(y[i] * rad), std::sin(x[i] * rad) * std::cos(y[i] * rad),
                           std::sin(y[i] * rad)};
            for (int r = 0; r < 3; ++r) { lo[r] = std::min(lo[r], u[r]); hi[r] = std::max(hi[r], u[r]); }
            continue;
        }
        double d[3] = {x[i] - h->an.c[0], y[i] - h->an.c[1], dim == 3 ? z[i] - h->an.c[2] : 0.0};
        for (int r = 0; r < dim; ++r) {
            double v = h->an.c[r];
            for (int c = 0; c < dim; ++c) v += h->an.m[r * dim + c] * d[c];
            lo[r] = std::min(lo[r], v); hi[r] = std::max(hi[r], v);
        }
    }
}

static double box_diag2(int sdim, const double* lo, const double* hi) {
    double diag2 = 0.0;
    for (int r = 0; r < sdim; ++r) diag2 += (hi[r] - lo[r]) * (hi[r] - lo[r]);
    return diag2;
}

// ---- description (shared by set_problem / describe_problem / set_problem_knn) ----
static int layout(kb200_ctx* h, bool knn_only);
static int describe(kb200_ctx* h, bool knn_only, int dim, int dtype, int64_t n,
                    const double* x, const double* y, const double* z, const double* values,
                    const double* center, const double* aniso, int model, const double* vparams, int n_vparams,
                    int exact_values, double eps, int n_rl, int n_hd, const double* drift_data) {
    if (!h) return KB200_EBADARG;
    drop_problem(h);
    if (dim != 2 && dim != 3) return fail(h, KB200_EBADARG, "dim must be 2 or 3");
    if (h->geo && dim != 2) return fail(h, KB200_EBADARG, "geographic coordinates are two-dimensional (lon, lat)");
    if (h->geo && (n_rl || n_hd)) return fail(h, KB200_EUNSUPPORTED, "universal kriging has no geographic mode (uk.py:337)");
    if (dtype < KB200_F64 || dtype > KB200_F64X4)
        return fail(h, KB200_EBADARG, "dtype must be KB200_F64, KB200_F32, KB200_F64X, KB200_F64X5 or KB200_F64X4");
    if (n < 1 || (!knn_only && n > (int64_t)(KB_MAXRB - 1) * KB_BM) || n > (1LL << 30)) return fail(h, KB200_EBADARG, "n out of range");
    if (!x || !y || (dim == 3 && !z) || !values || !center || !aniso || (!vparams && model != KB200_VG_TABLE))
        return fail(h, KB200_EBADARG, "null input array");
    if (model < KB200_VG_LINEAR || model > KB200_VG_TABLE)
        return fail(h, KB200_EUNSUPPORTED, "variogram model has no device implementation");
    int need = (model == KB200_VG_TABLE) ? 0 : (model == KB200_VG_LINEAR) ? 2 : 3;
    if (model == KB200_VG_TABLE) {
        if (h->tab_n < 16) return fail(h, KB200_ESTATE, "KB200_VG_TABLE: call kb200_set_variogram_table first");
        if (n_vparams != 0 && !vparams) return fail(h, KB200_EBADARG, "null input array");
    } else if (n_vparams != need) return fail(h, KB200_EBADARG, "wrong number of variogram parameters");
    if (!(n_rl == 0 || n_rl == dim)) return fail(h, KB200_EBADARG, "n_rl must be 0 or dim");
    if (n_hd < 0 || n_rl + n_hd > KB200_MAX_DRIFT) return fail(h, KB200_EBADARG, "too many drift terms");
    if (n_hd > 0 && !drift_data) return fail(h, KB200_EBADARG, "drift_data is null");
    if (knn_only && (n_rl || n_hd)) return fail(h, KB200_EUNSUPPORTED, "moving window supports ordinary kriging only");
    const int n_dev = h->dd.n_wells + h->dd.ext;
    if (n_dev > n_hd) return fail(h, KB200_EBADARG, "device drift terms (kb200_set_device_drift) exceed the n_hd described drift columns");
    if (n_dev && dim != 2) return fail(h, KB200_EUNSUPPORTED, "point_log / external_Z drift terms are two-dimensional (uk.py)");
    h->n_dev = n_dev;
    if (h->nf) {
        if (n != h->nf_n) return fail(h, KB200_EBADARG, "kb200_set_values: the fields have " + std::to_string(h->nf_n) +
                                      " rows, the problem " + std::to_string(n) + " data points");
        if (!knn_only && dtype != KB200_F64) return fail(h, KB200_EUNSUPPORTED, "value fields run in float64 only");
        if (!knn_only && h->pinv) return fail(h, KB200_EUNSUPPORTED, "value fields are not supported with pseudo_inv=True");
    }
    h->slices = dtype == KB200_F64X ? 6 : dtype == KB200_F64X5 ? 5 : dtype == KB200_F64X4 ? 4 : 0;

    h->dim = h->geo ? KB_GEO : dim; h->dtype = dtype; h->n = (int)n; h->n_rl = n_rl; h->n_hd = n_hd;
    // dual rows: K + 1 drift/unbiasedness rows and one zeta row per value field (n + na <= n + 80 stays within
    // KB_MAXRB row blocks for every n the check above admits)
    h->K1 = n_rl + n_hd + 1; h->na = h->K1 + (h->nf ? h->nf : 1);
    h->aux_cols = std::max(KB_MAXAUX, h->na);
    h->vg.model = model;
    h->vg.p0 = need > 0 ? vparams[0] : 0.0; h->vg.p1 = need > 1 ? vparams[1] : 0.0; h->vg.p2 = (need == 3) ? vparams[2] : 0.0;
    h->vg.inv_a = 0.0;
    if (model == KB200_VG_EXPONENTIAL || model == KB200_VG_HOLE_EFFECT) h->vg.inv_a = 1.0 / (h->vg.p1 / 3.0);
    else if (model == KB200_VG_GAUSSIAN) { const double r = h->vg.p1 * (4.0 / 7.0); h->vg.inv_a = 1.0 / (r * r); }
    else if (model == KB200_VG_SPHERICAL) h->vg.inv_a = 1.0 / h->vg.p1;
    h->vg.tab = h->wTab.as<double2>(); h->vg.tab_n = h->tab_n;
    h->vg.tab_inv_h = h->tab_n > 1 ? (h->tab_n - 1) / std::sqrt(h->tab_dmax) : 0.0;
    h->vg.eps = eps; h->vg.exact = exact_values ? 1 : 0;
    for (int i = 0; i < 9; ++i) h->an.m[i] = 0.0;
    for (int i = 0; i < dim * dim; ++i) h->an.m[i] = aniso[i];
    for (int i = 0; i < 3; ++i) h->an.c[i] = i < dim ? center[i] : 0.0;
    h->hx.assign(x, x + n); h->hy.assign(y, y + n);
    if (dim == 3) h->hz.assign(z, z + n); else h->hz.assign(n, 0.0);
    h->hval.assign(values, values + n);
    if (n_hd) h->hdrift.assign(drift_data, drift_data + (size_t)n_hd * n); else h->hdrift.clear();

    // adjusted bounding box on the host (drift rescale + c0 for unbounded models)
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    const int sdim = h->geo ? 3 : dim;            // spatial dimensions of the device coordinates
    extend_box(h, dim, n, x, y, z, lo, hi);
    if (h->geo) for (int r = 0; r < 3; ++r) { lo[r] -= 1e-9; hi[r] += 1e-9; }   // device sincos may differ in the last ulp
    for (int r = 0; r < 3; ++r) { h->bb_lo[r] = r < sdim ? lo[r] : 0.0; h->bb_hi[r] = r < sdim ? hi[r] : 0.0; }
    const double diag2 = box_diag2(sdim, lo, hi);
    if (model == KB200_VG_TABLE && h->tab_dmax < (h->geo ? 180.0 : std::sqrt(diag2)))
        return fail(h, KB200_EBADARG, "variogram table: dmax is smaller than the extent of the data");
    double c0 = host_gamma(h, h->vg, h->geo ? 180.0 : std::sqrt(diag2));
    if (!(c0 > 0.0) || !std::isfinite(c0)) c0 = 1.0;
    h->vg.c0 = c0;
    for (int c = 0; c <= KB200_MAX_DRIFT; ++c) { h->ds.shift[c] = 0.0; h->ds.scale[c] = 1.0; }
    for (int c = 0; c < n_rl; ++c) {
        h->ds.shift[c] = 0.5 * (hi[c] + lo[c]);
        double half = 0.5 * (hi[c] - lo[c]);
        h->ds.scale[c] = half > 0.0 ? 1.0 / half : 1.0;
    }
    for (int c = 0; c < n_hd; ++c) {
        const double* col = drift_data + (size_t)c * n;
        double mean = 0.0;
        for (int64_t i = 0; i < n; ++i) mean += col[i];
        mean /= (double)n;
        double amax = 0.0;
        for (int64_t i = 0; i < n; ++i) amax = std::max(amax, std::fabs(col[i] - mean));
        h->ds.shift[n_rl + c] = mean;
        h->ds.scale[n_rl + c] = amax > 0.0 ? 1.0 / amax : 1.0;
    }

    if (h->pinv && !knn_only) {
        // pseudo-inverse of the reference's own matrix: gamma form (c0 = 0), raw drift columns (pinv.cu)
        if (dtype != KB200_F64) return fail(h, KB200_EUNSUPPORTED, "pseudo_inv=True runs in float64 only");
        if (n + h->K1 > kbk_pinv_max_nt())
            return fail(h, KB200_EUNSUPPORTED, "pseudo_inv=True supports at most " + std::to_string(kbk_pinv_max_nt() - h->K1) + " data points");
        h->vg.c0 = 0.0;
        for (int c = 0; c <= KB200_MAX_DRIFT; ++c) { h->ds.shift[c] = 0.0; h->ds.scale[c] = 1.0; }
    }
    int rc = layout(h, knn_only);
    if (rc) return rc;
    h->described = true;
    return KB200_OK;
}

// Tile stream map and blob layout of a problem of h->n data points; (re)allocates the blob
static int layout(kb200_ctx* h, bool knn_only) {
    const int64_t n = h->n;
    h->n_pad = (int)align_up((size_t)n, KB_BM);
    h->ld = h->n_pad;
    h->nrb = knn_only ? 0 : (int)((n + h->na + KB_BM - 1) / KB_BM);
    int nk = (int)((n + KB_BK - 1) / KB_BK);
    h->pm.nrb = h->nrb;
    long long off = 0;
    for (int I = 0; I < h->nrb; ++I) {
        bool has_dual = (I + 1) * KB_BM > n;     // block holds rows >= n (dual rows live there)
        int kt = has_dual ? nk : std::min(nk, (I + 1) * KB_BM / KB_BK);
        h->pm.ktiles[I] = kt;
        h->pm.tile_off[I] = off;
        off += kt;
    }
    size_t esz = 8;   // fp64 value, or TF32 hi + lo pair: both 8 bytes per element
    size_t o = 0;
    o += align_up(HDR_DOUBLES * sizeof(double), 256);
    h->off_consts = o; o += align_up((size_t)std::max(512, h->K1 * h->na) * sizeof(double), 256);   // S^-1 | phi_v
    h->off_ax = o; o += align_up((size_t)h->n_pad * 8, 256);
    h->off_ay = o; o += align_up((size_t)h->n_pad * 8, 256);
    h->off_az = o; o += align_up((size_t)h->n_pad * 8, 256);
    h->off_tiles = o;
    if (h->slices) {
        o += (size_t)kbk_i8_total_tiles(h->slices, (int)n, h->na, nullptr) * kbk_i8_tile_bytes(h->slices);
        o = align_up(o, 256);
        h->off_rowscale = o; o += align_up((size_t)kbk_i8_rows(h->slices, (int)n, h->na) * sizeof(double), 256);
    } else {
        o += (size_t)off * KB_BM * KB_BK * esz;
    }
    h->blob_bytes = knn_only ? h->off_tiles : o;
    cudaSetDevice(h->device);
    CU(h, h->blob.reserve(h->blob_bytes));
    return KB200_OK;
}

extern "C" int kb200_describe_problem(kb200_handle h, int dim, int dtype, int64_t n,
                                      const double* x, const double* y, const double* z, const double* values,
                                      const double* center, const double* aniso,
                                      int model, const double* vparams, int n_vparams,
                                      int exact_values, double eps, int n_rl, int n_hd, const double* drift_data) {
    if (h && h->nf) return fail(h, KB200_EUNSUPPORTED, "value fields (kb200_set_values) have no factor-blob form");
    return describe(h, false, dim, dtype, n, x, y, z, values, center, aniso, model, vparams, n_vparams,
                    exact_values, eps, n_rl, n_hd, drift_data);
}

extern "C" int64_t kb200_blob_bytes(kb200_handle h) { return (h && h->described) ? (int64_t)h->blob_bytes : 0; }
extern "C" void* kb200_blob_ptr(kb200_handle h) { return (h && h->described) ? h->blob.p : nullptr; }

extern "C" int kb200_blob_commit(kb200_handle h) {
    if (!h || !h->described) return fail(h, KB200_ESTATE, "describe the problem first");
    cudaSetDevice(h->device);
    double hdr[HDR_DOUBLES];
    CU(h, cudaMemcpyAsync(hdr, h->blob.p, sizeof(hdr), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    if (!read_header(h, hdr)) return fail(h, KB200_ESTATE, "blob does not hold a factored problem");
    h->ready = true;
    return KB200_OK;
}

static float ev_ms(cudaEvent_t a, cudaEvent_t b) { float t = 0.f; cudaEventElapsedTime(&t, a, b); return t; }

// The described data to wRaw (with `fields`, the value fields too) and its adjusted coordinates to the blob axes,
// zero beyond n. Timed as h2d: EV_UPLOAD .. EV_ADJUSTED.
static int upload_data(kb200_ctx* h, bool fields, int* launches) {
    cudaStream_t st = h->stream;
    const size_t col = (size_t)h->n * sizeof(double);
    CU(h, h->wRaw.reserve((4 + h->n_hd + (fields ? h->nf : 0)) * col));
    const BlobView b = blob_view(h);
    CU(h, cudaEventRecord(h->ev[EV_UPLOAD], st));
    CU(h, cudaMemcpyAsync(raw_col(h, RAW_X), h->hx.data(), col, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(raw_col(h, RAW_Y), h->hy.data(), col, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(raw_col(h, RAW_Z), h->hz.data(), col, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(raw_col(h, RAW_V), h->hval.data(), col, cudaMemcpyHostToDevice, st));
    if (h->n_hd) CU(h, cudaMemcpyAsync(raw_col(h, RAW_DRIFT), h->hdrift.data(), h->n_hd * col, cudaMemcpyHostToDevice, st));
    if (fields && h->nf)
        CU(h, cudaMemcpyAsync(kriged_values(h), h->hfields.data(), h->nf * col, cudaMemcpyHostToDevice, st));
    for (double* a : {b.ax, b.ay, b.az}) CU(h, cudaMemsetAsync(a, 0, (size_t)h->n_pad * 8, st));
    CU(h, kbk_adjust_data(h->dim, h->an, h->n, raw_col(h, RAW_X), raw_col(h, RAW_Y), raw_col(h, RAW_Z),
                          b.ax, b.ay, b.az, st)); ++*launches;
    CU(h, cudaEventRecord(h->ev[EV_ADJUSTED], st));
    return KB200_OK;
}

// The three factorisations of kb200_set_problem. Each returns the gform of its tiles (or an error code < 0); the
// flag it leaves in wFlag is non-zero when the drift/unbiasedness block is singular.

// pseudo_inv=True: A^+ of the bordered gamma-form matrix (pinv.cu), then the quadratic-form solve
static int factor_pinv(kb200_ctx* h, const BlobView& b, int* launches) {
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad, nt = nn + h->K1;
    double* Fz = aux_block(h, AUX_F);
    double* Uz = aux_block(h, AUX_U);
    int* flag = h->wFlag.as<int>();
    CU(h, h->wVario.reserve(kbk_pinv_workspace_doubles(nt) * sizeof(double)));
    CU(h, cudaMemsetAsync(flag, 0, sizeof(int), st));
    CU(h, cudaEventRecord(h->ev[EV_ASM], st));
    CU(h, kbk_assemble(h->dim, h->vg, nn, np, h->ld, 0, b.ax, b.ay, b.az, h->wC.as<double>(), st)); ++*launches;
    CU(h, cudaEventRecord(h->ev[EV_INVERT], st));
    CU(h, kbk_build_fz(nn, np, h->n_rl, h->n_hd, b.ax, b.ay, b.az, h->ds, raw_col(h, RAW_DRIFT), raw_col(h, RAW_V), Fz,
                       st)); ++*launches;
    CU(h, kbk_pinv(nn, h->K1, np, h->wC.as<double>(), h->ld, Fz, raw_col(h, RAW_V), Uz, b.consts, h->wVario.as<double>(),
                   flag, st, launches, &h->pinv_sweeps, &h->pinv_rank));
    h->tm[TM_ASSEMBLE] += ev_ms(h->ev[EV_ASM], h->ev[EV_INVERT]);     // kbk_pinv ends in a synchronise
    if (h->pinv_sweeps < 0) { h->launches += *launches; return fail(h, KB200_ESINGULAR, "pseudo-inverse: the Jacobi SVD did not converge"); }
    CU(h, cudaMemsetAsync(flag, 0, sizeof(int), st));
    CU(h, cudaEventRecord(h->ev[EV_DUAL], st));
    CU(h, kbk_pack_gform(h->wC.as<double>(), h->ld, nn, np, h->na, Uz, h->pm, b.tiles, st)); ++*launches;
    return 2;
}

// C is not positive definite: the variogram is not conditionally negative definite in this dimension (e.g. hole-effect
// on dense scatter). General fallback, from the unshifted c0: blocked Gauss-Jordan inverse with partial pivoting +
// quadratic-form solve (DESIGN.md §3b). fp64 only.
static int factor_general(kb200_ctx* h, const BlobView& b, double c0, int* launches) {
    if (h->dtype != KB200_F64) {
        h->launches += *launches;
        return fail(h, KB200_EUNSUPPORTED, "dtype float32 / float64x need a positive definite covariance form "
                    "(the variogram is not valid in this dimension); use float64");
    }
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad, ld = h->ld;
    double* G = h->wC.as<double>();
    int* flag = h->wFlag.as<int>();
    h->vg.c0 = c0;
    CU(h, cudaMemsetAsync(flag, 0, sizeof(int), st));
    CU(h, cudaEventRecord(h->ev[EV_FACTOR], st));
    CU(h, kbk_assemble(h->dim, h->vg, nn, np, ld, 0, b.ax, b.ay, b.az, G, st)); ++*launches;
    CU(h, h->wVario.reserve(kbk_general_inverse_workspace_bytes(np)));
    CU(h, kbk_general_inverse(G, ld, np, h->wVario.p, flag, 3.6e-15 * h->vg.c0, st, launches));
    CU(h, cudaEventRecord(h->ev[EV_INVERT], st));
    int hflag = 0;
    CU(h, cudaMemcpyAsync(&hflag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_CHOLESKY] += ev_ms(h->ev[EV_FACTOR], h->ev[EV_INVERT]);
    if (hflag != 0) {
        h->launches += *launches;
        return fail(h, KB200_ESINGULAR, "kriging matrix is singular (zero pivot in column " +
                    std::to_string(hflag - 1) + ")");
    }
    double* Uz = aux_block(h, AUX_U);
    CU(h, cudaEventRecord(h->ev[EV_DUAL], st));
    CU(h, kbk_dual_gform(G, ld, nn, np, h->n_rl, h->n_hd, h->nf ? h->nf : 1, b.ax, b.ay, b.az, h->ds,
                         raw_col(h, RAW_DRIFT), kriged_values(h), aux_block(h, AUX_F), Uz, b.consts, flag, st, launches));
    CU(h, kbk_pack_gform(G, ld, nn, np, h->na, Uz, h->pm, b.tiles, st)); ++*launches;
    return 1;
}

// W = L^-1 in wW: the dual vectors, and W packed into the tiles of the handle's dtype
static int dual_pack(kb200_ctx* h, const BlobView& b, int* launches) {
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad, ld = h->ld;
    double* W = h->wW.as<double>();
    double* Uz = aux_block(h, AUX_U);
    CU(h, cudaEventRecord(h->ev[EV_DUAL], st));
    CU(h, kbk_dual(W, ld, nn, np, h->n_rl, h->n_hd, h->nf ? h->nf : 1, b.ax, b.ay, b.az, h->ds, raw_col(h, RAW_DRIFT),
                   kriged_values(h), aux_block(h, AUX_F), aux_block(h, AUX_H), Uz, b.consts, h->wFlag.as<int>(), st,
                   launches));
    if (h->dtype == KB200_F32) {
        CU(h, kbk_pack_tf32(W, ld, nn, np, h->na, Uz, h->pm, b.tiles, st)); ++*launches;
    } else if (h->slices) {
        const int nrb8 = kbk_i8_nrb(h->slices, nn, h->na);
        std::vector<long long> toff(nrb8 + 1);
        kbk_i8_total_tiles(h->slices, nn, h->na, toff.data());
        // workspace (T1 scratch is free now): tile offsets | row exponents
        long long* d_toff = reinterpret_cast<long long*>(h->wT.as<char>());
        int* d_rowexp = reinterpret_cast<int*>(h->wT.as<char>() + align_up((size_t)(nrb8 + 1) * sizeof(long long), 256));   // kbk_i8_rows ints
        CU(h, cudaMemcpyAsync(d_toff, toff.data(), (size_t)(nrb8 + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
        CU(h, kbk_pack_i8(h->slices, W, ld, nn, np, h->na, Uz, d_rowexp, b.rowscale, d_toff, b.tiles, st));
        *launches += 2;                        // row scales + pack
        CU(h, cudaStreamSynchronize(st));      // toff is a host temporary
    } else {
        CU(h, kbk_pack(W, ld, nn, np, h->na, Uz, h->pm, b.tiles, st)); ++*launches;
    }
    return 0;
}

// C = L L^T (L in wC): W = L^-1 of the rows [n0, n_pad), then dual_pack
static int factor_cholesky_pack(kb200_ctx* h, const BlobView& b, int n0, int* launches) {
    CU(h, kbk_inverse_rows(h->wC.as<double>(), h->wW.as<double>(), h->wT.as<double>(), h->ld, h->n_pad, n0, h->stream,
                           launches));
    return dual_pack(h, b, launches);
}

// the high-priority side stream and the ordering events kbk_cholesky_rows needs for n_pad rows (kept on the handle)
static int cholesky_streams(kb200_ctx* h, int n_pad) {
    if (!h->hi_stream) {
        int lo = 0, hi = 0;
        CU(h, cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU(h, cudaStreamCreateWithPriority(&h->hi_stream, cudaStreamNonBlocking, hi));
    }
    const size_t need = 2 * (size_t)((n_pad / 64 + 3) / 4) + 1;
    while (h->fev.size() < need) {
        cudaEvent_t e;
        CU(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        h->fev.push_back(e);
    }
    return KB200_OK;
}

// Assembles the rows [n0, n_pad) of C with the handle's c0 and factors them (kbk_cholesky_rows; n0 = 0 for a new
// problem). Returns the pivot flag (0, or 1 + the column of a non-positive pivot counted from n0) or an error code < 0.
static int assemble_cholesky(kb200_ctx* h, const BlobView& b, int n0, int* launches) {
    cudaStream_t st = h->stream;
    const int np = h->n_pad, ld = h->ld;
    int* flag = h->wFlag.as<int>();
    const int rc = cholesky_streams(h, np - n0); if (rc) return rc;
    CU(h, cudaMemsetAsync(flag, 0, sizeof(int), st));
    CU(h, cudaEventRecord(h->ev[EV_ASM], st));
    CU(h, kbk_assemble(h->dim, h->vg, h->n, np, ld, n0 / 64, b.ax, b.ay, b.az, h->wC.as<double>(), st)); ++*launches;
    CU(h, cudaEventRecord(h->ev[EV_FACTOR], st));
    CU(h, kbk_cholesky_rows(h->wC.as<double>(), h->wW.as<double>(), h->wT.as<double>(), ld, np, n0, flag,
                            3.6e-15 * h->vg.c0, st, h->hi_stream, h->fev.data(), (int)h->fev.size(), launches));
    CU(h, cudaEventRecord(h->ev[EV_INVERT], st));
    int hflag = 0;
    CU(h, cudaMemcpyAsync(&hflag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_ASSEMBLE] += ev_ms(h->ev[EV_ASM], h->ev[EV_FACTOR]);
    h->tm[TM_CHOLESKY] += ev_ms(h->ev[EV_FACTOR], h->ev[EV_INVERT]);
    return hflag;
}

// The end of every global set-up, after the dual vectors and the pack: the header, the flag of the drift block, the
// timings and launches of the call. The handle then holds the problem.
static int finish_problem(kb200_ctx* h, const BlobView& b, int gform, int launches) {
    cudaStream_t st = h->stream;
    h->gform = gform;
    double hdr[HDR_DOUBLES];
    write_header(h, hdr);
    CU(h, cudaMemcpyAsync(b.hdr, hdr, sizeof(hdr), cudaMemcpyHostToDevice, st));
    CU(h, cudaEventRecord(h->ev[EV_PACKED], st));
    int hflag = 0;
    CU(h, cudaMemcpyAsync(&hflag, h->wFlag.as<int>(), sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_H2D] += ev_ms(h->ev[EV_UPLOAD], h->ev[EV_ADJUSTED]);
    h->tm[TM_TRTRI] += ev_ms(h->ev[EV_INVERT], h->ev[EV_DUAL]);
    h->tm[TM_PACK_DUAL] += ev_ms(h->ev[EV_DUAL], h->ev[EV_PACKED]);
    h->launches += launches;
    if (hflag != 0) return fail(h, KB200_ESINGULAR, "drift/unbiasedness block F^T C^-1 F is singular");
    h->ready = true;
    h->local_factor = true;
    return KB200_OK;
}

extern "C" int kb200_set_problem(kb200_handle h, int dim, int dtype, int64_t n,
                                 const double* x, const double* y, const double* z, const double* values,
                                 const double* center, const double* aniso,
                                 int model, const double* vparams, int n_vparams,
                                 int exact_values, double eps, int n_rl, int n_hd, const double* drift_data) {
    int rc = describe(h, false, dim, dtype, n, x, y, z, values, center, aniso, model, vparams, n_vparams,
                      exact_values, eps, n_rl, n_hd, drift_data);
    if (rc != KB200_OK) return rc;
    const int np = h->n_pad, ld = h->ld;
    const size_t mat = (size_t)np * ld * sizeof(double);
    CU(h, h->wC.reserve(mat)); CU(h, h->wW.reserve(mat)); CU(h, h->wT.reserve(mat));
    CU(h, h->wF.reserve((size_t)3 * h->aux_cols * np * sizeof(double)));
    CU(h, h->wFlag.reserve(256));
    const BlobView b = blob_view(h);
    int launches = 0;
    rc = upload_data(h, true, &launches); if (rc) return rc;

    // covariance shift: c0 = sill for bounded models; for linear/power grow c0 until C is
    // positive definite (DESIGN.md §3). A model that is not a valid variogram in this
    // dimension (e.g. hole-effect in 2-D/3-D) never becomes positive definite. pseudo_inv=True
    // factors nothing: the pseudo-inverse works on -Gamma itself.
    const bool unbounded = (h->vg.model == KB200_VG_LINEAR || h->vg.model == KB200_VG_POWER || h->vg.model == KB200_VG_TABLE);
    const int max_try = unbounded ? 5 : 1;
    const double c0_first = h->vg.c0;
    int hflag = 0;
    for (int attempt = 0; !h->pinv && attempt < max_try; ++attempt) {
        hflag = assemble_cholesky(h, b, 0, &launches); if (hflag < 0) return hflag;
        if (hflag != 0 && std::getenv("KB200_DEBUG")) std::fprintf(stderr, "[kb200] cholesky flag %d (attempt %d, c0 %g)\n", hflag, attempt, h->vg.c0);
        if (hflag == 0) break;
        h->vg.c0 *= 2.0;
    }
    CU(h, cudaMemsetAsync(b.consts, 0, (size_t)std::max(512, h->K1 * h->na) * sizeof(double), h->stream));
    const int gform = h->pinv ? factor_pinv(h, b, &launches)
                    : hflag ? factor_general(h, b, c0_first, &launches)
                    : factor_cholesky_pack(h, b, 0, &launches);
    if (gform < 0) return gform;
    return finish_problem(h, b, gform, launches);
}

// ---- appended stations (DESIGN.md §5g) ----------------------------------------------------------------------------
// rows and columns [0, keep) of a matrix of stride ld_old into a new allocation of `bytes` with the handle's stride
static int restride(kb200_ctx* h, DevBuf& b, int ld_old, int keep, size_t bytes) {
    DevBuf nb;
    CU(h, nb.reserve(bytes));
    if (keep > 0)
        CU(h, cudaMemcpy2DAsync(nb.p, (size_t)h->ld * 8, b.p, (size_t)ld_old * 8, (size_t)keep * 8, keep,
                                cudaMemcpyDeviceToDevice, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    b.release();
    std::swap(b.p, nb.p); std::swap(b.cap, nb.cap);
    return KB200_OK;
}

// The held problem grows by m stations (checked by kb200_append_data): the set-up of kb200_set_problem on the rows
// [n0, n_pad), n0 = the old n rounded down to the tile. Any error leaves it half-extended: the caller drops it.
static int append_extend(kb200_ctx* h, int m, const double* x, const double* y, const double* z, const double* values,
                         const double* drift_cols, const double* lo, const double* hi) {
    const int n_old = h->n, ld_old = h->ld, n0 = n_old / 64 * 64, nn = n_old + m;
    h->hx.insert(h->hx.end(), x, x + m);
    h->hy.insert(h->hy.end(), y, y + m);
    if (h->dim == 3) h->hz.insert(h->hz.end(), z, z + m); else h->hz.resize(nn, 0.0);
    h->hval.insert(h->hval.end(), values, values + m);
    if (h->n_hd) {                                    // column-major n x n_hd: each column grows by its m new rows
        std::vector<double> d((size_t)h->n_hd * nn);
        for (int c = 0; c < h->n_hd; ++c) {
            std::copy(h->hdrift.begin() + (size_t)c * n_old, h->hdrift.begin() + (size_t)(c + 1) * n_old, d.begin() + (size_t)c * nn);
            std::copy(drift_cols + (size_t)c * m, drift_cols + (size_t)(c + 1) * m, d.begin() + (size_t)c * nn + n_old);
        }
        h->hdrift.swap(d);
    }
    for (int r = 0; r < 3; ++r) { h->bb_lo[r] = lo[r]; h->bb_hi[r] = hi[r]; }
    h->n = nn;
    int rc = layout(h, false); if (rc) return rc;
    const int np = h->n_pad, ld = h->ld;
    const size_t mat = (size_t)np * ld * sizeof(double);
    if (ld != ld_old) {                               // n_pad grew: L11 and W11 move to the new stride
        rc = restride(h, h->wC, ld_old, n0, mat); if (rc) return rc;
        rc = restride(h, h->wW, ld_old, n0, mat); if (rc) return rc;
    }
    CU(h, h->wT.reserve(mat));
    CU(h, h->wF.reserve((size_t)3 * h->aux_cols * np * sizeof(double)));
    const BlobView b = blob_view(h);
    int launches = 0;
    rc = upload_data(h, true, &launches); if (rc) return rc;
    const int hflag = assemble_cholesky(h, b, n0, &launches); if (hflag < 0) return hflag;
    if (hflag != 0) {
        h->launches += launches;
        return fail(h, KB200_ESINGULAR, "kriging matrix is singular (zero pivot in column " + std::to_string(n0 + hflag - 1) + ")");
    }
    CU(h, cudaMemsetAsync(b.consts, 0, (size_t)std::max(512, h->K1 * h->na) * sizeof(double), h->stream));
    rc = factor_cholesky_pack(h, b, n0, &launches); if (rc) return rc;
    return finish_problem(h, b, 0, launches);
}

extern "C" int kb200_append_data(kb200_handle h, int64_t m, const double* x, const double* y, const double* z,
                                 const double* values, const double* drift_cols) {
    if (!h) return KB200_EBADARG;
    if (!h->ready || !h->local_factor)
        return fail(h, KB200_EUNSUPPORTED, "append: no global problem was factored on this handle");
    if (h->gform != 0)
        return fail(h, KB200_EUNSUPPORTED, "append: the held problem is not a positive definite covariance form "
                    "(pseudo-inverse or the indefinite fallback)");
    if (h->nf) return fail(h, KB200_EUNSUPPORTED, "append: value fields (kb200_set_values) have no append form");
    const int dim = h->dim == 3 ? 3 : 2;
    if (m < 1 || !x || !y || (dim == 3 && !z) || !values || (h->n_hd && !drift_cols))
        return fail(h, KB200_EBADARG, "append: m >= 1 and non-null arrays (drift_cols with drift columns)");
    if (h->n + m > (int64_t)(KB_MAXRB - 1) * KB_BM) return fail(h, KB200_EBADARG, "n out of range");
    double lo[3], hi[3];
    for (int r = 0; r < 3; ++r) { lo[r] = h->bb_lo[r]; hi[r] = h->bb_hi[r]; }
    const int sdim = h->geo ? 3 : dim;
    extend_box(h, dim, m, x, y, z, lo, hi);
    if (h->vg.model == KB200_VG_TABLE && h->tab_dmax < (h->geo ? 180.0 : std::sqrt(box_diag2(sdim, lo, hi))))
        return fail(h, KB200_EUNSUPPORTED, "append: the variogram table's dmax does not cover the extended data");
    cudaSetDevice(h->device);
    const int rc = append_extend(h, (int)m, x, y, z, values, drift_cols, lo, hi);
    if (rc) drop_problem(h);
    return rc;
}

// ---- device-evaluated drift terms -----------------------------------------------------------------------
extern "C" int kb200_set_device_drift(kb200_handle h, int n_wells, const double* wells,
                                      int64_t ext_nx, int64_t ext_ny, const double* ext_x, const double* ext_y,
                                      const double* ext_z) {
    if (!h) return KB200_EBADARG;
    if (n_wells < 0 || n_wells > KB200_MAX_DRIFT || (n_wells > 0 && !wells))
        return fail(h, KB200_EBADARG, "device drift: bad point_log description");
    const bool ext = ext_nx > 0 || ext_ny > 0;
    if (ext && (ext_nx < 1 || ext_ny < 1 || ext_nx > (1 << 30) || ext_ny > (1 << 30) || !ext_x || !ext_y || !ext_z))
        return fail(h, KB200_EBADARG, "device drift: bad external_Z raster description");
    drop_problem(h);
    cudaSetDevice(h->device);
    h->dd = DeviceDrift{};
    if (n_wells) {
        CU(h, h->wWells.reserve((size_t)3 * n_wells * 8));
        CU(h, cudaMemcpyAsync(h->wWells.p, wells, (size_t)3 * n_wells * 8, cudaMemcpyHostToDevice, h->stream));
        h->dd.n_wells = n_wells; h->dd.wells = h->wWells.as<double>();
    }
    if (ext) {
        const size_t nx = (size_t)ext_nx, ny = (size_t)ext_ny;
        CU(h, h->wExt.reserve((nx + ny + nx * ny) * 8));
        double* d = h->wExt.as<double>();
        CU(h, cudaMemcpyAsync(d, ext_x, nx * 8, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(d + nx, ext_y, ny * 8, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(d + nx + ny, ext_z, nx * ny * 8, cudaMemcpyHostToDevice, h->stream));
        bool sorted = true;
        for (size_t i = 1; i < nx && sorted; ++i) sorted = ext_x[i] >= ext_x[i - 1];
        for (size_t i = 1; i < ny && sorted; ++i) sorted = ext_y[i] >= ext_y[i - 1];
        h->dd.ext = 1; h->dd.ext_nx = (int)ext_nx; h->dd.ext_ny = (int)ext_ny; h->dd.ext_sorted = sorted ? 1 : 0;
        h->dd.ext_x = d; h->dd.ext_y = d + nx; h->dd.ext_z = d + nx + ny;
    }
    CU(h, cudaStreamSynchronize(h->stream));     // the caller's arrays may go away
    return KB200_OK;
}

// ---- execute --------------------------------------------------------------
// One persistent launch of the solve kernel of the handle's dtype over points [s.first, s.first + s.count) with point
// tiles of `tp` points. One kernel serves every point count: the summation order per point must not depend on how the
// points are sharded or chunked (concatenated shards == single call, bit for bit; SURVEY.md §4 (iii)).
static int launch_solve(kb200_ctx* h, const Src& s, double* d_z, double* d_ss, int tp) {
    cudaStream_t st = h->stream;
    const BlobView b = blob_view(h);
    const bool wg = h->dtype != KB200_F64;
    long long ntiles = (s.count + tp - 1) / tp;
    int grid = (int)std::min<long long>(ntiles, h->num_sms);
    CU(h, h->wScratch.reserve(wg ? kbk_solve_wgmma_scratch_bytes(h->slices, h->n, grid)
                                 : kbk_solve_pt_scratch_doubles(h->n, grid) * sizeof(double)));
    SolvePtParams pp{};
    pp.vg = h->vg; pp.an = h->an; pp.ps = s.point_source();
    pp.n = h->n; pp.na = h->na; pp.nrb = h->nrb; pp.n_rl = h->n_rl; pp.n_hd = h->n_hd;
    pp.ax = b.ax; pp.ay = b.ay; pp.az = b.az;
    pp.tiles = b.tiles; pp.pm = h->pm; pp.ds = h->ds;
    pp.consts = b.consts;
    pp.dd = h->dd; pp.n_dev = h->n_dev;
    pp.drift_pts = s.d_drift; pp.drift_stride = s.drift_stride; pp.drift_first = s.drift_first;
    pp.m = s.count; pp.scratch = h->wScratch.as<double>(); pp.gform = h->gform;
    pp.z_out = d_z; pp.ss_out = d_ss;
    pp.nf = h->nf; pp.zstride = h->zstride;
    if (h->nf) {
        CU(h, h->wFstage.reserve((size_t)grid * h->na * tp * sizeof(double)));
        pp.fstage = h->wFstage.as<double>();
    }
    pp.rowscale = b.rowscale;
    if (wg) CU(h, kbk_solve_wgmma(h->slices, h->dim, pp, grid, st));
    else CU(h, kbk_solve_pt(h->dim, pp, grid, tp, st));
    h->launches += 1; h->solve_launches += 1;
    return KB200_OK;
}

// Relative cost of one round of the fp64 kernel with 64 / 32 / 16-point tiles (a tile streams all of W once whatever its
// width; the DMMA work is proportional to the width), at N=5000 (scripts/tile_timing.py).
static double tile_cost(int tp) { return tp == 64 ? 1.0 : (tp == 32 ? KB_TILE_COST_32 : KB_TILE_COST_16); }

// NOTE: the summation order per point does not depend on the tile width or on the number of launches either, so the
// split below is free to choose them.
static int run_solve(kb200_ctx* h, const Src& s, double* d_z, double* d_ss) {
    if (h->dtype != KB200_F64) return launch_solve(h, s, d_z, d_ss, KB_WG_TM);
    // fp64 DMMA kernel: full rounds of 64-point tiles over all SMs, then the leftover points as ONE more launch whose tile
    // width minimises rounds x cost: a partial round of 64-point tiles keeps a few SMs busy for a whole tile time
    const long long S = h->num_sms;
    const int TW = h->nf ? KB_TN_FIELDS : KB_TN;               // widest tile of the kernel variant
    if (const char* e = std::getenv("KB200_TILE")) {           // profiling override: one launch, fixed width
        const int t = std::min(std::atoi(e), TW);
        if (t == 64 || t == 32 || t == 16) return launch_solve(h, s, d_z, d_ss, t);
    }
    const long long nt64 = (s.count + TW - 1) / TW;
    const long long main_pts = std::min<long long>(s.count, (nt64 / S) * S * TW);
    const long long rem = s.count - main_pts;
    if (main_pts > 0) {
        int rc = launch_solve(h, s.sub(0, main_pts), d_z, d_ss, TW); if (rc) return rc;
    }
    if (rem > 0) {
        int best = TW; double bc = 1e300;
        for (int tp : {64, 32, 16}) {
            if (tp > TW) continue;
            const long long nt = (rem + tp - 1) / tp;
            const double c = (double)((nt + S - 1) / S) * tile_cost(tp);
            if (c < bc * 0.999) { bc = c; best = tp; }
        }
        int rc = launch_solve(h, s.sub(main_pts, rem), d_z + main_pts, d_ss + main_pts, best); if (rc) return rc;
    }
    return KB200_OK;
}

// Launch `total` points in chunks and bring (z, ss) to the caller's HOST buffers. Large outputs travel through two
// pinned staging buffers on a second stream while the next chunk computes; the host drains a buffer into the
// caller's (pageable) memory while the GPU works. launch(o, m, d_z, d_ss) enqueues points [o, o+m) of the call.
// With value fields z has nf blocks of `total` (field f at z + f * total), on the device as in the caller's buffer.
template <class Launch>
static int run_to_host(kb200_ctx* h, int64_t total, double* z_out, double* ss_out, Launch launch) {
    cudaStream_t st = h->stream;
    const int nzb = h->nf ? h->nf : 1;               // z blocks; a staging buffer holds nzb + 1 blocks (z ..., ss)
    h->zstride = total;
    CU(h, h->wOut.reserve((size_t)(nzb + 1) * total * 8));
    double* dz = h->wOut.as<double>();
    double* dss = dz + (size_t)nzb * total;
    CU(h, cudaEventRecord(h->ev[EV_RUN], st));
    if (total < KB_STAGE_MIN) {
        int rc = launch((int64_t)0, total, dz, dss); if (rc) return rc;
        CU(h, cudaEventRecord(h->ev[EV_RUN_END], st));
        CU(h, cudaMemcpyAsync(z_out, dz, (size_t)nzb * total * 8, cudaMemcpyDeviceToHost, st));
        CU(h, cudaMemcpyAsync(ss_out, dss, total * 8, cudaMemcpyDeviceToHost, st));
        CU(h, cudaEventRecord(h->ev[EV_D2H_END], st));
        CU(h, cudaStreamSynchronize(st));
        h->tm[TM_D2H] += ev_ms(h->ev[EV_RUN_END], h->ev[EV_D2H_END]);
        return KB200_OK;
    }
    if (!h->copy_stream) {
        CU(h, cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CU(h, cudaEventCreateWithFlags(&h->evk[i], cudaEventDisableTiming));
            CU(h, cudaEventCreate(&h->evc[i]));
        }
    }
    if (h->pin_blocks < nzb + 1) {
        for (int i = 0; i < 2; ++i) {
            if (h->pin[i]) { CU(h, cudaFreeHost(h->pin[i])); h->pin[i] = nullptr; }
            CU(h, cudaHostAlloc(&h->pin[i], (size_t)(nzb + 1) * KB_STAGE_PTS * 8, cudaHostAllocDefault));
        }
        h->pin_blocks = nzb + 1;
    }
    const int64_t nch = (total + KB_STAGE_PTS - 1) / KB_STAGE_PTS;
    auto chunk_len = [&](int64_t c) { return std::min<int64_t>(KB_STAGE_PTS, total - c * KB_STAGE_PTS); };
    auto drain = [&](int64_t c) -> int {          // staged chunk c -> the caller's buffers
        const int b = (int)(c & 1);
        CU(h, cudaEventSynchronize(h->evc[b]));
        const double* p = reinterpret_cast<const double*>(h->pin[b]);
        const int64_t m = chunk_len(c);
        for (int f = 0; f < nzb; ++f)
            std::memcpy(z_out + (size_t)f * total + c * KB_STAGE_PTS, p + (size_t)f * KB_STAGE_PTS, (size_t)m * 8);
        std::memcpy(ss_out + c * KB_STAGE_PTS, p + (size_t)nzb * KB_STAGE_PTS, (size_t)m * 8);
        return KB200_OK;
    };
    for (int64_t c = 0; c < nch; ++c) {
        const int b = (int)(c & 1);
        const int64_t o = c * KB_STAGE_PTS, m = chunk_len(c);
        int rc = launch(o, m, dz + o, dss + o); if (rc) return rc;
        CU(h, cudaEventRecord(h->evk[b], st));
        if (c == nch - 1) CU(h, cudaEventRecord(h->ev[EV_RUN_END], st));
        if (c >= 2) { rc = drain(c - 2); if (rc) return rc; }
        double* p = reinterpret_cast<double*>(h->pin[b]);
        CU(h, cudaStreamWaitEvent(h->copy_stream, h->evk[b], 0));
        for (int f = 0; f < nzb; ++f)
            CU(h, cudaMemcpyAsync(p + (size_t)f * KB_STAGE_PTS, dz + (size_t)f * total + o, (size_t)m * 8,
                                  cudaMemcpyDeviceToHost, h->copy_stream));
        CU(h, cudaMemcpyAsync(p + (size_t)nzb * KB_STAGE_PTS, dss + o, (size_t)m * 8, cudaMemcpyDeviceToHost, h->copy_stream));
        CU(h, cudaEventRecord(h->evc[b], h->copy_stream));
    }
    for (int64_t c = std::max<int64_t>(0, nch - 2); c < nch; ++c) { int rc = drain(c); if (rc) return rc; }
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_D2H] += ev_ms(h->ev[EV_RUN_END], h->evc[(nch - 1) & 1]);
    return KB200_OK;
}

static int check_ready(kb200_ctx* h) {
    if (!h) return KB200_EBADARG;
    if (!h->ready) return fail(h, KB200_ESTATE, "no factored problem: call kb200_set_problem (or blob_commit) first");
    cudaSetDevice(h->device);
    return KB200_OK;
}
static int n_host_drift(const kb200_ctx* h) { return h->n_hd - h->n_dev; }

static int check_grid(kb200_ctx* h, int64_t nx, int64_t ny, int64_t nz, int64_t first, int64_t count) {
    if (nx < 1 || ny < 1 || nz < 1 || first < 0 || count < 0 || first + count > nx * ny * nz)
        return fail(h, KB200_EBADARG, "bad grid slice");
    if (h->dim != 3 && nz != 1) return fail(h, KB200_EBADARG, "nz must be 1 for 2-D");
    return KB200_OK;
}

// the caller's arrays of an execute call: the points or axes, the outputs and (if the problem has host drift columns)
// the drift values at the points
static int check_io(kb200_ctx* h, const double* a, const double* b, const double* c, const double* drift,
                    const double* z, const double* ss) {
    if (!a || !b || (h->dim == 3 && !c) || !z || !ss) return fail(h, KB200_EBADARG, "null pointer");
    if (n_host_drift(h) && !drift) return fail(h, KB200_EBADARG, "drift values at the points are required");
    return KB200_OK;
}

// the global solve of points already on the device, into the caller's device buffers
static int solve_dev(kb200_ctx* h, const Src& s, double* d_z, double* d_ss) {
    if (s.count <= 0) return KB200_OK;
    int rc = check_io(h, s.a, s.b, s.c, s.d_drift, d_z, d_ss); if (rc) return rc;
    h->zstride = s.count;
    CU(h, cudaEventRecord(h->ev[EV_RUN], h->stream));
    rc = run_solve(h, s, d_z, d_ss); if (rc) return rc;
    CU(h, cudaEventRecord(h->ev[EV_RUN_END], h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    h->tm[TM_SOLVE] += ev_ms(h->ev[EV_RUN], h->ev[EV_RUN_END]);
    return KB200_OK;
}

extern "C" int kb200_execute_points_dev(kb200_handle h, int64_t m,
                                        const double* d_px, const double* d_py, const double* d_pz,
                                        const double* d_drift_pts, double* d_z, double* d_ss) {
    int rc = check_ready(h); if (rc) return rc;
    return solve_dev(h, Src{false, 0, 0, 0, d_px, d_py, d_pz, 0, m, d_drift_pts, m, 0}, d_z, d_ss);
}

extern "C" int kb200_execute_grid_dev(kb200_handle h, int64_t nx, int64_t ny, int64_t nz,
                                      const double* d_gx, const double* d_gy, const double* d_gz,
                                      const double* d_drift_pts, int64_t first, int64_t count,
                                      double* d_z, double* d_ss) {
    int rc = check_ready(h); if (rc) return rc;
    rc = check_grid(h, nx, ny, nz, first, count); if (rc) return rc;
    return solve_dev(h, Src{true, nx, ny, nz, d_gx, d_gy, d_gz, first, count, d_drift_pts, count, 0}, d_z, d_ss);
}

// ---- moving window ----------------------------------------------------------
extern "C" int kb200_set_problem_knn(kb200_handle h, int dim, int64_t n,
                                     const double* x, const double* y, const double* z, const double* values,
                                     const double* center, const double* aniso,
                                     int model, const double* vparams, int n_vparams, int exact_values, double eps) {
    int rc = describe(h, true, dim, KB200_F64, n, x, y, z, values, center, aniso, model, vparams, n_vparams,
                      exact_values, eps, 0, 0, nullptr);
    if (rc != KB200_OK) return rc;
    cudaStream_t st = h->stream;
    const int nn = h->n;
    int launches = 0;
    rc = upload_data(h, false, &launches); if (rc) return rc;
    const BlobView b = blob_view(h);
    // uniform cell grid with ~2 points per cell over the adjusted bounding box
    KnnParams& kp = h->kp;
    kp = KnnParams{};
    double ext[3] = {0, 0, 0}, vol = 1.0; int live = 0;
    const int sdim = h->dim == KB_GEO ? 3 : h->dim;
    for (int r = 0; r < sdim; ++r) { ext[r] = h->bb_hi[r] - h->bb_lo[r]; if (ext[r] > 0.0) { vol *= ext[r]; ++live; } }
    double cell = live ? std::pow(vol * 2.0 / (double)nn, 1.0 / live) : 1.0;
    if (!(cell > 0.0) || !std::isfinite(cell)) cell = 1.0;
    int g[3] = {1, 1, 1};
    for (;;) {
        long long tot = 1;
        for (int r = 0; r < sdim; ++r) {
            double cnt = std::floor(ext[r] / cell) + 1.0;
            g[r] = (int)std::min(cnt, 4096.0);
            tot *= g[r];
        }
        if (tot <= (1LL << 22)) break;
        cell *= 1.5;
    }
    // a cell edge slightly larger than ext/g keeps every data point inside the grid after clamping
    for (int r = 0; r < sdim; ++r) if (g[r] == 4096) cell = std::max(cell, ext[r] / 4095.0);
    kp.dim = h->dim; kp.n = nn; kp.gx = g[0]; kp.gy = g[1]; kp.gz = g[2];
    kp.ox = h->bb_lo[0]; kp.oy = h->bb_lo[1]; kp.oz = h->bb_lo[2];
    kp.cell = cell; kp.inv_cell = 1.0 / cell;
    int ncells = g[0] * g[1] * g[2];
    h->k_ncells = ncells;
    CU(h, h->kSorted.reserve((size_t)nn * (4 * sizeof(double) + 2 * sizeof(int))));
    CU(h, h->kCells.reserve((size_t)2 * (ncells + 1) * sizeof(int)));
    CU(h, h->wFlag.reserve(256));
    double* sx = h->kSorted.as<double>();
    double *sy = sx + nn, *sz = sy + nn, *sv = sz + nn;
    int* sorig = reinterpret_cast<int*>(sv + nn);
    int* cell_of = sorig + nn;
    int* cell_start = h->kCells.as<int>();
    int* cursor = cell_start + (ncells + 1);
    CU(h, kbk_knn_build(h->dim, nn, b.ax, b.ay, b.az, raw_col(h, RAW_V), kp, sx, sy, sz, sv, sorig, cell_of, cell_start,
                        cursor, ncells, st, &launches));
    if (h->nf) {                                   // value fields, field-major in the cell-sorted order
        const size_t fb = (size_t)h->nf * nn * sizeof(double);
        CU(h, h->kFields.reserve(2 * fb));
        double* raw_f = h->kFields.as<double>() + (size_t)h->nf * nn;
        CU(h, cudaMemcpyAsync(raw_f, h->hfields.data(), fb, cudaMemcpyHostToDevice, st));
        CU(h, kbk_knn_sort_fields(nn, h->nf, sorig, raw_f, h->kFields.as<double>(), st)); ++launches;
        kp.values = h->kFields.as<double>(); kp.nv = h->nf;
    }
    CU(h, cudaEventRecord(h->ev[EV_KNN_BUILT], st));
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_H2D] += ev_ms(h->ev[EV_UPLOAD], h->ev[EV_ADJUSTED]);
    h->tm[TM_KNN_SEARCH] += ev_ms(h->ev[EV_ADJUSTED], h->ev[EV_KNN_BUILT]);
    h->launches += launches;
    h->knn_ready = true;
    return KB200_OK;
}

// mode, sg, qg: kbk_knn_solve's mode and group arrays (1: leave-one-out, 2: leave-group-out of the stations)
static int run_knn(kb200_ctx* h, int k, const Src& s, double* d_z, double* d_ss, int chol, int mode = 0,
                   const int* sg = nullptr, const int* qg = nullptr) {
    cudaStream_t st = h->stream;
    KnnParams kp = h->kp;
    kp.vg = h->vg; kp.an = h->an; kp.k = k;
    {   // radius (in cells) of the ball expected to hold k points at the mean density
        double ppc = (double)h->n / (double)std::max(1, h->k_ncells);
        int live = 0;
        if (kp.gx > 1) ++live; if (kp.gy > 1) ++live; if (kp.gz > 1) ++live;
        double cells = (double)k / std::max(ppc, 1e-9);
        double R = live >= 3 ? std::cbrt(cells * 3.0 / (4.0 * 3.14159265358979)) : (live == 2 ? std::sqrt(cells / 3.14159265358979) : 0.5 * cells);
        kp.r0 = (int)std::min(64.0, std::max(1.0, std::ceil(R)));
    }
    kp.ps = s.point_source(); kp.m = s.count; kp.z_out = d_z; kp.ss_out = d_ss; kp.flag = h->wFlag.as<int>(); kp.zstride = h->zstride;
    CU(h, kbk_knn_solve(kp, chol, st, mode, sg, qg));
    h->launches += 1; h->solve_launches += 1;
    return KB200_OK;
}

static int check_knn(kb200_ctx* h, int k) {
    if (!h) return KB200_EBADARG;
    if (!h->knn_ready) return fail(h, KB200_ESTATE, "call kb200_set_problem_knn first");
    cudaSetDevice(h->device);
    if (k < 2) return fail(h, KB200_EBADARG, "n_closest_points has to be at least two!");
    if (k > h->n) return fail(h, KB200_EBADARG, "n_closest_points exceeds the number of data points");
    if (kbk_knn_smem_per_warp(k, 0, 1, 1) > 200 * 1024) return fail(h, KB200_EUNSUPPORTED, "n_closest_points too large for the shared-memory local solver");
    return KB200_OK;
}

// Run the moving window and handle the solver flag: 2 = a local covariance block was not positive definite (variogram
// not valid in this dimension) -> repeat with the pivoted-LU solver (dgesv semantics); 1 = exactly singular local
// system -> ValueError('Singular matrix') (cok.pyx:176-179). run(chol) enqueues the whole call between EV_RUN and
// EV_RUN_END.
template <class Run>
static int knn_retry(kb200_ctx* h, Run run) {
    int* flag = h->wFlag.as<int>();
    for (int chol = 1; chol >= 0; --chol) {
        CU(h, cudaMemsetAsync(flag, 0, sizeof(int), h->stream));
        int rc = run(chol); if (rc) return rc;
        int hflag = 0;
        CU(h, cudaMemcpyAsync(&hflag, flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        h->tm[TM_KNN_SOLVE] += ev_ms(h->ev[EV_RUN], h->ev[EV_RUN_END]);
        if (hflag == 0) return KB200_OK;
        if (hflag != 2 || chol == 0) return fail(h, KB200_ESINGULAR, "Singular matrix");
    }
    return KB200_OK;
}

static int knn_to_host(kb200_ctx* h, int k, const Src& s, double* z_out, double* ss_out, int mode = 0,
                       const int* sg = nullptr, const int* qg = nullptr) {
    return knn_retry(h, [&](int chol) {
        return run_to_host(h, s.count, z_out, ss_out, [&](int64_t o, int64_t c, double* dz, double* dss) {
            return run_knn(h, k, s.sub(o, c), dz, dss, chol, mode, sg, qg);
        });
    });
}

extern "C" int kb200_execute_knn_grid_dev(kb200_handle h, int k, int64_t nx, int64_t ny, int64_t nz,
                                          const double* d_gx, const double* d_gy, const double* d_gz,
                                          int64_t first, int64_t count, double* d_z, double* d_ss) {
    int rc = check_knn(h, k); if (rc) return rc;
    rc = check_grid(h, nx, ny, nz, first, count); if (rc) return rc;
    if (count == 0) return KB200_OK;
    rc = check_io(h, d_gx, d_gy, d_gz, nullptr, d_z, d_ss); if (rc) return rc;
    const Src s{true, nx, ny, nz, d_gx, d_gy, d_gz, first, count, nullptr, 0, 0};
    h->zstride = count;
    return knn_retry(h, [&](int chol) {
        CU(h, cudaEventRecord(h->ev[EV_RUN], h->stream));
        int rc = run_knn(h, k, s, d_z, d_ss, chol); if (rc) return rc;
        CU(h, cudaEventRecord(h->ev[EV_RUN_END], h->stream));
        return KB200_OK;
    });
}

// ---- execute to host buffers ----------------------------------------------------------------------------------
// The prediction points of a host execute call: explicit points or grid axes. The caller's arrays (its outputs and
// host drift columns) cover its slice [cfirst, cfirst + ccount) of the points; this call computes [first, first + count).
struct Query {
    bool grid; int64_t nx, ny, nz;
    const double *a, *b, *c;      // px, py, pz or gx, gy, gz
    const double* drift;
    int64_t cfirst, ccount, first, count;
};

// host drift columns [n_host][stride] -> device columns [n_host][m] holding items [off, off + m) of each column
static int upload_drift(kb200_ctx* h, const double* drift_pts, int64_t stride, int64_t off, int64_t m, const double** dd) {
    *dd = nullptr;
    const int nh = n_host_drift(h);
    if (!nh) return KB200_OK;
    CU(h, h->wDrift.reserve((size_t)nh * m * 8));
    for (int c = 0; c < nh; ++c)
        CU(h, cudaMemcpyAsync(h->wDrift.as<double>() + (size_t)c * m, drift_pts + (size_t)c * stride + off, (size_t)m * 8,
                              cudaMemcpyHostToDevice, h->stream));
    *dd = h->wDrift.as<double>();
    return KB200_OK;
}

// The query's explicit points [first, first + count) (or all its grid axes) and its host drift columns to the device,
// timed as h2d (EV_H2D .. EV_H2D_END). *s is the device source of the query's points; s->sub(o, c) that of [o, o + c).
static int upload_query(kb200_ctx* h, const Query& q, Src* s) {
    cudaStream_t st = h->stream;
    const int64_t off = q.first - q.cfirst;
    const int64_t len[3] = {q.grid ? q.nx : q.count, q.grid ? q.ny : q.count, q.grid ? q.nz : q.count};
    const double* src[3] = {q.a, q.b, q.c};
    CU(h, h->wPts.reserve((size_t)(len[0] + len[1] + len[2]) * 8));
    double* col[3] = {h->wPts.as<double>(), h->wPts.as<double>() + len[0], h->wPts.as<double>() + len[0] + len[1]};
    CU(h, cudaEventRecord(h->ev[EV_H2D], st));
    for (int r = 0; r < (h->dim == 3 ? 3 : 2); ++r)
        CU(h, cudaMemcpyAsync(col[r], src[r] + (q.grid ? 0 : off), len[r] * 8, cudaMemcpyHostToDevice, st));
    const double* dd = nullptr;
    int rc = upload_drift(h, q.drift, q.ccount, off, q.count, &dd); if (rc) return rc;
    CU(h, cudaEventRecord(h->ev[EV_H2D_END], st));
    *s = Src{q.grid, q.nx, q.ny, q.nz, col[0], col[1], col[2], q.grid ? q.first : 0, q.count, dd, q.count, 0};
    return KB200_OK;
}

// One handle's share of a host execute call, by the global solve or (knn) the moving window with k neighbours
static int exec_host(kb200_ctx* h, bool knn, int k, const Query& q, double* z_out, double* ss_out) {
    int rc = knn ? check_knn(h, k) : check_ready(h); if (rc) return rc;
    if (q.grid) { rc = check_grid(h, q.nx, q.ny, q.nz, q.first, q.count); if (rc) return rc; }
    if (q.count <= 0) return KB200_OK;
    rc = check_io(h, q.a, q.b, q.c, q.drift, z_out, ss_out); if (rc) return rc;
    Src s{};
    rc = upload_query(h, q, &s); if (rc) return rc;
    const int64_t off = q.first - q.cfirst;
    rc = knn ? knn_to_host(h, k, s, z_out + off, ss_out + off)
             : run_to_host(h, q.count, z_out + off, ss_out + off, [&](int64_t o, int64_t c, double* dz, double* dss) {
                   return run_solve(h, s.sub(o, c), dz, dss);
               });
    if (rc) return rc;
    h->tm[TM_H2D] += ev_ms(h->ev[EV_H2D], h->ev[EV_H2D_END]);
    if (!knn) h->tm[TM_SOLVE] += ev_ms(h->ev[EV_RUN], h->ev[EV_RUN_END]);
    return KB200_OK;
}

extern "C" int kb200_execute_points(kb200_handle h, int64_t m,
                                    const double* px, const double* py, const double* pz,
                                    const double* drift_pts, double* z_out, double* ss_out) {
    return exec_host(h, false, 0, Query{false, 0, 0, 0, px, py, pz, drift_pts, 0, m, 0, m}, z_out, ss_out);
}

extern "C" int kb200_execute_grid(kb200_handle h, int64_t nx, int64_t ny, int64_t nz,
                                  const double* gx, const double* gy, const double* gz,
                                  const double* drift_pts, int64_t first, int64_t count,
                                  double* z_out, double* ss_out) {
    return exec_host(h, false, 0, Query{true, nx, ny, nz, gx, gy, gz, drift_pts, first, count, first, count}, z_out, ss_out);
}

extern "C" int kb200_execute_knn_grid(kb200_handle h, int k, int64_t nx, int64_t ny, int64_t nz,
                                      const double* gx, const double* gy, const double* gz,
                                      int64_t first, int64_t count, double* z_out, double* ss_out) {
    return exec_host(h, true, k, Query{true, nx, ny, nz, gx, gy, gz, nullptr, first, count, first, count}, z_out, ss_out);
}

extern "C" int kb200_execute_knn_points(kb200_handle h, int k, int64_t m,
                                        const double* px, const double* py, const double* pz,
                                        double* z_out, double* ss_out) {
    return exec_host(h, true, k, Query{false, 0, 0, 0, px, py, pz, nullptr, 0, m, 0, m}, z_out, ss_out);
}

// ---- single-process multi-GPU: a group of handles driven by one caller thread --------------------------------
// SURVEY.md §8(b)/(e): the caller makes ONE call from one host thread; inside, one worker thread per device runs
// the per-device call on that device's handle (CUDA work of different devices overlaps, and so do the host-side
// drains of the staged outputs). Device 0 factors; the factor blob goes to the peers by cudaMemcpyPeerAsync over
// NVLink (the single transfer of the path); prediction points are cut into contiguous blocks in the reference's
// flattened order (ok.py:864-866), so the gathered result equals the single-GPU result bit for bit.
struct kb200_group_ctx {
    std::vector<kb200_ctx*> m;
    bool peers = false;
    std::string err;
};

static int gfail(kb200_group_ctx* g, int code, const std::string& msg) { if (g) g->err = msg; return code; }

template <class F>
static int group_parallel(kb200_group_ctx* g, F f) {
    const int G = (int)g->m.size();
    std::vector<int> rc(G, KB200_OK);
    std::vector<std::thread> th;
    th.reserve(G);
    for (int i = 1; i < G; ++i) th.emplace_back([&, i]() { rc[i] = f(i); });
    rc[0] = f(0);
    for (auto& t : th) t.join();
    for (int i = 0; i < G; ++i)
        if (rc[i] != KB200_OK) return gfail(g, rc[i], "device " + std::to_string(g->m[i]->device) + ": " + g->m[i]->err);
    return KB200_OK;
}

// f(member, first, n) on every member, with points [0, count) cut into one contiguous block per member
template <class F>
static int group_sharded(kb200_group_ctx* g, int64_t count, F f) {
    if (!g || g->m.empty()) return KB200_EBADARG;
    const int64_t G = (int64_t)g->m.size(), base = count / G, rem = count % G;
    return group_parallel(g, [&](int i) {
        return f(g->m[i], i * base + std::min<int64_t>(i, rem), base + (i < rem ? 1 : 0));
    });
}

extern "C" int kb200_group_create(kb200_group* out, int n_gpus, const int* devices) {
    if (!out) return KB200_EBADARG;
    *out = nullptr;
    int cnt = 0;
    if (cudaGetDeviceCount(&cnt) != cudaSuccess || cnt == 0) return KB200_ECUDA;
    if (n_gpus < 1 || n_gpus > cnt) return KB200_EBADARG;
    kb200_group_ctx* g = new kb200_group_ctx();
    for (int i = 0; i < n_gpus; ++i) {
        kb200_handle h = nullptr;
        int rc = kb200_create(&h, devices ? devices[i] : i);
        if (rc != KB200_OK) { for (auto* m : g->m) kb200_destroy(m); delete g; return rc; }
        g->m.push_back(h);
    }
    *out = g;
    return KB200_OK;
}

extern "C" void kb200_group_destroy(kb200_group g) {
    if (!g) return;
    for (auto* m : g->m) kb200_destroy(m);
    delete g;
}

extern "C" const char* kb200_group_last_error(kb200_group g) { return g ? g->err.c_str() : "null group"; }
extern "C" int kb200_group_size(kb200_group g) { return g ? (int)g->m.size() : 0; }
extern "C" kb200_handle kb200_group_member(kb200_group g, int i) {
    return (g && i >= 0 && i < (int)g->m.size()) ? g->m[i] : nullptr;
}

extern "C" int kb200_group_set_problem(kb200_group g, int dim, int dtype, int64_t n,
                                       const double* x, const double* y, const double* z, const double* values,
                                       const double* center, const double* aniso,
                                       int model, const double* vparams, int n_vparams,
                                       int exact_values, double eps, int n_rl, int n_hd, const double* drift_data) {
    if (!g || g->m.empty()) return KB200_EBADARG;
    for (auto* m : g->m) if (m->nf) return gfail(g, KB200_EUNSUPPORTED, "value fields (kb200_set_values) have no group form");
    // member 0 assembles + factors while the peers describe the problem (allocating their blobs)
    int rc = group_parallel(g, [&](int i) {
        if (i == 0) return kb200_set_problem(g->m[0], dim, dtype, n, x, y, z, values, center, aniso, model, vparams,
                                             n_vparams, exact_values, eps, n_rl, n_hd, drift_data);
        return kb200_describe_problem(g->m[i], dim, dtype, n, x, y, z, values, center, aniso, model, vparams,
                                      n_vparams, exact_values, eps, n_rl, n_hd, drift_data);
    });
    if (rc) return rc;
    const int G = (int)g->m.size();
    kb200_ctx* h0 = g->m[0];
    if (G > 1 && !g->peers) {
        for (int i = 1; i < G; ++i) {
            int can = 0;
            cudaDeviceCanAccessPeer(&can, g->m[i]->device, h0->device);
            if (can) { cudaSetDevice(g->m[i]->device); cudaDeviceEnablePeerAccess(h0->device, 0); cudaGetLastError(); }
        }
        g->peers = true;
    }
    cudaSetDevice(h0->device);
    for (int i = 1; i < G; ++i) {
        if (g->m[i]->blob_bytes != h0->blob_bytes) return gfail(g, KB200_ESTATE, "group: blob size mismatch");
        cudaError_t e = cudaMemcpyPeerAsync(g->m[i]->blob.p, g->m[i]->device, h0->blob.p, h0->device, h0->blob_bytes, h0->stream);
        if (e != cudaSuccess) return gfail(g, KB200_ECUDA, std::string("cudaMemcpyPeerAsync: ") + cudaGetErrorString(e));
    }
    if (cudaStreamSynchronize(h0->stream) != cudaSuccess) return gfail(g, KB200_ECUDA, "group: blob copy failed");
    for (int i = 1; i < G; ++i) {
        rc = kb200_blob_commit(g->m[i]);
        if (rc) return gfail(g, rc, g->m[i]->err);
    }
    return KB200_OK;
}

extern "C" int kb200_group_set_problem_knn(kb200_group g, int dim, int64_t n,
                                           const double* x, const double* y, const double* z, const double* values,
                                           const double* center, const double* aniso,
                                           int model, const double* vparams, int n_vparams, int exact_values, double eps) {
    if (!g || g->m.empty()) return KB200_EBADARG;
    for (auto* m : g->m) if (m->nf) return gfail(g, KB200_EUNSUPPORTED, "value fields (kb200_set_values) have no group form");
    // every device builds its own cell grid from the coordinates (1.6-2.4 MB of input; nothing to broadcast)
    return group_parallel(g, [&](int i) {
        return kb200_set_problem_knn(g->m[i], dim, n, x, y, z, values, center, aniso, model, vparams, n_vparams,
                                     exact_values, eps);
    });
}

extern "C" int kb200_group_execute_grid(kb200_group g, int64_t nx, int64_t ny, int64_t nz,
                                        const double* gx, const double* gy, const double* gz,
                                        const double* drift_pts, int64_t first, int64_t count,
                                        double* z_out, double* ss_out) {
    return group_sharded(g, count, [&](kb200_ctx* h, int64_t f, int64_t c) {
        return exec_host(h, false, 0, Query{true, nx, ny, nz, gx, gy, gz, drift_pts, first, count, first + f, c}, z_out, ss_out);
    });
}

extern "C" int kb200_group_execute_points(kb200_group g, int64_t m,
                                          const double* px, const double* py, const double* pz,
                                          const double* drift_pts, double* z_out, double* ss_out) {
    return group_sharded(g, m, [&](kb200_ctx* h, int64_t f, int64_t c) {
        return exec_host(h, false, 0, Query{false, 0, 0, 0, px, py, pz, drift_pts, 0, m, f, c}, z_out, ss_out);
    });
}

extern "C" int kb200_group_execute_knn_grid(kb200_group g, int k, int64_t nx, int64_t ny, int64_t nz,
                                            const double* gx, const double* gy, const double* gz,
                                            int64_t first, int64_t count, double* z_out, double* ss_out) {
    return group_sharded(g, count, [&](kb200_ctx* h, int64_t f, int64_t c) {
        return exec_host(h, true, k, Query{true, nx, ny, nz, gx, gy, gz, nullptr, first, count, first + f, c}, z_out, ss_out);
    });
}

extern "C" int kb200_group_execute_knn_points(kb200_group g, int k, int64_t m,
                                              const double* px, const double* py, const double* pz,
                                              double* z_out, double* ss_out) {
    return group_sharded(g, m, [&](kb200_ctx* h, int64_t f, int64_t c) {
        return exec_host(h, true, k, Query{false, 0, 0, 0, px, py, pz, nullptr, 0, m, f, c}, z_out, ss_out);
    });
}

// ---- constructor-side helpers (SURVEY.md 8f next-2) -----------------------------------------------
extern "C" int kb200_experimental_variogram(kb200_handle h, int dim, int64_t n,
                                            const double* x, const double* y, const double* z, const double* values,
                                            int nlags, double* counts, double* lag_sum, double* semi_sum,
                                            double* dminmax) {
    if (!h) return KB200_EBADARG;
    if (dim != 2 && dim != 3) return fail(h, KB200_EBADARG, "dim must be 2 or 3");
    if (h->geo && dim != 2) return fail(h, KB200_EBADARG, "Geographic coordinate type only supported for 2D datasets.");
    if (n < 2 || n > 2000000000LL) return fail(h, KB200_EBADARG, "the experimental variogram needs 2 <= n < 2^31 points");
    if (nlags < 1 || nlags > 4096) return fail(h, KB200_EBADARG, "nlags must be in [1, 4096]");
    if (!x || !y || (dim == 3 && !z) || !values || !counts || !lag_sum || !semi_sum)
        return fail(h, KB200_EBADARG, "null array");
    cudaSetDevice(h->device);
    cudaStream_t st = h->stream;
    const int nn = (int)n, kdim = h->geo ? KB_GEO : dim;
    // persistent CTAs: as many per SM as the (private-bin) shared memory allows, up to 8 — the pair loop is a
    // chain of shared-memory read-modify-writes and square roots, so it needs warps to hide latency
    const size_t ev_sm = kbk_ev_smem(nlags, nlags <= kbk_ev_priv_max_lags() ? 1 : 0) + 1024;
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (size_t)(220 * 1024) / ev_sm));
    const int grid = kbk_ev_grid(nn, per_sm * h->num_sms);
    // workspace: x | y | z | v | edges | bmin | bmax | part | out
    const size_t o_edges = 4 * (size_t)nn, o_bmin = o_edges + nlags + 1, o_bmax = o_bmin + grid,
                 o_part = o_bmax + grid, o_out = o_part + (size_t)grid * 3 * nlags, total = o_out + 3 * (size_t)nlags;
    CU(h, h->wVario.reserve(total * sizeof(double)));
    double* w = h->wVario.as<double>();
    double *dx = w, *dy = w + nn, *dz = w + 2 * (size_t)nn, *dv = w + 3 * (size_t)nn;
    CU(h, cudaMemcpyAsync(dx, x, (size_t)nn * 8, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(dy, y, (size_t)nn * 8, cudaMemcpyHostToDevice, st));
    if (dim == 3) CU(h, cudaMemcpyAsync(dz, z, (size_t)nn * 8, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(dv, values, (size_t)nn * 8, cudaMemcpyHostToDevice, st));
    CU(h, kbk_ev_minmax(kdim, nn, dx, dy, dz, grid, w + o_bmin, w + o_bmax, st));
    std::vector<double> mm(2 * (size_t)grid);
    CU(h, cudaMemcpyAsync(mm.data(), w + o_bmin, 2 * (size_t)grid * 8, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    double dmin = mm[0], dmax = mm[grid];
    for (int b = 1; b < grid; ++b) { dmin = std::min(dmin, mm[b]); dmax = std::max(dmax, mm[grid + b]); }
    if (!(dmax >= dmin)) return fail(h, KB200_EBADARG, "pair distances are not finite");
    // equal-width lag edges exactly as core.py:471-476 (same fp64 expression, evaluated on the host)
    const double dd = (dmax - dmin) / nlags;
    std::vector<double> edges(nlags + 1);
    for (int k = 0; k < nlags; ++k) edges[k] = dmin + k * dd;
    edges[nlags] = dmax + 0.001;
    CU(h, cudaMemcpyAsync(w + o_edges, edges.data(), (size_t)(nlags + 1) * 8, cudaMemcpyHostToDevice, st));
    CU(h, kbk_ev_bin(kdim, nn, dx, dy, dz, dv, nlags, w + o_edges, dd > 0.0 ? 1.0 / dd : 0.0, grid,
                     w + o_part, w + o_out, st));
    std::vector<double> out(3 * (size_t)nlags);
    CU(h, cudaMemcpyAsync(out.data(), w + o_out, out.size() * 8, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    for (int k = 0; k < nlags; ++k) { counts[k] = out[k]; lag_sum[k] = out[nlags + k]; semi_sum[k] = out[2 * (size_t)nlags + k]; }
    if (dminmax) { dminmax[0] = dmin; dminmax[1] = dmax; }
    h->launches += 3;
    return KB200_OK;
}

extern "C" int kb200_statistics(kb200_handle h, double* delta, double* sigma) {
    if (!h || !delta || !sigma) return KB200_EBADARG;
    if (!h->ready) return fail(h, KB200_ESTATE, "no factored problem: call kb200_set_problem first");
    if (h->nf) return fail(h, KB200_EUNSUPPORTED, "cross-validation statistics belong to the problem's own values, "
                           "not to kb200_set_values fields");
    if (h->gform) return fail(h, KB200_EUNSUPPORTED, "cross-validation statistics need the positive definite "
                              "covariance form (this problem runs on the general fallback)");
    if (!h->local_factor) return fail(h, KB200_ESTATE, "the Cholesky factor is not on this handle "
                                      "(problem received through kb200_blob_commit)");
    cudaSetDevice(h->device);
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad;
    const BlobView b = blob_view(h);
    const double* Hz = aux_block(h, AUX_H);
    const int K = h->n_rl + h->n_hd;                       // Hz row K = L^-1 1, row K+1 = L^-1 Z
    CU(h, h->wVario.reserve((size_t)nn * (2 * sizeof(double) + sizeof(int)) + 256));
    double* d_delta = h->wVario.as<double>();
    double* d_sigma = d_delta + nn;
    int* d_dup = reinterpret_cast<int*>(d_sigma + nn);
    CU(h, kbk_statistics(h->dim, nn, b.ax, b.ay, b.az, h->wC.as<double>(), h->ld,
                         Hz + (size_t)K * np, Hz + (size_t)(K + 1) * np, d_dup, d_delta, d_sigma, st));
    CU(h, cudaMemcpyAsync(delta, d_delta, (size_t)nn * 8, cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(sigma, d_sigma, (size_t)nn * 8, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->launches += 2;
    return KB200_OK;
}

// ---- debug tap (tests only) ------------------------------------------------
extern "C" int64_t kb200_debug_fetch(kb200_handle h, int what, double* out, int64_t cap) {
    if (!h || !out) return KB200_EBADARG;
    if (!h->described) return KB200_ESTATE;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    const size_t mat = (size_t)h->n_pad * h->ld;
    const void* src = nullptr; size_t cnt = 0;
    if (what == 1) { src = h->wC.p; cnt = mat; }
    else if (what == 2) { src = h->wW.p; cnt = mat; }
    else if (what == 4) { src = h->wT.p; cnt = mat; }     // G = W^T W after a kb200_lgo call (gform 0)
    else if (what == 3) {
        size_t nU = (size_t)h->na * h->n_pad;
        size_t nc = (size_t)h->K1 * h->na;            // Sinv ((K+1)^2) | phi_v ((K+1) per field)
        size_t total = nU + nc + 1;
        if ((int64_t)total > cap) return KB200_EBADARG;
        if (cudaMemcpy(out, aux_block(h, AUX_U), nU * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return KB200_ECUDA;
        if (cudaMemcpy(out + nU, blob_view(h).consts, nc * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return KB200_ECUDA;
        out[total - 1] = h->vg.c0;
        return (int64_t)total;
    } else return KB200_EBADARG;
    if (!src) return KB200_ESTATE;
    if ((int64_t)cnt > cap) return KB200_EBADARG;
    if (cudaMemcpy(out, src, cnt * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return KB200_ECUDA;
    return (int64_t)cnt;
}

// ---- leave-one-out cross-validation of every station (DESIGN.md §5e) ---------------------------------------------
// |P_ii| at or below this fraction of its two terms is the rounding noise of their difference: without station i the
// drift block is singular (e.g. universal kriging with n - 1 < K + 1 stations, or the rest collinear for a linear drift)
static const double KB_LOO_TOL = 1e-10;

// the preconditions of the global cross-validation paths; what ("leave-one-out", "leave-group-out") names the feature
static int check_cv(kb200_ctx* h, const double* z_out, const double* ss_out, const char* what) {
    if (!h || !z_out || !ss_out) return KB200_EBADARG;
    if (!h->ready) return fail(h, KB200_ESTATE, "no factored problem: call kb200_set_problem first");
    if (h->gform == 2) return fail(h, KB200_EUNSUPPORTED, std::string(what) + " needs the inverse of the kriging matrix; "
                                   "the pseudo-inverse (pseudo_inv=True) does not give it");
    if (!h->local_factor) return fail(h, KB200_ESTATE, "the factorisation is not on this handle "
                                      "(problem received through kb200_blob_commit)");
    return KB200_OK;
}

// exact_values: the stations j != i within eps of every station i (grp, a device array: only those of another group),
// ascending j. The lists stay on the device (h->wPairs), station i's at pj/pd + off[i], and st lists the stations that
// have any. Only the counts come to the host, where more than LOO_MAXDUP for one station refuse the call.
struct NearPairs {
    std::vector<int> cnt, hoff, st;            // host: count and list offset of every station, the stations with near
                                               // pairs (ascending)
    const int* d_st = nullptr; const int* off = nullptr; const int* pj = nullptr; const double* pd = nullptr;
};
static int near_pairs(kb200_ctx* h, const int* grp, const char* what, const char* others, NearPairs& np, int* launches) {
    cudaStream_t st = h->stream;
    const int nn = h->n;
    const BlobView b = blob_view(h);
    // ints: cnt [n] | off [n + 1] | st [n], then doubles: pd, then ints: pj
    const size_t pd_at = align_up((3 * (size_t)nn + 1) * sizeof(int), sizeof(double));
    CU(h, h->wPairs.reserve(pd_at));
    int* cnt = h->wPairs.as<int>();
    CU(h, kbk_loo_pairs(h->dim, nn, b.ax, b.ay, b.az, h->vg.eps, grp, cnt, nullptr, nullptr, nullptr, st)); ++*launches;
    np.cnt.resize(nn);
    CU(h, cudaMemcpyAsync(np.cnt.data(), cnt, (size_t)nn * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    std::vector<int>& hoff = np.hoff;
    hoff.assign(nn + 1, 0);
    for (int i = 0; i < nn; ++i) {
        if (np.cnt[i] > LOO_MAXDUP)
            return fail(h, KB200_EUNSUPPORTED, std::string(what) + ": station " + std::to_string(i) + " has " +
                        std::to_string(np.cnt[i]) + " " + others + " within eps (at most " + std::to_string(LOO_MAXDUP) + ")");
        hoff[i + 1] = hoff[i] + np.cnt[i];
        if (np.cnt[i]) np.st.push_back(i);
    }
    if (np.st.empty()) return KB200_OK;
    const size_t tot = (size_t)hoff[nn];
    CU(h, h->wPairs.reserve(pd_at + tot * (sizeof(double) + sizeof(int))));      // the counts are on the host now
    int* off = h->wPairs.as<int>() + nn;
    int* dst = off + nn + 1;
    double* pd = reinterpret_cast<double*>(h->wPairs.as<char>() + pd_at);
    int* pj = reinterpret_cast<int*>(pd + tot);
    CU(h, cudaMemcpyAsync(off, hoff.data(), (size_t)(nn + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(dst, np.st.data(), np.st.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(h, kbk_loo_pairs(h->dim, nn, b.ax, b.ay, b.az, h->vg.eps, grp, nullptr, off, pj, pd, st)); ++*launches;
    np.d_st = dst; np.off = off; np.pj = pj; np.pd = pd;
    return KB200_OK;
}

extern "C" int kb200_loo(kb200_handle h, double* z_out, double* ss_out) {
    int rc = check_cv(h, z_out, ss_out, "leave-one-out"); if (rc) return rc;
    cudaSetDevice(h->device);
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad, nv = h->nf ? h->nf : 1;
    const int nch = (nn + LOO_RC - 1) / LOO_RC;
    // doubles: part [nch][n] | pii [n] | alpha [nv][n] | z [nv][n] | ss [n], then the int bad
    const size_t nd = ((size_t)nch + 2 + 2 * (size_t)nv) * nn;
    CU(h, h->wLoo.reserve(nd * sizeof(double) + sizeof(int)));
    double* part = h->wLoo.as<double>();
    double* pii = part + (size_t)nch * nn;
    double* alpha = pii + nn;
    double* dz = alpha + (size_t)nv * nn;
    double* dss = dz + (size_t)nv * nn;
    int* bad = reinterpret_cast<int*>(h->wLoo.as<double>() + nd);
    const BlobView b = blob_view(h);
    int launches = 0;
    NearPairs dup;
    if (h->vg.exact) { rc = near_pairs(h, nullptr, "leave-one-out", "other stations", dup, &launches); if (rc) return rc; }

    CvParams p{};
    p.n = nn; p.n_pad = np; p.ld = h->ld; p.K1 = h->K1; p.nv = nv; p.gform = h->gform; p.nchunks = nch;
    p.tol = KB_LOO_TOL; p.vg = h->vg;
    p.W = h->wW.as<double>(); p.G = h->wC.as<double>(); p.part = part;
    p.Uz = aux_block(h, AUX_U);
    p.consts = b.consts;
    p.Z = kriged_values(h);
    p.pii = pii; p.alpha = alpha; p.z_out = dz; p.ss_out = dss; p.bad = bad;
    const int big = INT_MAX;
    CU(h, cudaMemcpyAsync(bad, &big, sizeof(int), cudaMemcpyHostToDevice, st));
    CU(h, cudaEventRecord(h->ev[EV_RUN], st));
    if (h->gform == 0) { CU(h, kbk_loo_colsq(p.W, p.ld, nn, part, st)); ++launches; }
    CU(h, kbk_loo_finalize(p, st)); ++launches;
    if (!dup.st.empty()) {
        CU(h, kbk_loo_dup(p, (int)dup.st.size(), dup.d_st, dup.off, dup.pj, dup.pd, st)); ++launches;
    }
    CU(h, cudaEventRecord(h->ev[EV_RUN_END], st));
    int hbad = big;
    CU(h, cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(z_out, dz, (size_t)nv * nn * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(ss_out, dss, (size_t)nn * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->tm[TM_SOLVE] += ev_ms(h->ev[EV_RUN], h->ev[EV_RUN_END]);
    h->launches += launches; h->solve_launches += launches;
    if (hbad != big)
        return fail(h, KB200_ESINGULAR, "leave-one-out: without station " + std::to_string(hbad) +
                    " the drift terms are not determined (singular drift block)");
    return KB200_OK;
}

// the stations' raw coordinates as the query points of the moving-window cross-validation
static Src station_queries(kb200_ctx* h) {
    return Src{false, 0, 0, 0, raw_col(h, RAW_X), raw_col(h, RAW_Y), raw_col(h, RAW_Z), 0, h->n, nullptr, 0, 0};
}

extern "C" int kb200_knn_loo(kb200_handle h, int k, double* z_out, double* ss_out) {
    int rc = check_knn(h, k); if (rc) return rc;
    if (k > h->n - 1) return fail(h, KB200_EBADARG, "leave-one-out: n_closest_points must be at most n - 1");
    if (!z_out || !ss_out) return fail(h, KB200_EBADARG, "null pointer");
    return knn_to_host(h, k, station_queries(h), z_out, ss_out, 1);
}

// ---- leave-group-out cross-validation (DESIGN.md §5f) ---------------------------------------------------------------
// group[i] in [0, n_groups), n_groups >= 2, no empty group; sizes[g] = stations of group g
static int check_groups(kb200_ctx* h, const int32_t* group, int n_groups, std::vector<int>& sizes) {
    if (!group) return fail(h, KB200_EBADARG, "null pointer");
    if (n_groups < 2 || n_groups > h->n) return fail(h, KB200_EBADARG, "leave-group-out: n_groups must be in [2, n]");
    sizes.assign(n_groups, 0);
    for (int i = 0; i < h->n; ++i) {
        if (group[i] < 0 || group[i] >= n_groups)
            return fail(h, KB200_EBADARG, "leave-group-out: group of station " + std::to_string(i) + " outside [0, n_groups)");
        ++sizes[group[i]];
    }
    for (int g = 0; g < n_groups; ++g)
        if (!sizes[g]) return fail(h, KB200_EBADARG, "leave-group-out: group " + std::to_string(g) + " is empty");
    return KB200_OK;
}

extern "C" int kb200_lgo(kb200_handle h, const int32_t* group, int n_groups, double* z_out, double* ss_out) {
    int rc = check_cv(h, z_out, ss_out, "leave-group-out"); if (rc) return rc;
    std::vector<int> sizes;
    rc = check_groups(h, group, n_groups, sizes); if (rc) return rc;
    if (n_groups == h->n) return kb200_loo(h, z_out, ss_out);      // every group a singleton: leave-one-out
    cudaSetDevice(h->device);
    cudaStream_t st = h->stream;
    const int nn = h->n, np = h->n_pad, ld = h->ld, nv = h->nf ? h->nf : 1;
    const BlobView b = blob_view(h);
    int launches = 0;

    // host lists: stations group by group (ascending inside a group), positions, block offsets, small / large groups
    std::vector<int> goff(n_groups + 1, 0), mem(nn), pos(nn), small, large;
    std::vector<long long> boff(n_groups);
    for (int g = 0; g < n_groups; ++g) goff[g + 1] = goff[g] + sizes[g];
    {
        std::vector<int> cur(goff.begin(), goff.end() - 1);
        for (int i = 0; i < nn; ++i) { pos[i] = cur[group[i]] - goff[group[i]]; mem[cur[group[i]]++] = i; }
    }
    long long nblk = 0; int max_small = 0, max_m = 0;
    for (int g = 0; g < n_groups; ++g) {
        boff[g] = nblk; nblk += (long long)sizes[g] * sizes[g];
        max_m = std::max(max_m, sizes[g]);
        if (sizes[g] <= LGO_SMALL) { small.push_back(g); max_small = std::max(max_small, sizes[g]); }
        else large.push_back(g);
    }

    // workspace (doubles): blk | scale [n] | alpha [nv][n] | e [nv][n] | z [nv][n] | ss [n] | pii [n]; then long long:
    // boff; then int: grp | mem | goff | pos | small | bad | the leave-one-out finalize's bad
    const size_t ndbl = (size_t)nblk + (size_t)nn * (3 + 3 * (size_t)nv);
    const size_t nint = 3 * (size_t)nn + goff.size() + small.size() + 2;
    CU(h, h->wLgo.reserve(ndbl * 8 + boff.size() * 8 + nint * 4));
    double* blk = h->wLgo.as<double>();
    double* scale = blk + nblk;
    double* alpha = scale + nn;
    double* de = alpha + (size_t)nv * nn;
    double* dz = de + (size_t)nv * nn;
    double* dss = dz + (size_t)nv * nn;
    double* lpii = dss + nn;
    long long* dboff = reinterpret_cast<long long*>(lpii + nn);
    int* dgrp = reinterpret_cast<int*>(dboff + boff.size());
    int* dmem = dgrp + nn; int* dgoff = dmem + nn; int* dpos = dgoff + goff.size(); int* dsmall = dpos + nn;
    int* bad = dsmall + small.size(); int* lbad = bad + 1;
    auto up = [&](void* d, const void* s, size_t bytes) {
        return bytes ? cudaMemcpyAsync(d, s, bytes, cudaMemcpyHostToDevice, st) : cudaSuccess;
    };
    CU(h, up(dgrp, group, (size_t)nn * 4)); CU(h, up(dmem, mem.data(), (size_t)nn * 4));
    CU(h, up(dgoff, goff.data(), goff.size() * 4)); CU(h, up(dpos, pos.data(), (size_t)nn * 4));
    CU(h, up(dsmall, small.data(), small.size() * 4)); CU(h, up(dboff, boff.data(), boff.size() * 8));
    const int big = INT_MAX;
    CU(h, up(bad, &big, 4));

    // exact_values: near pairs of stations in different groups (the pairs inside a group are held out together), and
    // in wLoo (free during this call) the correction's scratch of each such station: soff | P_jS and P_jS Q (|D| x m)
    NearPairs dup;
    if (h->vg.exact) {
        rc = near_pairs(h, dgrp, "leave-group-out", "stations of other groups", dup, &launches); if (rc) return rc;
    }
    const int nst = (int)dup.st.size();
    std::vector<long long> soff(1, 0);
    for (int i : dup.st) soff.push_back(soff.back() + 2LL * dup.cnt[i] * sizes[group[i]]);
    CU(h, h->wLoo.reserve((soff.size() + (size_t)soff.back()) * 8));
    long long* dsoff = h->wLoo.as<long long>();
    double* dscr = reinterpret_cast<double*>(dsoff + soff.size());
    CU(h, up(dsoff, soff.data(), soff.size() * 8));

    // G = C^-1: W^T W into wT (free after kb200_set_problem), or the Gauss-Jordan inverse already in wC
    CU(h, cudaEventRecord(h->ev[EV_RUN], st));
    const double* G = h->wC.as<double>();
    if (h->gform == 0) {
        CU(h, kbk_gram_lower(h->wW.as<double>(), ld, np, h->wT.as<double>(), ld, st)); ++launches;
        G = h->wT.as<double>();
    }
    CU(h, cudaEventRecord(h->ev[EV_INVERT], st));
    CvParams p{};
    p.n = nn; p.n_pad = np; p.ld = ld; p.K1 = h->K1; p.nv = nv; p.gform = 1; p.nchunks = 0;
    p.tol = KB_LOO_TOL; p.vg = h->vg; p.G = G; p.Uz = aux_block(h, AUX_U); p.consts = b.consts;
    p.Z = kriged_values(h); p.pii = lpii; p.alpha = alpha;
    p.grp = dgrp; p.mem = dmem; p.goff = dgoff; p.pos = dpos; p.boff = dboff; p.blk = blk; p.scale = scale; p.e = de;
    p.z_out = dz; p.ss_out = dss; p.bad = lbad;
    // alpha_v = P Z_v: the leave-one-out finalize on G (its other outputs are overwritten below, and a station whose
    // P_ii is at rounding level, lbad, is no refusal of its group)
    CU(h, kbk_loo_finalize(p, st)); ++launches;
    p.bad = bad;
    CU(h, kbk_lgo_gather(p, n_groups, max_m, st)); ++launches;
    CU(h, kbk_lgo_small(p, (int)small.size(), dsmall, max_small, st)); launches += small.empty() ? 0 : 1;

    // large groups, one after another in one padded workspace: Cholesky -> triangular inverse -> W^T W, or Gauss-Jordan.
    // The padding's diagonal is the group's largest scale, so that it never looks like a pivot at rounding level.
    int large_bad = big;
    if (!large.empty()) {
        std::vector<double> hscale(nn);
        CU(h, cudaMemcpyAsync(hscale.data(), scale, (size_t)nn * 8, cudaMemcpyDeviceToHost, st));
        CU(h, cudaStreamSynchronize(st));
        const int mp = (int)align_up((size_t)max_m, 64);
        const size_t mat = (size_t)mp * mp;
        CU(h, h->wLgoM.reserve(3 * mat * sizeof(double) + 256));
        double* A = h->wLgoM.as<double>();
        double* Wm = A + mat;
        double* T1 = Wm + mat;
        int* flag = reinterpret_cast<int*>(T1 + mat);
        if (h->gform == 1) CU(h, h->wVario.reserve(kbk_general_inverse_workspace_bytes(mp)));
        rc = cholesky_streams(h, mp); if (rc) return rc;
        for (int g : large) {
            const int m = sizes[g], gp = (int)align_up((size_t)m, 64);
            double smax = 0.0;
            for (int a = goff[g]; a < goff[g + 1]; ++a) smax = std::max(smax, hscale[a]);
            if (!(smax > 0.0)) smax = 1.0;
            int hflag = 0;
            CU(h, cudaMemsetAsync(flag, 0, sizeof(int), st));
            CU(h, kbk_lgo_pad(blk + boff[g], m, A, gp, smax, st)); ++launches;
            if (h->gform == 0) {
                CU(h, kbk_cholesky_rows(A, Wm, T1, gp, gp, 0, flag, KB_LOO_TOL * smax, st, h->hi_stream, h->fev.data(),
                                        (int)h->fev.size(), &launches));
                CU(h, kbk_inverse_rows(A, Wm, T1, gp, gp, 0, st, &launches));
                CU(h, kbk_gram_lower(Wm, gp, gp, A, gp, st)); ++launches;
            } else {
                CU(h, kbk_general_inverse(A, gp, gp, h->wVario.p, flag, KB_LOO_TOL * smax, st, &launches));
            }
            CU(h, kbk_lgo_unpad(A, gp, blk + boff[g], m, st)); ++launches;
            CU(h, cudaMemcpyAsync(&hflag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
            CU(h, cudaStreamSynchronize(st));
            if (hflag != 0) { large_bad = g; break; }           // ascending order: the lowest large group that fails
        }
    }
    CU(h, cudaEventRecord(h->ev[EV_DUAL], st));
    CU(h, kbk_lgo_finalize(p, st)); ++launches;
    if (nst) { CU(h, kbk_lgo_dup(p, nst, dup.d_st, dup.off, dup.pj, dup.pd, dsoff, dscr, st)); ++launches; }
    CU(h, cudaEventRecord(h->ev[EV_RUN_END], st));
    int hbad = big;
    CU(h, cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(z_out, dz, (size_t)nv * nn * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(ss_out, dss, (size_t)nn * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    hbad = std::min(hbad, large_bad);
    h->tm[TM_SOLVE] += ev_ms(h->ev[EV_RUN], h->ev[EV_RUN_END]);
    h->tm[TM_TRTRI] += ev_ms(h->ev[EV_RUN], h->ev[EV_INVERT]);       // the Gram product W^T W
    h->tm[TM_FINALIZE] += ev_ms(h->ev[EV_INVERT], h->ev[EV_DUAL]);   // alpha, the blocks and their inverses
    h->launches += launches; h->solve_launches += launches;
    if (hbad != big)
        return fail(h, KB200_ESINGULAR, "leave-group-out: without group " + std::to_string(hbad) + " (lowest station " +
                    std::to_string(mem[goff[hbad]]) + ") the drift terms are not determined (singular drift block)");
    return KB200_OK;
}

extern "C" int kb200_knn_lgo(kb200_handle h, int k, const int32_t* group, int n_groups, double* z_out, double* ss_out) {
    int rc = check_knn(h, k); if (rc) return rc;
    if (!z_out || !ss_out) return fail(h, KB200_EBADARG, "null pointer");
    std::vector<int> sizes;
    rc = check_groups(h, group, n_groups, sizes); if (rc) return rc;
    const int gmax = (int)(std::max_element(sizes.begin(), sizes.end()) - sizes.begin());
    if (k > h->n - sizes[gmax])
        return fail(h, KB200_EBADARG, "leave-group-out: n_closest_points must be at most n - " + std::to_string(sizes[gmax]) +
                    " (the size of group " + std::to_string(gmax) + ")");
    const int nn = h->n;
    CU(h, h->wLgo.reserve((size_t)2 * nn * sizeof(int)));
    int* qg = h->wLgo.as<int>();
    int* sg = qg + nn;
    const int* sorig = reinterpret_cast<const int*>(h->kSorted.as<double>() + 4 * (size_t)nn);
    CU(h, cudaMemcpyAsync(qg, group, (size_t)nn * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CU(h, kbk_knn_sort_groups(nn, sorig, qg, sg, h->stream));
    h->launches += 1;
    return knn_to_host(h, k, station_queries(h), z_out, ss_out, 2, sg, qg);
}
