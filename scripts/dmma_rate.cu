// dmma_rate.cu — fp64 tensor-core (DMMA) throughput and fragment-map probe for sm_90a.
//
// Built by pykrige_b200/csrc/Makefile into scripts/libdmma_rate.so (not part of libkrige_b200.so); driven by
// scripts/dmma_rate.py and tests/test_dmma_fragments_gpu.py through three C entry points:
//   dmma_rate_run   steady-state rate of one mma.sync shape: one CTA per SM, 4 * warps_per_smsp warps, every warp
//                   issues DR_ACC independent MMAs per iteration (enough to cover the DMMA latency), per-CTA clock64
//                   cycles and the launch time by CUDA events;
//   dmma_stage_run  one phase-M stage of the fp64 solve kernel repeated for as long as asked (operands from shared
//                   memory, m16n8k4 or m16n8k16): scripts/dmma_rate.py --sustain samples power and clock around it;
//   dmma_frag_run   one MMA of one shape on one warp, D = A B + C with row-major A (M x K), B (K x 8), C / D (M x 8):
//                   the per-lane fragment maps below are exactly what the solve kernel assumes.
// Shapes: 0 = m8n8k4, 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16 (all .row.col.f64).
// Fragment maps (g = lane >> 2, t = lane & 3):
//   m8n8k4     a = A[g][t],  b = B[t][g],  c_i = C[g][2t + i]
//   m16n8kK    a_i = A[g + 8 (i & 1)][t + 4 (i >> 1)] (i < K/2),  b_i = B[t + 4 i][g] (i < K/4),
//              c_i = C[g + 8 (i >> 1)][2t + (i & 1)]
#include <cuda_runtime.h>
#include <stdint.h>

template <int SHAPE> struct Shape;
template <> struct Shape<0> { enum { M = 8, K = 4, NA = 1, NB = 1, NC = 2 }; };
template <> struct Shape<1> { enum { M = 16, K = 4, NA = 2, NB = 1, NC = 4 }; };
template <> struct Shape<2> { enum { M = 16, K = 8, NA = 4, NB = 2, NC = 4 }; };
template <> struct Shape<3> { enum { M = 16, K = 16, NA = 8, NB = 4, NC = 4 }; };

template <int SHAPE>
__device__ __forceinline__ void mma(double* c, const double* a, const double* b) {
    if (SHAPE == 0) {
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                     : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    } else if (SHAPE == 1) {
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    } else if (SHAPE == 2) {
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    }
}

#define DR_ACC 8

template <int SHAPE>
__global__ void __launch_bounds__(512, 1) rate_kernel(const double* __restrict__ in, int iters, double* __restrict__ out,
                                                      long long* __restrict__ cycles) {
    typedef Shape<SHAPE> S;
    const int lane = threadIdx.x & 31;
    double a[S::NA], b[S::NB], c[DR_ACC][S::NC];
#pragma unroll
    for (int i = 0; i < S::NA; ++i) a[i] = in[lane * 16 + i];
#pragma unroll
    for (int i = 0; i < S::NB; ++i) b[i] = in[lane * 16 + 8 + i];
#pragma unroll
    for (int j = 0; j < DR_ACC; ++j)
#pragma unroll
        for (int i = 0; i < S::NC; ++i) c[j][i] = 0.0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int j = 0; j < DR_ACC; ++j) mma<SHAPE>(c[j], a, b);
    }
    __syncthreads();
    const long long t1 = clock64();
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < DR_ACC; ++j)
#pragma unroll
        for (int i = 0; i < S::NC; ++i) s += c[j][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int SHAPE>
__global__ void frag_kernel(const double* __restrict__ A, const double* __restrict__ B, const double* __restrict__ C,
                            double* __restrict__ D) {
    typedef Shape<SHAPE> S;
    const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    double a[S::NA], b[S::NB], c[S::NC];
    if (SHAPE == 0) {
        a[0] = A[g * S::K + t];
        b[0] = B[t * 8 + g];
        c[0] = C[g * 8 + 2 * t];
        c[1] = C[g * 8 + 2 * t + 1];
    } else {
#pragma unroll
        for (int i = 0; i < S::NA; ++i) a[i] = A[(g + 8 * (i & 1)) * S::K + t + 4 * (i >> 1)];
#pragma unroll
        for (int i = 0; i < S::NB; ++i) b[i] = B[(t + 4 * i) * 8 + g];
#pragma unroll
        for (int i = 0; i < S::NC; ++i) c[i] = C[(g + 8 * (i >> 1)) * 8 + 2 * t + (i & 1)];
    }
    mma<SHAPE>(c, a, b);
    if (SHAPE == 0) {
        D[g * 8 + 2 * t] = c[0];
        D[g * 8 + 2 * t + 1] = c[1];
    } else {
#pragma unroll
        for (int i = 0; i < S::NC; ++i) D[(g + 8 * (i >> 1)) * 8 + 2 * t + (i & 1)] = c[i];
    }
}

// One 16-deep stage of the fp64 solve kernel's phase M, repeated: 8 warps per CTA (2 per SM sub-partition, as the
// consumer warpgroups), each multiplying the A fragments of two 16-row m-tiles by the B fragments of 8 n-tiles, all read
// from shared memory in the solve kernel's tile orders. K = 4: four m16n8k4 per (m-tile, n-tile) per stage, K = 16: one
// m16n8k16. The stage index cycles over ST_STAGES buffers so that the loads cannot be hoisted out of the loop.
#define ST_STAGES 4
template <int K>
__global__ void __launch_bounds__(256, 1) stage_kernel(long long iters, double* __restrict__ out) {
    __shared__ double2 ta[ST_STAGES][2 * 4 * 32];      // [stage][m-tile][k4][lane]: a[2 k4], a[2 k4 + 1]
    __shared__ double tb[ST_STAGES][4 * 8 * 32];       // [stage][k4][n-tile][lane]: b[k4]
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < ST_STAGES * 2 * 4 * 32; i += blockDim.x)
        (&ta[0][0])[i] = make_double2(1e-3 * ((i % 7) + 1), 1e-3 * ((i % 5) + 1));
    for (int i = threadIdx.x; i < ST_STAGES * 4 * 8 * 32; i += blockDim.x) (&tb[0][0])[i] = 1e-3 * ((i % 3) + 1);
    __syncthreads();
    double acc[2][8][4];
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[q][nt][i] = 0.0;
    for (long long it = 0; it < iters; ++it) {
        const int s = (int)(it % ST_STAGES);
        double fa[2][8];
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
                const double2 v = ta[s][(q * 4 + k4) * 32 + lane];
                fa[q][2 * k4] = v.x; fa[q][2 * k4 + 1] = v.y;
            }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            double fb[4];
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) fb[k4] = tb[s][(k4 * 8 + nt) * 32 + lane];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (K == 16) {
                    mma<3>(acc[q][nt], fa[q], fb);
                } else {
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4) mma<1>(acc[q][nt], &fa[q][2 * k4], &fb[k4]);
                }
            }
        }
    }
    double r = 0.0;
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) r += acc[q][nt][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = r;
}

static const int kM[4] = {8, 16, 16, 16};
static const int kK[4] = {4, 4, 8, 16};

extern "C" {

// FMAs one warp-wide MMA of the shape performs
long long dmma_shape_fmas(int shape) {
    if (shape < 0 || shape > 3) return -1;
    return (long long)kM[shape] * 8 * kK[shape];
}

// Runs the rate kernel of `shape` once on every SM with 4 * warps_per_smsp warps per CTA, `iters` iterations of DR_ACC
// MMAs per warp. Returns cudaError_t; *ms = launch time (CUDA events), cycles[sm] = clock64 cycles of each CTA,
// *fmas_per_cta = FMAs one CTA performed.
int dmma_rate_run(int shape, int warps_per_smsp, int iters, float* ms, long long* cycles, int* sms,
                  long long* fmas_per_cta) {
    if (shape < 0 || shape > 3 || warps_per_smsp < 1 || warps_per_smsp > 4) return (int)cudaErrorInvalidValue;
    int dev = 0, nsm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    const int threads = 128 * warps_per_smsp;
    double *in = nullptr, *out = nullptr;
    long long* cyc = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    double hin[32 * 16];
    for (int i = 0; i < 32 * 16; ++i) hin[i] = 1e-3 * (double)((i % 7) + 1);
    if ((e = cudaMalloc(&in, sizeof(hin))) != cudaSuccess) goto done;
    if ((e = cudaMalloc(&out, sizeof(double) * nsm * threads)) != cudaSuccess) goto done;
    if ((e = cudaMalloc(&cyc, sizeof(long long) * nsm)) != cudaSuccess) goto done;
    if ((e = cudaMemcpy(in, hin, sizeof(hin), cudaMemcpyHostToDevice)) != cudaSuccess) goto done;
    if ((e = cudaEventCreate(&e0)) != cudaSuccess) goto done;
    if ((e = cudaEventCreate(&e1)) != cudaSuccess) goto done;
    cudaEventRecord(e0);
    switch (shape) {
        case 0: rate_kernel<0><<<nsm, threads>>>(in, iters, out, cyc); break;
        case 1: rate_kernel<1><<<nsm, threads>>>(in, iters, out, cyc); break;
        case 2: rate_kernel<2><<<nsm, threads>>>(in, iters, out, cyc); break;
        default: rate_kernel<3><<<nsm, threads>>>(in, iters, out, cyc); break;
    }
    cudaEventRecord(e1);
    if ((e = cudaGetLastError()) != cudaSuccess) goto done;
    if ((e = cudaEventSynchronize(e1)) != cudaSuccess) goto done;
    cudaEventElapsedTime(ms, e0, e1);
    e = cudaMemcpy(cycles, cyc, sizeof(long long) * nsm, cudaMemcpyDeviceToHost);
    *sms = nsm;
    *fmas_per_cta = (long long)iters * DR_ACC * (threads / 32) * dmma_shape_fmas(shape);
done:
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    cudaFree(in);
    cudaFree(out);
    cudaFree(cyc);
    return (int)e;
}

// Runs stage_kernel<k> (k = 4 or 16) once on every SM for `iters` stages per warp. Returns cudaError_t; *ms = launch
// time (CUDA events), *fmas = FMAs of the whole launch. Blocks until the kernel ends (ctypes releases the GIL, so a
// Python thread can sample NVML meanwhile).
int dmma_stage_run(int k, long long iters, float* ms, long long* fmas) {
    if ((k != 4 && k != 16) || iters < 1) return (int)cudaErrorInvalidValue;
    int dev = 0, nsm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    double* out = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if ((e = cudaMalloc(&out, sizeof(double) * nsm * 256)) != cudaSuccess) goto done;
    if ((e = cudaEventCreate(&e0)) != cudaSuccess) goto done;
    if ((e = cudaEventCreate(&e1)) != cudaSuccess) goto done;
    cudaEventRecord(e0);
    if (k == 16) stage_kernel<16><<<nsm, 256>>>(iters, out);
    else stage_kernel<4><<<nsm, 256>>>(iters, out);
    cudaEventRecord(e1);
    if ((e = cudaGetLastError()) != cudaSuccess) goto done;
    if ((e = cudaEventSynchronize(e1)) != cudaSuccess) goto done;
    cudaEventElapsedTime(ms, e0, e1);
    *fmas = iters * (long long)nsm * 8 * (2 * 8 * 16 * 8 * 16);     // warps x (2 m-tiles x 8 n-tiles x 16x8x16)
done:
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    cudaFree(out);
    return (int)e;
}

// D = A B + C by one MMA of `shape` (host arrays, row-major: A M x K, B K x 8, C and D M x 8). Returns cudaError_t.
int dmma_frag_run(int shape, const double* A, const double* B, const double* C, double* D) {
    if (shape < 0 || shape > 3) return (int)cudaErrorInvalidValue;
    const size_t na = (size_t)kM[shape] * kK[shape], nb = (size_t)kK[shape] * 8, nc = (size_t)kM[shape] * 8;
    double *dA = nullptr, *dB = nullptr, *dC = nullptr, *dD = nullptr;
    cudaError_t e;
    if ((e = cudaMalloc(&dA, na * 8)) != cudaSuccess) goto done;
    if ((e = cudaMalloc(&dB, nb * 8)) != cudaSuccess) goto done;
    if ((e = cudaMalloc(&dC, nc * 8)) != cudaSuccess) goto done;
    if ((e = cudaMalloc(&dD, nc * 8)) != cudaSuccess) goto done;
    if ((e = cudaMemcpy(dA, A, na * 8, cudaMemcpyHostToDevice)) != cudaSuccess) goto done;
    if ((e = cudaMemcpy(dB, B, nb * 8, cudaMemcpyHostToDevice)) != cudaSuccess) goto done;
    if ((e = cudaMemcpy(dC, C, nc * 8, cudaMemcpyHostToDevice)) != cudaSuccess) goto done;
    switch (shape) {
        case 0: frag_kernel<0><<<1, 32>>>(dA, dB, dC, dD); break;
        case 1: frag_kernel<1><<<1, 32>>>(dA, dB, dC, dD); break;
        case 2: frag_kernel<2><<<1, 32>>>(dA, dB, dC, dD); break;
        default: frag_kernel<3><<<1, 32>>>(dA, dB, dC, dD); break;
    }
    if ((e = cudaGetLastError()) != cudaSuccess) goto done;
    e = cudaMemcpy(D, dD, nc * 8, cudaMemcpyDeviceToHost);
done:
    cudaFree(dA);
    cudaFree(dB);
    cudaFree(dC);
    cudaFree(dD);
    return (int)e;
}

}  // extern "C"
