// dmma_shapes.cu - issue rate of the fp64 mma.sync shapes on one GPU (standalone, not part of the library).
//
// One register-only kernel per shape: m8n8k4 (the sm_80 shape) and m16n8k4 / m16n8k8 / m16n8k16 (added by sm_90).
// Every SM runs one CTA of 16 warps (four per sub-partition, as predict_acq16_kernel), every warp keeps
// kChains independent accumulator chains, so the MMA latency is covered and only the issue rate of the
// tensor pipe is left.  Each CTA reads its SM's clock (clock64) around the loop; the kernel time comes
// from CUDA events.  Prints one JSON line per shape:
//   flop_per_clk_sm  flop of one CTA / SM cycles of that CTA (median over CTAs): independent of the clock
//   tflops           all flop / event time;  sm_mhz = median cycles / event time (the clock during the run)
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_shapes dmma_shapes.cu
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e_ = (x);                                                          \
        if (e_ != cudaSuccess) {                                                       \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); \
            exit(1);                                                                   \
        }                                                                              \
    } while (0)

constexpr int kThreads = 512;  // 16 warps
constexpr int kChains = 8;     // independent accumulators per warp
constexpr int kSmemBytes = 160 * 1024;  // only to keep a second CTA off the SM

// per shape: M, N, K and the fp64 registers of the A, B and C fragments per thread
template <int S> struct Shape;
template <> struct Shape<0> { static constexpr int M = 8, N = 8, K = 4, NA = 1, NB = 1, NC = 2; };
template <> struct Shape<1> { static constexpr int M = 16, N = 8, K = 4, NA = 2, NB = 1, NC = 4; };
template <> struct Shape<2> { static constexpr int M = 16, N = 8, K = 8, NA = 4, NB = 2, NC = 4; };
template <> struct Shape<3> { static constexpr int M = 16, N = 8, K = 16, NA = 8, NB = 4, NC = 4; };
static const char* kNames[4] = {"m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16"};

template <int S> __device__ __forceinline__ void mma(double* c, const double* a, const double* b);
template <> __device__ __forceinline__ void mma<0>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c[0]), "+d"(c[1])
                 : "d"(a[0]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<1>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<2>(double* c, const double* a, const double* b) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
template <> __device__ __forceinline__ void mma<3>(double* c, const double* a, const double* b) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
          "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <int S>
__global__ void __launch_bounds__(kThreads, 1) shape_kernel(const double* in, double* out, long long* cycles,
                                                            int* smid, int iters) {
    using T = Shape<S>;
    const int lane = threadIdx.x & 31;
    double a[T::NA], b[T::NB], c[kChains][T::NC];
#pragma unroll
    for (int i = 0; i < T::NA; ++i) a[i] = in[(lane + i) & 63];
#pragma unroll
    for (int i = 0; i < T::NB; ++i) b[i] = in[(lane + 7 * i + 3) & 63];
#pragma unroll
    for (int ch = 0; ch < kChains; ++ch)
#pragma unroll
        for (int i = 0; i < T::NC; ++i) c[ch][i] = 0.0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int ch = 0; ch < kChains; ++ch) mma<S>(c[ch], a, b);
    }
    __syncthreads();
    const long long t1 = clock64();
    double s = 0.0;
#pragma unroll
    for (int ch = 0; ch < kChains; ++ch)
#pragma unroll
        for (int i = 0; i < T::NC; ++i) s += c[ch][i];
    out[blockIdx.x * kThreads + threadIdx.x] = s;
    if (threadIdx.x == 0) {
        cycles[blockIdx.x] = t1 - t0;
        unsigned id;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
        smid[blockIdx.x] = (int)id;
    }
}

template <int S>
static void run(int nsm, const double* d_in, double* d_out, long long* d_cyc, int* d_smid) {
    using T = Shape<S>;
    // the same flop per CTA for every shape: 2^17 m8n8k4 steps of every chain (~50 ms at 1.5 GHz, 128 flop/clk/SM)
    const int iters = (1 << 17) / ((T::M * T::N * T::K) / 256);
    CK(cudaFuncSetAttribute(shape_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    shape_kernel<S><<<nsm, kThreads, kSmemBytes>>>(d_in, d_out, d_cyc, d_smid, iters / 8);  // warm-up
    CK(cudaGetLastError());
    CK(cudaEventRecord(e0));
    shape_kernel<S><<<nsm, kThreads, kSmemBytes>>>(d_in, d_out, d_cyc, d_smid, iters);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    std::vector<long long> cyc(nsm);
    std::vector<int> sm(nsm);
    CK(cudaMemcpy(cyc.data(), d_cyc, sizeof(long long) * nsm, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(sm.data(), d_smid, sizeof(int) * nsm, cudaMemcpyDeviceToHost));
    std::sort(cyc.begin(), cyc.end());
    std::sort(sm.begin(), sm.end());
    const int distinct = (int)(std::unique(sm.begin(), sm.end()) - sm.begin());
    const double flop_cta = (double)(kThreads / 32) * kChains * iters * 2.0 * T::M * T::N * T::K;
    const double med = (double)cyc[nsm / 2];
    printf("{\"shape\": \"%s\", \"flop_per_clk_sm\": %.2f, \"tflops\": %.3f, \"sm_mhz\": %.0f, \"ms\": %.3f, "
           "\"cycles_min\": %lld, \"cycles_max\": %lld, \"ctas\": %d, \"distinct_sms\": %d}\n",
           kNames[S], flop_cta / med, flop_cta * nsm / (ms * 1e-3) / 1e12, med / (ms * 1e-3) / 1e6, ms, cyc.front(),
           cyc.back(), nsm, distinct);
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int nsm = prop.multiProcessorCount;
    std::vector<double> h(64);
    for (int i = 0; i < 64; ++i) h[i] = 1e-3 * (1 + (i % 7));
    double *d_in, *d_out;
    long long* d_cyc;
    int* d_smid;
    CK(cudaMalloc(&d_in, 64 * sizeof(double)));
    CK(cudaMalloc(&d_out, (size_t)nsm * kThreads * sizeof(double)));
    CK(cudaMalloc(&d_cyc, nsm * sizeof(long long)));
    CK(cudaMalloc(&d_smid, nsm * sizeof(int)));
    CK(cudaMemcpy(d_in, h.data(), 64 * sizeof(double), cudaMemcpyHostToDevice));
    printf("{\"device\": \"%s\", \"sms\": %d}\n", prop.name, nsm);
    for (int rep = 0; rep < 2; ++rep) {  // two passes: the spread between them is the noise
        run<0>(nsm, d_in, d_out, d_cyc, d_smid);
        run<1>(nsm, d_in, d_out, d_cyc, d_smid);
        run<2>(nsm, d_in, d_out, d_cyc, d_smid);
        run<3>(nsm, d_in, d_out, d_cyc, d_smid);
    }
    CK(cudaFree(d_in));
    CK(cudaFree(d_out));
    CK(cudaFree(d_cyc));
    CK(cudaFree(d_smid));
    return 0;
}
