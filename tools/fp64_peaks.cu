// fp64_peaks.cu -- measured FP64 denominators for the S > 20 roofline (SURVEY.md section 6 / BASELINE.md section 2):
//   * register-resident DFMA chains (the CUDA-core fp64 pipe the 4-state kernels use)
//   * mma.sync.aligned.m8n8k4.f64 chains (SASS DMMA.8x8x4, the fp64 tensor path of k_walk_mma)
//   * a pure streaming write and a read+write copy (the HBM floor of the 4-state walk is its destination writes)
// Prints ONE JSON line.  Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peaks tools/fp64_peaks.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)

template <int ILP>
__global__ void __launch_bounds__(256) k_dfma(double* out, int iters, double a, double b) {
    double x[ILP];
#pragma unroll
    for (int i = 0; i < ILP; ++i) x[i] = a + threadIdx.x * 1e-9 + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ILP; ++i) x[i] = fma(x[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < ILP; ++i) s += x[i];
    if (s == 12345.678) out[blockIdx.x * blockDim.x + threadIdx.x] = s;      // never true: keeps the chain alive
}

template <int ILP>
__global__ void __launch_bounds__(256) k_dmma(double* out, int iters, double a, double b) {
    double d0[ILP], d1[ILP];
#pragma unroll
    for (int i = 0; i < ILP; ++i) { d0[i] = threadIdx.x * 1e-9 + i; d1[i] = -d0[i]; }
    const double fa = a + (threadIdx.x & 3) * 1e-6, fb = b + (threadIdx.x >> 2) * 1e-6;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ILP; ++i)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(d0[i]), "+d"(d1[i]) : "d"(fa), "d"(fb));
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < ILP; ++i) s += d0[i] + d1[i];
    if (s == 12345.678) out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// one 32-byte cell per thread as two 128-bit accesses (sm_90 has no 256-bit global access): what the walk kernels issue
__global__ void __launch_bounds__(256) k_fill(double4* dst, size_t n4, double v) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
        asm volatile("st.global.v2.f64 [%0], {%1,%1};\n\tst.global.v2.f64 [%0+16], {%1,%1};" :: "l"(dst + i), "d"(v) : "memory");
}

__global__ void __launch_bounds__(256) k_copy(double4* dst, const double4* src, size_t n4) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        double a, b, c, d;
        asm volatile("ld.global.v2.f64 {%0,%1}, [%4];\n\tld.global.v2.f64 {%2,%3}, [%4+16];"
                     : "=d"(a), "=d"(b), "=d"(c), "=d"(d) : "l"(src + i) : "memory");
        asm volatile("st.global.v2.f64 [%0], {%1,%2};\n\tst.global.v2.f64 [%0+16], {%3,%4};"
                     :: "l"(dst + i), "d"(a), "d"(b), "d"(c), "d"(d) : "memory");
    }
}

template <typename F>
static double best_ms(F launch, int reps) {
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    for (int w = 0; w < 3; ++w) launch();
    CK(cudaDeviceSynchronize());
    double best = 1e30;
    for (int r = 0; r < reps; ++r) {
        CK(cudaEventRecord(a));
        launch();
        CK(cudaEventRecord(b));
        CK(cudaEventSynchronize(b));
        float ms; CK(cudaEventElapsedTime(&ms, a, b));
        best = std::min(best, (double)ms);
    }
    CK(cudaGetLastError());
    return best;
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    double* out; CK(cudaMalloc(&out, sizeof(double) * 1024 * 1024));
    // ---- DFMA: 8 blocks x 256 threads per SM, 8 independent chains per thread
    const int iters = 20000;
    double dfma = 0.0, dmma = 0.0;
    int dfmaBlocks = 0, dmmaBlocks = 0;
    for (int per : {2, 4, 8}) {
        const int blocks = sms * per;
        const double ms = best_ms([&] { k_dfma<8><<<blocks, 256>>>(out, iters, 1.0000001, 1e-9); }, 5);
        const double tf = 2.0 * 8 * iters * (double)blocks * 256 / (ms * 1e-3) / 1e12;
        if (tf > dfma) { dfma = tf; dfmaBlocks = per; }
    }
    for (int per : {1, 2, 4, 8}) {
        const int blocks = sms * per;
        const double ms = best_ms([&] { k_dmma<8><<<blocks, 256>>>(out, iters, 1.0000001, 1e-9); }, 5);
        const double tf = 512.0 * 8 * iters * (double)blocks * 8 / (ms * 1e-3) / 1e12;     // 8 warps per block
        if (tf > dmma) { dmma = tf; dmmaBlocks = per; }
    }
    // ---- HBM: 4 GiB streams (far larger than the 126 MB L2)
    const size_t bytes = size_t(4) << 30, n4 = bytes / sizeof(double4);
    double4 *a, *b;
    CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes));
    CK(cudaMemset(a, 0, bytes)); CK(cudaMemset(b, 0, bytes));
    double msFill = 1e30, msCopy = 1e30;
    int fillBlocks = 0, copyBlocks = 0;
    for (int per : {4, 8, 16, 32, 64}) {
        const double f = best_ms([&] { k_fill<<<sms * per, 256>>>(a, n4, 1.0); }, 6);
        const double c = best_ms([&] { k_copy<<<sms * per, 256>>>(b, a, n4); }, 6);
        if (f < msFill) { msFill = f; fillBlocks = per; }
        if (c < msCopy) { msCopy = c; copyBlocks = per; }
    }
    int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("{\"gpu\": \"%s\", \"sms\": %d, \"sm_clock_attr_mhz\": %.0f, "
           "\"dfma_tflops\": %.2f, \"dfma_blocks_per_sm\": %d, \"dmma_m8n8k4_tflops\": %.2f, \"dmma_blocks_per_sm\": %d, "
           "\"write_gbs\": %.1f, \"write_blocks_per_sm\": %d, \"copy_gbs\": %.1f, \"copy_blocks_per_sm\": %d, "
           "\"how\": \"register-resident chains, 8 independent accumulators per thread, 20000 iterations, best of 5 (CUDA events); "
           "fill/copy of 4 GiB with 256-bit accesses, grid-stride, best of 6 over 4..64 blocks of 256 threads per SM; copy counts read+write bytes\"}\n",
           prop.name, sms, clk / 1000.0, dfma, dfmaBlocks, dmma, dmmaBlocks,
           bytes / (msFill * 1e-3) / 1e9, fillBlocks, 2.0 * bytes / (msCopy * 1e-3) / 1e9, copyBlocks);
    return 0;
}
