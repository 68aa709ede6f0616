// probe.cu -- measured FP64 peaks of the device the library runs on: the whole-chip issue rate of independent
// mma.sync.m8n8k4.f64 (DMMA) and of independent DFMA.  bench.py reports the Cholesky / Schur rooflines against the DMMA
// figure measured in the same run.
#include "ovs_common.h"

namespace {

__device__ __forceinline__ void probe_dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// 8 independent accumulators per warp, `iters` rounds: 8 x iters DMMAs of 256 FMA each per warp
__global__ void __launch_bounds__(256) k_probe_dmma(double* out, int iters, double seed) {
    double e[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) { e[j][0] = seed + j + threadIdx.x; e[j][1] = seed * 0.5; }
    const double a = 1.0000001, b = 0.25 + seed * 1e-9;
    for (int i = 0; i < iters; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) probe_dmma(e[j][0], e[j][1], a, b);
    double s = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += e[j][0] + e[j][1];
    if (s == 12345.678) out[blockIdx.x * 256 + threadIdx.x] = s;   // keeps the chain alive, never true
}

// 8 independent DFMA chains per thread
__global__ void __launch_bounds__(256) k_probe_dfma(double* out, int iters, double seed) {
    double c[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) c[j] = seed + j + threadIdx.x;
    const double m = 1.0000001, y = seed * 1e-9;
    for (int i = 0; i < iters; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) c[j] = fma(c[j], m, y);
    double s = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += c[j];
    if (s == 12345.678) out[blockIdx.x * 256 + threadIdx.x] = s;
}

}  // namespace

extern "C" int ovs_probe_fp64_peaks(int device, double* dmma_tflops, double* dfma_tflops) {
    OVS_REQUIRE(dmma_tflops && dfma_tflops, OVS_ERR_INVALID_ARG, "null argument");
    int rc = ovs::select_device(device);
    if (rc != OVS_OK) return rc;
    cudaDeviceProp prop;
    OVS_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    const int blocks = prop.multiProcessorCount * 4;       // 32 warps per SM
    const int iters = 4096;
    double* d_out = nullptr;
    OVS_CUDA_CHECK(cudaMalloc(&d_out, (size_t)blocks * 256 * sizeof(double)));
    cudaEvent_t e0, e1;
    OVS_CUDA_CHECK(cudaEventCreate(&e0)); OVS_CUDA_CHECK(cudaEventCreate(&e1));
    double best[2] = {0, 0};
    for (int which = 0; which < 2; ++which) {
        for (int rep = 0; rep < 4; ++rep) {
            OVS_CUDA_CHECK(cudaEventRecord(e0, 0));
            if (which == 0) k_probe_dmma<<<blocks, 256>>>(d_out, iters, 1.25);
            else k_probe_dfma<<<blocks, 256>>>(d_out, iters, 1.25);
            OVS_LAUNCH_CHECK();
            OVS_CUDA_CHECK(cudaEventRecord(e1, 0));
            OVS_CUDA_CHECK(cudaEventSynchronize(e1));
            float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
            // DMMA: 8 warps x 8 x iters x 256 FMA per block; DFMA: 256 threads x 8 x iters FMA per block
            const double fma = (which == 0) ? (double)blocks * 8 * 8.0 * iters * 256.0 : (double)blocks * 256 * 8.0 * iters;
            const double tf = 2.0 * fma / (ms * 1e-3) / 1e12;
            if (rep > 0 && tf > best[which]) best[which] = tf;     // first launch is the warm-up
        }
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d_out);
    *dmma_tflops = best[0]; *dfma_tflops = best[1];
    return OVS_OK;
}
