// block_sum.cuh -- the CTA-wide form of pnp_sum (pnp_math.cuh), shared by the solvers whose recompute kernels sum over every
// inlier of a problem with one 256-thread CTA: the PnP solver's EPnP (optimize.cu, k_pnp_refine) and the essential, homography
// and fundamental-matrix solvers' A^T A (two_view_ransac.cu, k_two_view_refine).  Device only.
#pragma once
#include "pnp_math.cuh"

namespace ovs {

constexpr int kBlockSumThreads = kPnpSumSlots;       // one thread per partial sum
constexpr int kBlockSumChunk = 8;                    // components reduced per pass

#if defined(__CUDACC__)
// pnp_sum across the CTA: thread t forms partial s_t over the points t, t + 256, ..; then, kBlockSumChunk components at a time,
// thread c adds the 256 partials of component c in order.  Same bits as PnpSeqSum.
struct PnpBlockSum {
    int n;
    double* red;                                     // shared, kBlockSumChunk x 256
    double* res;                                     // shared, K (78 for EPnP)
    template <int K, class F> __device__ void run(F f, double* out) const {
        const int t = threadIdx.x;
        double s[K], v[K];
        for (int c = 0; c < K; ++c) s[c] = 0.0;
        for (int i = t; i < n; i += kBlockSumThreads) {
            f(i, v);
            for (int c = 0; c < K; ++c) s[c] += v[c];
        }
#pragma unroll
        for (int c0 = 0; c0 < K; c0 += kBlockSumChunk) {
#pragma unroll
            for (int c = c0; c < c0 + kBlockSumChunk && c < K; ++c) red[(c - c0) * kBlockSumThreads + t] = s[c];
            __syncthreads();
            if (t < kBlockSumChunk && c0 + t < K) {
                double acc = 0.0;
                for (int u = 0; u < kBlockSumThreads; ++u) acc += red[t * kBlockSumThreads + u];
                res[c0 + t] = acc;
            }
            __syncthreads();
        }
        for (int c = 0; c < K; ++c) out[c] = res[c];
        __syncthreads();
    }
};
#endif

}  // namespace ovs
