// ransac.cuh -- the building blocks of the batched RANSAC solvers: Sim3 and PnP (optimize.cu) and the essential, homography and
// fundamental-matrix solvers (two_view_ransac.cu).  Device: the warp-per-hypothesis inlier count and lane-order score, the
// best-hypothesis key and the CTA-wide index-order compaction.  Host: the offsets check (a solve's buffers are staged through
// staging.h).
#pragma once
#include <cstddef>
#include <cstdint>

#include "ovs_common.h"

namespace ovs {

// ------------------------------------------------------------------------------------------------------------------ device
// One warp over a problem's n items, lane l taking items l, l + 32, ..: the number of items i for which in(i) holds (every lane).
template <class In>
__device__ __forceinline__ unsigned warp_count(int n, int lane, In in) {
    unsigned cnt = 0;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool f = i < n && in(i);
        cnt += __popc(__ballot_sync(0xffffffffu, f));
    }
    return cnt;
}

// check_inliers by one warp: check(i, part) tests item i and adds its terms to the lane's partial score.  Returns the inlier
// count and the 32 partials added in lane order (every lane): the same bits as essential_score_seq / two_view_score_seq.
template <class Check>
__device__ __forceinline__ int warp_score(int n, int lane, Check check, double* score) {
    double part = 0.0;
    const int cnt = (int)warp_count(n, lane, [&](int i) { return check(i, part); });
    double total = 0.0;
    for (int l = 0; l < 32; ++l) total += __shfl_sync(0xffffffffu, part, l);
    *score = total;
    return cnt;
}

// The best hypothesis as one integer: the maximum of (count << 32) | ~k over a problem's hypotheses (atomicMax, so the order
// of the warps does not matter) is the first of the hypotheses with the most inliers, as in the sequential loop.  A problem's
// key starts at 0, so a hypothesis with no inlier is never best.
__device__ __forceinline__ unsigned long long best_key(unsigned cnt, int k) {
    return ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)k);
}
// The count and the hypothesis of a key; -1 when no hypothesis had an inlier.
__device__ __forceinline__ int best_of_key(unsigned long long key, unsigned* cnt) {
    *cnt = (unsigned)(key >> 32);
    return *cnt > 0 ? (int)(~(unsigned)(key & 0xffffffffull)) : -1;
}

// The items i < n for which keep(i) holds, written in index order to cidx[0 ..) by a CTA of Threads threads (every thread
// calls it).  s_warp: shared, one int per warp.
template <int Threads, class Keep>
__device__ __forceinline__ void cta_compact(int n, int* cidx, int* s_warp, Keep keep) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int running = 0;
    for (int base = 0; base < n; base += Threads) {
        const int i = base + t;
        const bool f = i < n && keep(i);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = running;
        for (int w = 0; w < warp; ++w) before += s_warp[w];
        if (f) cidx[before + __popc(bal & ((1u << lane) - 1u))] = i;
        for (int w = 0; w < Threads / 32; ++w) running += s_warp[w];
        __syncthreads();
    }
    __syncthreads();
}

// -------------------------------------------------------------------------------------------------------------------- host
// B + 1 offsets of a batch: off[0] == 0 and non-decreasing.
inline int check_offsets(const int32_t* off, int B, const char* what) {
    OVS_REQUIRE(off[0] == 0, OVS_ERR_INVALID_ARG, "%s[0] must be 0", what);
    for (int b = 0; b < B; ++b)
        OVS_REQUIRE(off[b + 1] >= off[b], OVS_ERR_INVALID_ARG, "%s must be non-decreasing (problem %d)", what, b);
    return OVS_OK;
}

}  // namespace ovs
