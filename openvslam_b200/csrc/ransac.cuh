// ransac.cuh -- the building blocks of the batched RANSAC solvers: Sim3 and PnP (optimize.cu) and the essential, homography and
// fundamental-matrix solvers (two_view_ransac.cu).  Device: the warp-per-hypothesis inlier count and lane-order score, the
// best-hypothesis key and the CTA-wide index-order compaction.  Host: the offsets check and the staging of a solve's buffers.
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

// Buffers carved one after another from a byte arena, each aligned to 256 bytes.  With a null base the carve only counts:
// `off` is then the size the arena needs.
struct Arena {
    uint8_t* base; size_t off;
    template <typename T> T* take(size_t n) {
        off = (off + 255) / 256 * 256;
        T* p = reinterpret_cast<T*>(base + off);
        off += n * sizeof(T);
        return p;
    }
};

// The buffers of one batched solve, carved from a pinned host arena and a device arena together.  Each input and output is
// named once and gets the same offset in both arenas, so the inputs go up in one copy and the outputs come back in another.
// Carve the inputs first, then the outputs, then the device-only scratch: `ordered` turns false when a take breaks that order
// (an input after an output would move the end of the inputs past outputs, and the copy back would miss them).
struct Staging {
    Arena h{nullptr, 0}, d{nullptr, 0};
    size_t in_end = 0;                               // bytes of the inputs
    int phase = 0;                                   // 0 inputs, 1 outputs, 2 device scratch
    bool ordered = true;
    template <typename T> T* in(T*& host, size_t n) {
        ordered = ordered && phase == 0;
        host = h.take<T>(n);
        in_end = h.off;
        return d.take<T>(n);
    }
    template <typename T> T* out(T*& host, size_t n) {
        ordered = ordered && phase <= 1;
        phase = 1;
        host = h.take<T>(n);
        return d.take<T>(n);
    }
    template <typename T> T* dev(size_t n) {
        phase = 2;
        return d.take<T>(n);
    }
    size_t out_begin() const { return (in_end + 255) / 256 * 256; }
    cudaError_t upload(cudaStream_t st) const { return cudaMemcpyAsync(d.base, h.base, in_end, cudaMemcpyHostToDevice, st); }
    cudaError_t download(cudaStream_t st) const {
        const size_t b = out_begin();
        return cudaMemcpyAsync(h.base + b, d.base + b, h.off - b, cudaMemcpyDeviceToHost, st);
    }
};

// Sizes the arenas by running carve(S) on null bases, has grow(host_bytes, device_bytes) make room (it may move hbase and
// dbase), then carves them for real into S.  A carve out of order is refused before anything is allocated.
template <class Grow, class Carve>
int stage(Staging& S, uint8_t*& hbase, uint8_t*& dbase, Grow grow, Carve carve) {
    S = Staging{};
    carve(S);
    OVS_REQUIRE(S.ordered, OVS_ERR_UNSUPPORTED, "staging carved out of order (inputs, then outputs, then device scratch)");
    const int rc = grow(S.h.off, S.d.off);
    if (rc != OVS_OK) return rc;
    S = Staging{{hbase, 0}, {dbase, 0}};
    carve(S);
    return OVS_OK;
}

}  // namespace ovs
