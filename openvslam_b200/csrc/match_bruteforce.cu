// match_bruteforce.cu -- 256-bit Hamming brute force for openvslam::match::robust
// (match/robust.{h,cc}: robust::brute_force_match, called by robust::match_frame_and_keyframe;
// distance = match::compute_descriptor_distance_32, match/base.h; names as in SURVEY.md 8a).
//
// k_hamming_topk    every query descriptor against a chunk of train descriptors staged in
//                   shared memory (broadcast 128-bit reads); each thread keeps its query in 8
//                   registers and a sorted top-8 of (distance << 16 | train index) keys.
//                   Grid = query blocks x train chunks so that 4000 x 4000 fills the 132 SMs of an H100.
// k_topk_merge      merges the per-chunk top-8 lists of a query.
//
// A sorted (distance, index) top-8 is what the reference's sequential `<` scan needs: best =
// lowest index among the minimum distances, second best = next key.  robust::brute_force_match
// also removes already-matched frame keypoints from later scans (a sequential dependency); the
// host replays that greedy rule on the top-8 lists (greedy_replay.h) and re-queries the GPU (with an
// exclusion bitmask) only when a list cannot decide -- see ovs_robust_brute_force_match_host.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "greedy_replay.h"
#include "match_common.h"

namespace {

constexpr int kTopK = OVS_MATCH_TOPK;   // 8
constexpr int kQueriesPerBlock = 128;
constexpr int kTrainTile = 128;  // descriptors staged per shared-memory tile (4 KB)

// 256-bit Hamming distance with FOUR population counts instead of eight: the eight 32-bit difference words go through a
// carry-save adder tree (bitwise full adders: sum = a ^ b ^ c, carry = majority(a, b, c), one LOP3 each), which leaves four words
// holding the bit counts' ones, twos, fours and eights; distance = popc(ones) + 2 popc(twos) + 4 popc(fours) + 8 popc(eights).
// POPC issues at a quarter of the integer ALU rate on sm_90, so it -- not the logic -- bounds a brute-force Hamming kernel
// (Harley-Seal, restricted to one descriptor pair so the result is exactly match::compute_descriptor_distance_32's).
__device__ __forceinline__ int hamming256(const uint4& qa, const uint4& qb, const uint4& ta, const uint4& tb) {
    const unsigned x0 = qa.x ^ ta.x, x1 = qa.y ^ ta.y, x2 = qa.z ^ ta.z, x3 = qa.w ^ ta.w;
    const unsigned x4 = qb.x ^ tb.x, x5 = qb.y ^ tb.y, x6 = qb.z ^ tb.z, x7 = qb.w ^ tb.w;
    const unsigned s0 = x0 ^ x1 ^ x2, c0 = (x0 & x1) | (x2 & (x0 ^ x1));
    const unsigned s1 = x3 ^ x4 ^ x5, c1 = (x3 & x4) | (x5 & (x3 ^ x4));
    const unsigned s2 = s0 ^ s1 ^ x6, c2 = (s0 & s1) | (x6 & (s0 ^ s1));
    const unsigned ones = s2 ^ x7, c3 = s2 & x7;
    const unsigned t0 = c0 ^ c1 ^ c2, f0 = (c0 & c1) | (c2 & (c0 ^ c1));
    const unsigned twos = t0 ^ c3, f1 = t0 & c3;
    const unsigned fours = f0 ^ f1, eights = f0 & f1;
    return __popc(ones) + 2 * __popc(twos) + 4 * __popc(fours) + 8 * __popc(eights);
}

__device__ __forceinline__ void topk_insert(unsigned (&k)[kTopK], unsigned key) {
    if (key < k[kTopK - 1]) {
        k[kTopK - 1] = key;
#pragma unroll
        for (int i = kTopK - 1; i > 0; --i)
            if (k[i] < k[i - 1]) { const unsigned t = k[i - 1]; k[i - 1] = k[i]; k[i] = t; }
    }
}

// desc_q [nq][32 B], desc_t [nt][32 B] (16-byte aligned).  Train chunk c covers
// [c * chunk, min(nt, (c+1) * chunk)).  out[(q * nchunks + c) * 8 + k].
__global__ void __launch_bounds__(kQueriesPerBlock) k_hamming_topk(const uint4* __restrict__ desc_q, int nq,
                                                                   const uint4* __restrict__ desc_t, int nt, int chunk,
                                                                   unsigned* __restrict__ out) {
    __shared__ uint4 tile[kTrainTile * 2];
    const int q = blockIdx.x * kQueriesPerBlock + threadIdx.x;
    const int c = blockIdx.y, nchunks = gridDim.y;
    const int t_begin = c * chunk, t_end = min(nt, t_begin + chunk);
    uint4 qa = make_uint4(0, 0, 0, 0), qb = qa;
    if (q < nq) { qa = __ldg(desc_q + 2 * (size_t)q); qb = __ldg(desc_q + 2 * (size_t)q + 1); }
    unsigned best[kTopK];
#pragma unroll
    for (int k = 0; k < kTopK; ++k) best[k] = 0xffffffffu;

    for (int t0 = t_begin; t0 < t_end; t0 += kTrainTile) {
        const int n = min(kTrainTile, t_end - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * n; i += kQueriesPerBlock) tile[i] = __ldg(desc_t + 2 * (size_t)t0 + i);
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < n; ++j) {
            const uint4 ta = tile[2 * j], tb = tile[2 * j + 1];
            const int d = hamming256(qa, qb, ta, tb);
            topk_insert(best, ((unsigned)d << 16) | (unsigned)(t0 + j));
        }
    }
    if (q < nq) {
        unsigned* o = out + ((size_t)q * nchunks + c) * kTopK;
#pragma unroll
        for (int k = 0; k < kTopK; ++k) o[k] = best[k];
    }
}

__global__ void __launch_bounds__(128) k_topk_merge(const unsigned* __restrict__ part, int nq, int nchunks,
                                                     unsigned* __restrict__ out) {
    const int q = blockIdx.x * 128 + threadIdx.x;
    if (q >= nq) return;
    unsigned best[kTopK];
#pragma unroll
    for (int k = 0; k < kTopK; ++k) best[k] = 0xffffffffu;
    const unsigned* p = part + (size_t)q * nchunks * kTopK;
    for (int i = 0; i < nchunks * kTopK; ++i) topk_insert(best, p[i]);
#pragma unroll
    for (int k = 0; k < kTopK; ++k) out[(size_t)q * kTopK + k] = best[k];
}

// Re-query of ONE descriptor against the train set with an exclusion mask (the greedy replay asks for it when a candidate list
// is used up): the train descriptors are spread over the 256 threads of one block, every thread keeps the sorted top-8 of
// its share, and eight rounds of block-wide minimum pick the overall top-8 in (distance, index) order.
__global__ void __launch_bounds__(256) k_hamming_one(const uint4* __restrict__ desc_q, const uint4* __restrict__ desc_t, int nt,
                                                      const unsigned* __restrict__ exclude, unsigned* __restrict__ out) {
    __shared__ unsigned wmin[8];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint4 qa = __ldg(desc_q), qb = __ldg(desc_q + 1);
    unsigned best[kTopK];
#pragma unroll
    for (int k = 0; k < kTopK; ++k) best[k] = 0xffffffffu;
    for (int j = tid; j < nt; j += 256) {
        if (exclude[j >> 5] & (1u << (j & 31))) continue;
        const uint4 ta = __ldg(desc_t + 2 * (size_t)j), tb = __ldg(desc_t + 2 * (size_t)j + 1);
        const int d = hamming256(qa, qb, ta, tb);
        topk_insert(best, ((unsigned)d << 16) | (unsigned)j);
    }
    for (int r = 0; r < kTopK; ++r) {
        const unsigned m = __reduce_min_sync(0xffffffffu, best[0]);
        if (lane == 0) wmin[wid] = m;
        __syncthreads();
        unsigned g = wmin[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) g = min(g, wmin[w]);
        if (g != 0xffffffffu && best[0] == g) {        // keys are unique (they carry the index): exactly one owner pops
#pragma unroll
            for (int k = 0; k + 1 < kTopK; ++k) best[k] = best[k + 1];
            best[kTopK - 1] = 0xffffffffu;
        }
        if (tid == 0) out[r] = g;
        __syncthreads();
    }
}

}  // namespace

namespace {

using ovs::grow_dev;
using ovs::grow_host;

// Launches the top-8 search; result keys end up in d_out[nq * 8].
int launch_topk(ovs_matcher* h, const uint8_t* d_q, int nq, const uint8_t* d_t, int nt, unsigned* d_out) {
    cudaStream_t st = h->stream;
    const int qblocks = (nq + kQueriesPerBlock - 1) / kQueriesPerBlock;
    // enough (query block, train chunk) pairs for ~8 resident blocks (32 warps) per SM -- a thread walks its chunk serially, so the
    // warps in flight are what hides the shared-memory and insertion latency (4000 x 4000: 32 x 32 blocks); chunks a multiple of the tile
    int nchunks = std::max(1, (8 * h->num_sms + qblocks - 1) / qblocks);
    const int max_chunks = std::max(1, (nt + kTrainTile - 1) / kTrainTile);
    nchunks = std::min(nchunks, max_chunks);
    int chunk = (nt + nchunks - 1) / nchunks;
    chunk = std::max(kTrainTile, (chunk + kTrainTile - 1) / kTrainTile * kTrainTile);
    nchunks = std::max(1, (nt + chunk - 1) / chunk);
    unsigned* d_first = d_out;
    if (nchunks > 1) {
        int rc = grow_dev(&h->d_part, &h->d_part_cap, (size_t)nq * nchunks * kTopK);
        if (rc != OVS_OK) return rc;
        d_first = h->d_part;
    }
    dim3 grid(qblocks, nchunks);
    k_hamming_topk<<<grid, kQueriesPerBlock, 0, st>>>((const uint4*)d_q, nq, (const uint4*)d_t, nt, chunk, d_first);
    OVS_LAUNCH_CHECK();
    if (nchunks > 1) {
        k_topk_merge<<<(nq + 127) / 128, 128, 0, st>>>(h->d_part, nq, nchunks, d_out);
        OVS_LAUNCH_CHECK();
    }
    return OVS_OK;
}

using ovs::key_dist;
inline int key_idx(unsigned key) { return key == 0xffffffffu ? -1 : (int)(key & 0xffffu); }

}  // namespace

extern "C" int ovs_matcher_create(int device, ovs_matcher** out) {
    OVS_REQUIRE(out, OVS_ERR_INVALID_ARG, "null argument");
    int rc = ovs::select_device(device);
    if (rc != OVS_OK) return rc;
    ovs_matcher* h = new (std::nothrow) ovs_matcher();
    OVS_REQUIRE(h, OVS_ERR_CUDA, "out of host memory");
    h->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->num_sms = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&h->ev[0], ovs::event_flags()) != cudaSuccess
        || cudaEventCreateWithFlags(&h->ev[1], ovs::event_flags()) != cudaSuccess) {
        ovs::set_error("stream/event creation failed: %s", cudaGetErrorString(cudaGetLastError()));
        ovs_matcher_destroy(h);
        return OVS_ERR_CUDA;
    }
    *out = h;
    return OVS_OK;
}

extern "C" void ovs_matcher_destroy(ovs_matcher* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) ovs::sync_stream(h->stream);
    cudaFree(h->d_q); cudaFree(h->d_t); cudaFree(h->d_part); cudaFree(h->d_keys); cudaFree(h->d_mask); cudaFree(h->d_ess);
    cudaFree(h->d_tv); cudaFree(h->d_tri); cudaFree(h->d_init); cudaFree(h->d_trk); cudaFree(h->d_fuse);
    for (auto& b : h->index_pool) cudaFree(b.base);
    cudaFreeHost(h->h_keys); cudaFreeHost(h->h_stage); cudaFreeHost(h->h_ess); cudaFreeHost(h->h_tv); cudaFreeHost(h->h_tri);
    cudaFreeHost(h->h_init); cudaFreeHost(h->h_trk); cudaFreeHost(h->h_fuse);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" int ovs_match_bruteforce_topk_device(ovs_matcher* h, const uint8_t* d_query, int nq, const uint8_t* d_train, int nt,
                                                uint32_t* d_keys_out) {
    OVS_REQUIRE(h && d_keys_out && nq >= 0 && nt >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(nt < 65536, OVS_ERR_UNSUPPORTED, "train set larger than 65535 descriptors");
    if (nq == 0) return OVS_OK;
    OVS_REQUIRE(d_query && (nt == 0 || d_train), OVS_ERR_INVALID_ARG, "null descriptors");
    OVS_REQUIRE(((uintptr_t)d_query & 15) == 0 && ((uintptr_t)d_train & 15) == 0, OVS_ERR_INVALID_ARG, "descriptors must be 16-byte aligned");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], h->stream));
    int rc = launch_topk(h, d_query, nq, d_train, nt, d_keys_out);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], h->stream));
    OVS_CUDA_CHECK(ovs::sync_event(h->ev[1]));
    float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
    h->last_kernel_us = ms * 1000.f;
    return OVS_OK;
}

namespace {
// Uploads both descriptor sets and leaves the merged keys in h->h_keys (pinned).
int topk_host_impl(ovs_matcher* h, const uint8_t* query, int nq, const uint8_t* train, int nt) {
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc;
    if ((rc = grow_dev(&h->d_q, &h->d_q_cap, (size_t)nq * 32)) != OVS_OK) return rc;
    if ((rc = grow_dev(&h->d_t, &h->d_t_cap, (size_t)std::max(nt, 1) * 32)) != OVS_OK) return rc;
    // one spare row at the end: the re-query slot of ovs_robust_brute_force_match_host
    if ((rc = grow_dev(&h->d_keys, &h->d_keys_cap, (size_t)(nq + 1) * kTopK)) != OVS_OK) return rc;
    if ((rc = grow_host(&h->h_keys, &h->h_keys_cap, (size_t)(nq + 1) * kTopK)) != OVS_OK) return rc;
    if ((rc = grow_host(&h->h_stage, &h->h_stage_cap, (size_t)(nq + nt) * 32)) != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    memcpy(h->h_stage, query, (size_t)nq * 32);
    if (nt) memcpy(h->h_stage + (size_t)nq * 32, train, (size_t)nt * 32);
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_q, h->h_stage, (size_t)nq * 32, cudaMemcpyHostToDevice, st));
    if (nt) OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_t, h->h_stage + (size_t)nq * 32, (size_t)nt * 32, cudaMemcpyHostToDevice, st));
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    rc = launch_topk(h, h->d_q, nq, h->d_t, nt, h->d_keys);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_keys, h->d_keys, (size_t)nq * kTopK * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
    h->last_kernel_us = ms * 1000.f;
    return OVS_OK;
}
}  // namespace

extern "C" int ovs_match_bruteforce_topk_host(ovs_matcher* h, const uint8_t* query, int nq, const uint8_t* train, int nt,
                                              uint32_t* keys_out) {
    OVS_REQUIRE(h && keys_out && nq >= 0 && nt >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(nt < 65536, OVS_ERR_UNSUPPORTED, "train set larger than 65535 descriptors");
    if (nq == 0) return OVS_OK;
    OVS_REQUIRE(query && (nt == 0 || train), OVS_ERR_INVALID_ARG, "null descriptors");
    int rc = topk_host_impl(h, query, nq, train, nt);
    if (rc != OVS_OK) return rc;
    memcpy(keys_out, h->h_keys, (size_t)nq * kTopK * sizeof(unsigned));
    return OVS_OK;
}

extern "C" int ovs_match_bruteforce_host(ovs_matcher* h, const uint8_t* desc1, int n1, const uint8_t* desc2, int n2,
                                         int32_t* best_idx, int32_t* best_dist, int32_t* second_dist) {
    OVS_REQUIRE(h && n1 >= 0 && n2 >= 0 && (n1 == 0 || (best_idx && best_dist && second_dist)), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n2 < 65536, OVS_ERR_UNSUPPORTED, "train set larger than 65535 descriptors");
    if (n1 == 0) return OVS_OK;
    OVS_REQUIRE(desc1 && (n2 == 0 || desc2), OVS_ERR_INVALID_ARG, "null descriptors");
    int rc = topk_host_impl(h, desc1, n1, desc2, n2);
    if (rc != OVS_OK) return rc;
    for (int q = 0; q < n1; ++q) {
        const unsigned* k = h->h_keys + (size_t)q * kTopK;
        best_idx[q] = key_idx(k[0]); best_dist[q] = key_dist(k[0]); second_dist[q] = key_dist(k[1]);
    }
    return OVS_OK;
}

// robust::brute_force_match(frm, keyfrm, matches):
//   for idx_2 over keyframe keypoints with a valid landmark (lm_valid_2[idx_2] != 0, or all if NULL):
//     scan frame descriptors idx_1 not yet matched -> best / second best
//     reject if best > HAMMING_DIST_THR_LOW or lowe_ratio * second < best
//     else emit (best_idx_1, idx_2) and mark idx_1 matched.
// pairs_out[2*i] = idx_1 (frame), pairs_out[2*i+1] = idx_2 (keyframe).
namespace {
// Sequential replay of the reference's greedy rule over the per-query candidate lists in h->h_keys (queries = keyframe
// descriptors at d_query, train = frame descriptors at d_train, both resident on the device for the re-queries).
int robust_replay(ovs_matcher* h, const uint8_t* d_query, const uint8_t* d_train, int n1, int n2, const uint8_t* lm_valid_2, float lowe_ratio,
                  int32_t* pairs_out, int capacity, int* num_matches) {
    int rc;
    std::vector<unsigned> claimed((size_t)(n1 + 31) / 32, 0u);
    const auto unclaimed = [&](int i, int) { return !((claimed[i >> 5] >> (i & 31)) & 1u); };
    const auto ratio = [&](const ovs::ReplayList<kTopK>& L, int second, ovs::Second) { return !(lowe_ratio * (float)(unsigned)second < (float)L.dist[0]); };
    const int complete_at = ovs::d_star(lowe_ratio);
    int nm = 0;
    for (int q = 0; q < n2; ++q) {
        if (lm_valid_2 && !lm_valid_2[q]) continue;
        // re-query this keyframe descriptor on the GPU against the unclaimed frame descriptors, into the spare row n2
        const auto requery = [&](unsigned* fresh) -> int {
            const int rc2 = grow_dev(&h->d_mask, &h->d_mask_cap, claimed.size());
            if (rc2 != OVS_OK) return rc2;
            OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_mask, claimed.data(), claimed.size() * sizeof(unsigned), cudaMemcpyHostToDevice, h->stream));
            unsigned* d_slot = h->d_keys + (size_t)n2 * kTopK;
            unsigned* h_slot = h->h_keys + (size_t)n2 * kTopK;
            k_hamming_one<<<1, 256, 0, h->stream>>>(reinterpret_cast<const uint4*>(d_query + (size_t)q * 32), reinterpret_cast<const uint4*>(d_train), n1,
                                                    h->d_mask, d_slot);
            OVS_LAUNCH_CHECK();
            OVS_CUDA_CHECK(cudaMemcpyAsync(h_slot, d_slot, kTopK * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
            OVS_CUDA_CHECK(ovs::sync_stream(h->stream));
            memcpy(fresh, h_slot, kTopK * sizeof(unsigned));
            ++h->num_requeries;
            return OVS_OK;
        };
        ovs::ReplayPick p;
        rc = ovs::replay_query<kTopK>(h->h_keys + (size_t)q * kTopK, OVS_HAMMING_DIST_THR_LOW, complete_at, key_idx, unclaimed, ratio, requery, &p);
        if (rc != OVS_OK) return rc;
        if (p.id < 0) continue;
        OVS_REQUIRE(nm < capacity, OVS_ERR_CAPACITY, "pairs_out capacity %d too small", capacity);
        pairs_out[2 * nm] = p.id; pairs_out[2 * nm + 1] = q;
        claimed[p.id >> 5] |= 1u << (p.id & 31);
        ++nm;
    }
    *num_matches = nm;
    return OVS_OK;
}
}  // namespace

extern "C" int ovs_robust_brute_force_match_host(ovs_matcher* h, const uint8_t* desc_frm, int n1, const uint8_t* desc_keyfrm, int n2,
                                                 const uint8_t* lm_valid_2, float lowe_ratio,
                                                 int32_t* pairs_out, int capacity, int* num_matches) {
    OVS_REQUIRE(h && num_matches && n1 >= 0 && n2 >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n1 < 65536, OVS_ERR_UNSUPPORTED, "frame has more than 65535 keypoints");
    *num_matches = 0;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    OVS_REQUIRE(desc_frm && desc_keyfrm && (capacity == 0 || pairs_out), OVS_ERR_INVALID_ARG, "null argument");
    // queries = keyframe descriptors, train = frame descriptors
    int rc = topk_host_impl(h, desc_keyfrm, n2, desc_frm, n1);
    if (rc != OVS_OK) return rc;
    return robust_replay(h, h->d_q, h->d_t, n1, n2, lm_valid_2, lowe_ratio, pairs_out, capacity, num_matches);
}

// The same with both descriptor sets already in device memory (e.g. straight from ovs_extract_device): only the candidate
// lists (32 B per keyframe keypoint) come to the host for the sequential replay.  lm_valid_2 and pairs_out are host arrays.
extern "C" int ovs_robust_brute_force_match_device(ovs_matcher* h, const uint8_t* d_desc_frm, int n1, const uint8_t* d_desc_keyfrm, int n2,
                                                   const uint8_t* lm_valid_2, float lowe_ratio,
                                                   int32_t* pairs_out, int capacity, int* num_matches) {
    OVS_REQUIRE(h && num_matches && n1 >= 0 && n2 >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n1 < 65536, OVS_ERR_UNSUPPORTED, "frame has more than 65535 keypoints");
    *num_matches = 0;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    OVS_REQUIRE(d_desc_frm && d_desc_keyfrm && (capacity == 0 || pairs_out), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(((uintptr_t)d_desc_frm & 15) == 0 && ((uintptr_t)d_desc_keyfrm & 15) == 0, OVS_ERR_INVALID_ARG, "descriptors must be 16-byte aligned");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc;
    if ((rc = grow_dev(&h->d_keys, &h->d_keys_cap, (size_t)(n2 + 1) * kTopK)) != OVS_OK) return rc;
    if ((rc = grow_host(&h->h_keys, &h->h_keys_cap, (size_t)(n2 + 1) * kTopK)) != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    rc = launch_topk(h, d_desc_keyfrm, n2, d_desc_frm, n1, h->d_keys);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_keys, h->d_keys, (size_t)n2 * kTopK * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
    h->last_kernel_us = ms * 1000.f;
    return robust_replay(h, d_desc_keyfrm, d_desc_frm, n1, n2, lm_valid_2, lowe_ratio, pairs_out, capacity, num_matches);
}

extern "C" int ovs_matcher_num_requeries(const ovs_matcher* h, int* out) {
    OVS_REQUIRE(h && out, OVS_ERR_INVALID_ARG, "null argument");
    *out = h->num_requeries;
    return OVS_OK;
}

extern "C" int ovs_matcher_last_kernel_us(const ovs_matcher* h, float* out_us) {
    OVS_REQUIRE(h && out_us, OVS_ERR_INVALID_ARG, "null argument");
    *out_us = h->last_kernel_us;
    return OVS_OK;
}

// Development aid / test hook: the brute-force re-query (k_hamming_one, one block of 256, as robust_replay launches it) of one
// query descriptor on host arrays, through the matcher's own buffers.  tests/test_candidate_lists_gpu.py compares its keys
// with an exact numpy top-8.
extern "C" int ovs_debug_hamming_one(ovs_matcher* h, const uint8_t* query, const uint8_t* train, int nt, const uint32_t* exclude_mask,
                                     uint32_t* keys_out) {
    OVS_REQUIRE(h && query && train && exclude_mask && keys_out && nt >= 1, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(nt < 65536, OVS_ERR_UNSUPPORTED, "train set larger than 65535 descriptors");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    const size_t words = ((size_t)nt + 31) / 32;
    int rc;
    if ((rc = grow_dev(&h->d_q, &h->d_q_cap, 32)) != OVS_OK) return rc;
    if ((rc = grow_dev(&h->d_t, &h->d_t_cap, (size_t)nt * 32)) != OVS_OK) return rc;
    if ((rc = grow_dev(&h->d_mask, &h->d_mask_cap, words)) != OVS_OK) return rc;
    if ((rc = grow_dev(&h->d_keys, &h->d_keys_cap, (size_t)kTopK)) != OVS_OK) return rc;
    if ((rc = grow_host(&h->h_keys, &h->h_keys_cap, (size_t)kTopK)) != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_q, query, 32, cudaMemcpyHostToDevice, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_t, train, (size_t)nt * 32, cudaMemcpyHostToDevice, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_mask, exclude_mask, words * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(h->d_keys, 0x5a, kTopK * sizeof(unsigned), st));   // a key the kernel leaves unwritten shows
    k_hamming_one<<<1, 256, 0, st>>>(reinterpret_cast<const uint4*>(h->d_q), reinterpret_cast<const uint4*>(h->d_t), nt, h->d_mask, h->d_keys);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_keys, h->d_keys, kTopK * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(keys_out, h->h_keys, kTopK * sizeof(unsigned));
    return OVS_OK;
}
