// essential_ransac.cu -- H100 (sm_90a) implementation of openvslam::solve::essential_solver::find_via_ransac
// (solve/essential_solver.cc) for a batch of independent problems, and of match::robust::match_frame_and_keyframe
// (match/robust.cc: the brute force of match_bruteforce.cu followed by find_via_ransac(50, false)), the tracker's last fallback.
//
// Three launches per batch, one copy each way, one host wait:
//   k_essential_hypotheses  one thread per (problem, hypothesis): the counter-based sampler's 8 matches and the eight-point E_21
//   k_essential_score       one warp per hypothesis: check_inliers over the problem's matches (lanes take them with a stride of
//                           32, count by ballot, the 32 partial scores added in lane order) -> score and count per hypothesis
//   k_essential_refine      one 256-thread CTA per problem: the best hypothesis (first strictly greater score, from 0), its flags
//                           and `valid`; with recompute the eight-point E_21 on all inliers (CTA-wide fixed-order sum) and the
//                           flags, count and score re-checked at it
// The arithmetic is essential_math.cuh (host + device); the conventions are in DESIGN.md section 5.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "block_sum.cuh"
#include "essential_math.cuh"
#include "match_common.h"

namespace {

constexpr int kEssHypThreads = 64;                   // k_essential_hypotheses
constexpr int kEssWarps = 4;                         // k_essential_score: hypotheses per CTA, one warp each
constexpr int kEssThreads = 32 * kEssWarps;
constexpr int kEssRefineThreads = ovs::kBlockSumThreads;   // k_essential_refine: one CTA per problem

struct EssArgs {
    int B, H, recompute;
    const int* off;                                  // B + 1 match offsets
    const double* bear_1; const double* bear_2;      // per match, or per keypoint when pairs is set
    const int* pairs;                                // null, or 2 per match (index into bear_1, index into bear_2)
    const uint64_t* seed;                            // B
    double* hyp;                                     // B x H x 9: every hypothesis's E_21
    double* hscore; int* hcount;                     // B x H
    int* cidx;                                       // per match: the best hypothesis's inliers, compacted per problem
    double* E; double* score; int* num_inliers; int* best_iter; uint8_t* valid; uint8_t* inlier;   // out
};

__device__ __forceinline__ ovs::EssPairs ess_pairs(const EssArgs& A, int o) {
    if (A.pairs) return ovs::EssPairs{A.bear_1, A.bear_2, A.pairs + 2 * (size_t)o};
    return ovs::EssPairs{A.bear_1 + 3 * (size_t)o, A.bear_2 + 3 * (size_t)o, nullptr};
}

__global__ void __launch_bounds__(kEssHypThreads) k_essential_hypotheses(EssArgs A) {
    const size_t g = (size_t)blockIdx.x * kEssHypThreads + threadIdx.x;
    if (g >= (size_t)A.B * (size_t)A.H) return;
    const int b = (int)(g / (size_t)A.H), k = (int)(g % (size_t)A.H);
    const int o = A.off[b], n = A.off[b + 1] - o;
    if (n < ovs::kEssMinSet) return;
    int idx[ovs::kEssMinSet];
    ovs::ransac_sample<ovs::kEssMinSet>(A.seed[b], k, n, idx);
    ovs::essential_from_pairs(ess_pairs(A, o), idx, ovs::PnpSeqSum{ovs::kEssMinSet}, A.hyp + 9 * g);
}

// check_inliers of E over a problem's n matches by one warp: returns the count (every lane) and the score in lane order (every
// lane); the same bits as essential_score_seq.
__device__ __forceinline__ int warp_score(const double* E, const ovs::EssPairs& P, int n, int lane, double* score) {
    double part = 0.0;
    int cnt = 0;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool in = i < n && ovs::essential_check(E, P.b1(i), P.b2(i), part);
        cnt += __popc(__ballot_sync(0xffffffffu, in));
    }
    double total = 0.0;
    for (int l = 0; l < 32; ++l) total += __shfl_sync(0xffffffffu, part, l);
    *score = total;
    return cnt;
}

// grid (hypothesis blocks, problems), one warp per hypothesis: its score and count.  The selection is the sequential loop's
// rule, applied in k order by k_essential_refine, so no atomics are needed here.
__global__ void __launch_bounds__(kEssThreads) k_essential_score(EssArgs A) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const int k = blockIdx.x * kEssWarps + warp;
    if (n < ovs::kEssMinSet || k >= A.H) return;
    const size_t g = (size_t)b * A.H + k;
    double E[9];
    for (int m = 0; m < 9; ++m) E[m] = A.hyp[9 * g + m];
    double score;
    const int cnt = warp_score(E, ess_pairs(A, o), n, lane, &score);
    if (lane == 0) { A.hscore[g] = score; A.hcount[g] = cnt; }
}

// One CTA per problem: the best hypothesis (the first whose score is strictly greater than the best so far, which starts at 0;
// a NaN score never wins), its flags and `valid` = (best score > 0 and at least 8 inliers); with recompute and valid, the
// eight-point E_21 on the compacted inliers (index order, CTA-wide sums) and its flags, count and score.
__global__ void __launch_bounds__(kEssRefineThreads) k_essential_refine(EssArgs A) {
    __shared__ double s_red[ovs::kBlockSumChunk * kEssRefineThreads];
    __shared__ double s_res[45];
    __shared__ int s_warp[kEssRefineThreads / 32];
    __shared__ int s_best;
    __shared__ double s_score;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const ovs::EssPairs P = ess_pairs(A, o);
    if (t == 0) {
        int best = -1;
        double bs = 0.0;
        if (n >= ovs::kEssMinSet)
            for (int k = 0; k < A.H; ++k) {
                const double sc = A.hscore[(size_t)b * A.H + k];
                if (bs < sc) { bs = sc; best = k; }
            }
        s_best = best; s_score = bs;
    }
    __syncthreads();
    const int best = s_best;
    double score = s_score;
    double E[9];
    for (int m = 0; m < 9; ++m) E[m] = best >= 0 ? A.hyp[9 * ((size_t)b * A.H + best) + m] : 0.0;
    const int cnt = best >= 0 ? A.hcount[(size_t)b * A.H + best] : 0;
    const bool valid = score > 0.0 && cnt >= ovs::kEssMinSet;
    int num = cnt;
    double dummy = 0.0;
    for (int i = t; i < n; i += kEssRefineThreads) A.inlier[o + i] = (best >= 0 && ovs::essential_check(E, P.b1(i), P.b2(i), dummy)) ? 1 : 0;
    if (valid && A.recompute) {
        int running = 0;
        for (int base = 0; base < n; base += kEssRefineThreads) {   // compaction in index order
            const int i = base + t;
            const bool f = i < n && ovs::essential_check(E, P.b1(i), P.b2(i), dummy);
            const unsigned bal = __ballot_sync(0xffffffffu, f);
            if (lane == 0) s_warp[warp] = __popc(bal);
            __syncthreads();
            int before = running;
            for (int w = 0; w < warp; ++w) before += s_warp[w];
            if (f) A.cidx[o + before + __popc(bal & ((1u << lane) - 1u))] = i;
            for (int w = 0; w < kEssRefineThreads / 32; ++w) running += s_warp[w];
            __syncthreads();
        }
        __syncthreads();
        double En[9];
        ovs::essential_from_pairs(P, A.cidx + o, ovs::PnpBlockSum{cnt, s_red, s_res}, En);
        for (int m = 0; m < 9; ++m) E[m] = En[m];
        int c2 = 0;
        for (int base = 0; base < n; base += kEssRefineThreads) {
            const int i = base + t;
            const bool f = i < n && ovs::essential_check(E, P.b1(i), P.b2(i), dummy);
            if (i < n) A.inlier[o + i] = f ? 1 : 0;
            c2 += __syncthreads_count(f);
        }
        num = c2;
        if (warp == 0) {
            double sc;
            warp_score(E, P, n, lane, &sc);
            if (lane == 0) s_score = sc;
        }
        __syncthreads();
        score = s_score;
    }
    if (t < 9) A.E[9 * (size_t)b + t] = E[t];
    if (t == 0) {
        A.score[b] = score;
        A.num_inliers[b] = num;
        A.best_iter[b] = best;
        A.valid[b] = valid ? 1 : 0;
    }
}

struct Arena {
    uint8_t* base; size_t off;
    template <typename T> T* take(size_t n) {
        off = (off + 255) / 256 * 256;
        T* p = reinterpret_cast<T*>(base + off);
        off += n * sizeof(T);
        return p;
    }
};

// The bearings of a solve: host arrays (uploaded with the other inputs) or device arrays (read in place).
struct EssBearings {
    const double* b1; size_t n1;
    const double* b2; size_t n2;
    bool on_device;
};

// One batched solve on the matcher's essential arenas.  off: host, B + 1 offsets of N = off[B] matches; pairs: host, 2 per match
// or null; outputs: host.  E / score / num_inliers / best_iter / valid per problem, inlier_out per match.
int essential_run(ovs_matcher* h, int B, const int32_t* off, const int32_t* pairs, const EssBearings& bear, int max_num_iter,
                  int recompute, const uint64_t* seeds, double* E_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter,
                  double* best_score, uint8_t* inlier_out) {
    const size_t N = (size_t)off[B], NB = (size_t)B, H = (size_t)max_num_iter;
    const size_t np = pairs ? 2 * N : 0;
    const size_t up1 = bear.on_device ? 0 : 3 * bear.n1, up2 = bear.on_device ? 0 : 3 * bear.n2;
    const size_t in_max = 256 * 5 + (NB + 1) * 4 + NB * 8 + np * 4 + (up1 + up2) * 8;
    const size_t out_max = 256 * 6 + NB * (9 * 8 + 8 + 4 + 4 + 1) + N;
    const size_t hbytes = in_max + out_max;
    const size_t dbytes = hbytes + 256 * 4 + NB * H * (9 * 8 + 8 + 4) + N * 4 + 4096;
    int rc;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    if ((rc = ovs::grow_dev(&h->d_ess, &h->d_ess_cap, dbytes)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&h->h_ess, &h->h_ess_cap, hbytes)) != OVS_OK) return rc;
    Arena Hh{h->h_ess, 0}, D{h->d_ess, 0};
    // inputs: the same carving sequence in both arenas, so one contiguous copy moves them
    int* hoff = Hh.take<int>(NB + 1); uint64_t* hseed = Hh.take<uint64_t>(NB);
    int* hpairs = pairs ? Hh.take<int>(np) : nullptr;
    double* hb1 = bear.on_device ? nullptr : Hh.take<double>(up1);
    double* hb2 = bear.on_device ? nullptr : Hh.take<double>(up2);
    const size_t in_bytes = Hh.off;
    // outputs: one contiguous copy back
    double* hE = Hh.take<double>(9 * NB);
    const size_t out_begin = (size_t)((uint8_t*)hE - h->h_ess);
    double* hscore = Hh.take<double>(NB); int* hnum = Hh.take<int>(NB); int* hbest = Hh.take<int>(NB);
    uint8_t* hvalid = Hh.take<uint8_t>(NB); uint8_t* hflags = Hh.take<uint8_t>(N);
    const size_t out_end = Hh.off;
    EssArgs A;
    A.B = B; A.H = max_num_iter; A.recompute = recompute ? 1 : 0;
    A.off = D.take<int>(NB + 1); A.seed = D.take<uint64_t>(NB);
    A.pairs = pairs ? D.take<int>(np) : nullptr;
    if (bear.on_device) { A.bear_1 = bear.b1; A.bear_2 = bear.b2; }
    else { A.bear_1 = D.take<double>(up1); A.bear_2 = D.take<double>(up2); }
    A.E = D.take<double>(9 * NB); A.score = D.take<double>(NB); A.num_inliers = D.take<int>(NB); A.best_iter = D.take<int>(NB);
    A.valid = D.take<uint8_t>(NB); A.inlier = D.take<uint8_t>(N);
    A.hyp = D.take<double>(9 * NB * H); A.hscore = D.take<double>(NB * H); A.hcount = D.take<int>(NB * H); A.cidx = D.take<int>(N);
    memcpy(hoff, off, 4 * (NB + 1)); memcpy(hseed, seeds, 8 * NB);
    if (pairs) memcpy(hpairs, pairs, 4 * np);
    if (!bear.on_device) {
        if (up1) memcpy(hb1, bear.b1, 8 * up1);
        if (up2) memcpy(hb2, bear.b2, 8 * up2);
    }
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_ess, h->h_ess, in_bytes, cudaMemcpyHostToDevice, st));
    if (max_num_iter > 0) {
        const size_t hyp_threads = NB * H;
        k_essential_hypotheses<<<(unsigned)((hyp_threads + kEssHypThreads - 1) / kEssHypThreads), kEssHypThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
        k_essential_score<<<dim3((max_num_iter + kEssWarps - 1) / kEssWarps, B), kEssThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
    }
    k_essential_refine<<<B, kEssRefineThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_ess + out_begin, h->d_ess + out_begin, out_end - out_begin, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(E_21, hE, 9 * 8 * NB); memcpy(best_score, hscore, 8 * NB);
    memcpy(num_inliers, hnum, 4 * NB); memcpy(best_iter, hbest, 4 * NB); memcpy(valid, hvalid, NB);
    if (N) memcpy(inlier_out, hflags, N);
    return OVS_OK;
}

int check_bearings(const double* b, int n, const char* what) {
    for (int i = 0; i < n; ++i) {
        const double* v = b + 3 * (size_t)i;
        OVS_REQUIRE(std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]) &&
                    std::fabs(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] - 1.0) <= 1e-6,
                    OVS_ERR_INVALID_ARG, "%s %d is not a finite unit vector", what, i);
    }
    return OVS_OK;
}

// robust::match_frame_and_keyframe after its brute force: the solver on the pairs (find_via_ransac(max_num_iter, false)), then
// matched_keyfrm_idx_of_frm[idx_1] = idx_2 for every inlier pair of a valid solution.
int robust_solve_pairs(ovs_matcher* h, const std::vector<int32_t>& pairs, int np, const EssBearings& bear, int max_num_iter, uint64_t seed,
                       int32_t* matched_keyfrm_idx_of_frm, int* num_inlier_matches) {
    if (np < ovs::kEssMinSet) return OVS_OK;   // find_via_ransac on fewer than 8 matches: invalid, nothing matched
    const int32_t off[2] = {0, np};
    double E[9], score;
    uint8_t valid;
    int32_t num, best;
    std::vector<uint8_t> flags((size_t)np);
    int rc = essential_run(h, 1, off, pairs.data(), bear, max_num_iter, 0, &seed, E, &valid, &num, &best, &score, flags.data());
    if (rc != OVS_OK) return rc;
    if (!valid) return OVS_OK;
    int cnt = 0;
    for (int i = 0; i < np; ++i) {
        if (!flags[i]) continue;
        matched_keyfrm_idx_of_frm[pairs[2 * i]] = pairs[2 * i + 1];
        ++cnt;
    }
    *num_inlier_matches = cnt;
    return OVS_OK;
}

}  // namespace

extern "C" int ovs_essential_solve_ransac_host(ovs_matcher* h, int B, const int32_t* match_offsets, const double* bearings_1,
                                               const double* bearings_2, int max_num_iter, int recompute, const uint64_t* seeds,
                                               double* E_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                               uint8_t* inlier_out) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(max_num_iter >= 0, OVS_ERR_INVALID_ARG, "max_num_iter must not be negative");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(match_offsets && seeds && E_21 && valid && num_inliers && best_iter && best_score, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(match_offsets[0] == 0, OVS_ERR_INVALID_ARG, "match_offsets[0] must be 0");
    for (int b = 0; b < B; ++b)
        OVS_REQUIRE(match_offsets[b + 1] >= match_offsets[b], OVS_ERR_INVALID_ARG, "match_offsets must be non-decreasing (problem %d)", b);
    const int n_all = match_offsets[B];
    OVS_REQUIRE(n_all == 0 || (bearings_1 && bearings_2 && inlier_out), OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    if ((rc = check_bearings(bearings_1, n_all, "bearings_1 of match")) != OVS_OK) return rc;
    if ((rc = check_bearings(bearings_2, n_all, "bearings_2 of match")) != OVS_OK) return rc;
    if (n_all == 0) {   // no match at all: no hypothesis, invalid
        for (int b = 0; b < B; ++b) {
            for (int k = 0; k < 9; ++k) E_21[9 * (size_t)b + k] = 0.0;
            valid[b] = 0; num_inliers[b] = 0; best_iter[b] = -1; best_score[b] = 0.0;
        }
        return OVS_OK;
    }
    const EssBearings bear{bearings_1, (size_t)n_all, bearings_2, (size_t)n_all, false};
    return essential_run(h, B, match_offsets, nullptr, bear, max_num_iter, recompute, seeds, E_21, valid, num_inliers, best_iter,
                         best_score, inlier_out);
}

extern "C" int ovs_robust_match_frame_and_keyframe_host(ovs_matcher* h, const uint8_t* desc_frm, const double* bearings_frm, int n1,
                                                        const uint8_t* desc_keyfrm, const double* bearings_keyfrm, int n2,
                                                        const uint8_t* lm_valid_2, float lowe_ratio, int max_num_iter, uint64_t seed,
                                                        int32_t* matched_keyfrm_idx_of_frm, int* num_inlier_matches) {
    OVS_REQUIRE(h && num_inlier_matches && n1 >= 0 && n2 >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(max_num_iter >= 0, OVS_ERR_INVALID_ARG, "max_num_iter must not be negative");
    OVS_REQUIRE(n1 == 0 || matched_keyfrm_idx_of_frm, OVS_ERR_INVALID_ARG, "null argument");
    *num_inlier_matches = 0;
    for (int i = 0; i < n1; ++i) matched_keyfrm_idx_of_frm[i] = -1;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    OVS_REQUIRE(bearings_frm && bearings_keyfrm, OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    if ((rc = check_bearings(bearings_frm, n1, "bearing of frame keypoint")) != OVS_OK) return rc;
    if ((rc = check_bearings(bearings_keyfrm, n2, "bearing of keyframe keypoint")) != OVS_OK) return rc;
    std::vector<int32_t> pairs(2 * (size_t)std::min(n1, n2));
    int np = 0;
    if ((rc = ovs_robust_brute_force_match_host(h, desc_frm, n1, desc_keyfrm, n2, lm_valid_2, lowe_ratio, pairs.data(),
                                                std::min(n1, n2), &np)) != OVS_OK)
        return rc;
    const EssBearings bear{bearings_frm, (size_t)n1, bearings_keyfrm, (size_t)n2, false};
    return robust_solve_pairs(h, pairs, np, bear, max_num_iter, seed, matched_keyfrm_idx_of_frm, num_inlier_matches);
}

extern "C" int ovs_robust_match_frame_and_keyframe_device(ovs_matcher* h, const uint8_t* d_desc_frm, const double* d_bearings_frm, int n1,
                                                          const uint8_t* d_desc_keyfrm, const double* d_bearings_keyfrm, int n2,
                                                          const uint8_t* lm_valid_2, float lowe_ratio, int max_num_iter, uint64_t seed,
                                                          int32_t* matched_keyfrm_idx_of_frm, int* num_inlier_matches) {
    OVS_REQUIRE(h && num_inlier_matches && n1 >= 0 && n2 >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(max_num_iter >= 0, OVS_ERR_INVALID_ARG, "max_num_iter must not be negative");
    OVS_REQUIRE(n1 == 0 || matched_keyfrm_idx_of_frm, OVS_ERR_INVALID_ARG, "null argument");
    *num_inlier_matches = 0;
    for (int i = 0; i < n1; ++i) matched_keyfrm_idx_of_frm[i] = -1;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    OVS_REQUIRE(d_bearings_frm && d_bearings_keyfrm, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(((uintptr_t)d_bearings_frm & 7) == 0 && ((uintptr_t)d_bearings_keyfrm & 7) == 0, OVS_ERR_INVALID_ARG,
                "bearings must be 8-byte aligned");
    std::vector<int32_t> pairs(2 * (size_t)std::min(n1, n2));
    int np = 0, rc;
    if ((rc = ovs_robust_brute_force_match_device(h, d_desc_frm, n1, d_desc_keyfrm, n2, lm_valid_2, lowe_ratio, pairs.data(),
                                                  std::min(n1, n2), &np)) != OVS_OK)
        return rc;
    const EssBearings bear{d_bearings_frm, (size_t)n1, d_bearings_keyfrm, (size_t)n2, true};
    return robust_solve_pairs(h, pairs, np, bear, max_num_iter, seed, matched_keyfrm_idx_of_frm, num_inlier_matches);
}
