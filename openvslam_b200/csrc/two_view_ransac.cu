// two_view_ransac.cu -- H100 (sm_90a) implementation of openvslam::solve::homography_solver::find_via_ransac and
// solve::fundamental_solver::find_via_ransac (solve/{homography,fundamental}_solver.cc), the two solvers perspective map
// initialisation (initialize::perspective::initialize) runs on every frame until the map exists, for a batch of independent
// problems.  One kernel template per stage, instantiated for H and for F.
//
// Four launches per batch (one with max_num_iter == 0), one copy each way, one host wait:
//   k_two_view_normalize      one thread per (problem, view): solve::common's normalize over all of the view's keypoints
//   k_two_view_hypotheses     one thread per (problem, hypothesis): the counter-based sampler's 8 matches, the minimal solve on
//                             their normalised points and the denormalisation
//   k_two_view_score          one warp per hypothesis: check_inliers over the problem's matches (lanes take them with a stride of
//                             32, count by ballot, the 32 partial scores added in lane order) -> score and count per hypothesis
//   k_two_view_refine         one 256-thread CTA per problem: the best hypothesis (first strictly greater score, from 0), its
//                             flags and `valid`; with recompute the model solved again on all inliers (CTA-wide fixed-order sum)
//                             and the flags, count and score re-checked at it
// The arithmetic is two_view_math.cuh (host + device); the conventions are in DESIGN.md section 5.
#include <cmath>
#include <cstring>

#include "block_sum.cuh"
#include "match_common.h"
#include "two_view_math.cuh"

namespace {

constexpr int kTvNormThreads = 64;                   // k_two_view_normalize
constexpr int kTvHypThreads = 64;                    // k_two_view_hypotheses
constexpr int kTvWarps = 4;                          // k_two_view_score: hypotheses per CTA, one warp each
constexpr int kTvThreads = 32 * kTvWarps;
constexpr int kTvRefineThreads = ovs::kBlockSumThreads;   // k_two_view_refine: one CTA per problem

struct TvArgs {
    int B, H, recompute;
    double inv_sigma_sq;
    const int* moff;                                 // B + 1 match offsets
    const int* koff_1; const int* koff_2;            // B + 1 keypoint offsets per view
    const float* kp_1; const float* kp_2;            // x, y per keypoint
    float* np_1; float* np_2;                        // normalised x, y per keypoint
    ovs::TwoViewNorm* norm;                          // B x 2 (view 1, view 2)
    const int* pairs;                                // 2 per match: keypoint of view 1, keypoint of view 2 (problem-local)
    const uint64_t* seed;                            // B
    double* hyp;                                     // B x H x 9: every hypothesis's model
    double* hscore; int* hcount;                     // B x H
    int* cidx;                                       // per match: the best hypothesis's inliers, compacted per problem
    double* M; double* score; int* num_inliers; int* best_iter; uint8_t* valid; uint8_t* inlier;   // out
};

__device__ __forceinline__ ovs::TwoViewPairs tv_pairs(const TvArgs& A, int b) {
    const size_t k1 = 2 * (size_t)A.koff_1[b], k2 = 2 * (size_t)A.koff_2[b];
    return ovs::TwoViewPairs{A.kp_1 + k1, A.kp_2 + k2, A.np_1 + k1, A.np_2 + k2, A.pairs + 2 * (size_t)A.moff[b]};
}

__global__ void __launch_bounds__(kTvNormThreads) k_two_view_normalize(TvArgs A) {
    const int g = blockIdx.x * kTvNormThreads + threadIdx.x;
    if (g >= 2 * A.B) return;
    const int b = g >> 1, view = g & 1;
    if (A.moff[b + 1] - A.moff[b] < ovs::kTwoViewMinSet) return;   // no hypothesis reads it
    const int* koff = view ? A.koff_2 : A.koff_1;
    const size_t o = 2 * (size_t)koff[b];
    A.norm[g] = ovs::two_view_normalize((view ? A.kp_2 : A.kp_1) + o, koff[b + 1] - koff[b], (view ? A.np_2 : A.np_1) + o);
}

template <int Model>
__global__ void __launch_bounds__(kTvHypThreads) k_two_view_hypotheses(TvArgs A) {
    const size_t g = (size_t)blockIdx.x * kTvHypThreads + threadIdx.x;
    if (g >= (size_t)A.B * (size_t)A.H) return;
    const int b = (int)(g / (size_t)A.H), k = (int)(g % (size_t)A.H);
    const int n = A.moff[b + 1] - A.moff[b];
    if (n < ovs::kTwoViewMinSet) return;
    int idx[ovs::kTwoViewMinSet];
    ovs::ransac_sample<ovs::kTwoViewMinSet>(A.seed[b], k, n, idx);
    ovs::two_view_solve<Model>(tv_pairs(A, b), idx, ovs::PnpSeqSum{ovs::kTwoViewMinSet}, A.norm[2 * b], A.norm[2 * b + 1], A.hyp + 9 * g);
}

// check_inliers of a model over a problem's n matches by one warp: returns the count (every lane) and the score in lane order
// (every lane); the same bits as two_view_score_seq.
template <int Model>
__device__ __forceinline__ int tv_warp_score(const ovs::TwoViewCheck<Model>& chk, const ovs::TwoViewPairs& P, int n, double iss, int lane,
                                             double* score) {
    double part = 0.0;
    int cnt = 0;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool in = i < n && chk(P.k1(i), P.k2(i), iss, part);
        cnt += __popc(__ballot_sync(0xffffffffu, in));
    }
    double total = 0.0;
    for (int l = 0; l < 32; ++l) total += __shfl_sync(0xffffffffu, part, l);
    *score = total;
    return cnt;
}

// grid (hypothesis blocks, problems), one warp per hypothesis: its score and count.  The selection is the sequential loop's
// rule, applied in k order by k_two_view_refine, so no atomics are needed here.
template <int Model>
__global__ void __launch_bounds__(kTvThreads) k_two_view_score(TvArgs A) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = A.moff[b + 1] - A.moff[b];
    const int k = blockIdx.x * kTvWarps + warp;
    if (n < ovs::kTwoViewMinSet || k >= A.H) return;
    const size_t g = (size_t)b * A.H + k;
    double M[9];
    for (int m = 0; m < 9; ++m) M[m] = A.hyp[9 * g + m];
    const ovs::TwoViewCheck<Model> chk(M);
    double score;
    const int cnt = tv_warp_score<Model>(chk, tv_pairs(A, b), n, A.inv_sigma_sq, lane, &score);
    if (lane == 0) { A.hscore[g] = score; A.hcount[g] = cnt; }
}

// One CTA per problem: the best hypothesis (the first whose score is strictly greater than the best so far, which starts at 0;
// a NaN score never wins), its flags and `valid` = (best score > 0 and at least 8 inliers); with recompute and valid, the model
// solved again on the compacted inliers (index order, CTA-wide sums) and its flags, count and score.
template <int Model>
__global__ void __launch_bounds__(kTvRefineThreads) k_two_view_refine(TvArgs A) {
    __shared__ double s_red[ovs::kBlockSumChunk * kTvRefineThreads];
    __shared__ double s_res[45];
    __shared__ int s_warp[kTvRefineThreads / 32];
    __shared__ int s_best;
    __shared__ double s_score;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int o = A.moff[b], n = A.moff[b + 1] - o;
    const double iss = A.inv_sigma_sq;
    if (t == 0) {
        int best = -1;
        double bs = 0.0;
        if (n >= ovs::kTwoViewMinSet)
            for (int k = 0; k < A.H; ++k) {
                const double sc = A.hscore[(size_t)b * A.H + k];
                if (bs < sc) { bs = sc; best = k; }
            }
        s_best = best; s_score = bs;
    }
    __syncthreads();
    const int best = s_best;
    double score = s_score;
    double M[9];
    for (int m = 0; m < 9; ++m) M[m] = best >= 0 ? A.hyp[9 * ((size_t)b * A.H + best) + m] : 0.0;
    const int cnt = best >= 0 ? A.hcount[(size_t)b * A.H + best] : 0;
    const bool valid = score > 0.0 && cnt >= ovs::kTwoViewMinSet;
    int num = cnt;
    double dummy = 0.0;
    if (best < 0) {
        for (int i = t; i < n; i += kTvRefineThreads) A.inlier[o + i] = 0;
    } else {
        const ovs::TwoViewPairs P = tv_pairs(A, b);
        {
            const ovs::TwoViewCheck<Model> chk(M);
            for (int i = t; i < n; i += kTvRefineThreads) A.inlier[o + i] = chk(P.k1(i), P.k2(i), iss, dummy) ? 1 : 0;
        }
        if (valid && A.recompute) {
            __syncthreads();   // the flags above are read back below
            int running = 0;
            for (int base = 0; base < n; base += kTvRefineThreads) {   // compaction in index order
                const int i = base + t;
                const bool f = i < n && A.inlier[o + i];
                const unsigned bal = __ballot_sync(0xffffffffu, f);
                if (lane == 0) s_warp[warp] = __popc(bal);
                __syncthreads();
                int before = running;
                for (int w = 0; w < warp; ++w) before += s_warp[w];
                if (f) A.cidx[o + before + __popc(bal & ((1u << lane) - 1u))] = i;
                for (int w = 0; w < kTvRefineThreads / 32; ++w) running += s_warp[w];
                __syncthreads();
            }
            __syncthreads();
            ovs::two_view_solve<Model>(P, A.cidx + o, ovs::PnpBlockSum{cnt, s_red, s_res}, A.norm[2 * b], A.norm[2 * b + 1], M);
            const ovs::TwoViewCheck<Model> chk(M);
            int c2 = 0;
            for (int base = 0; base < n; base += kTvRefineThreads) {
                const int i = base + t;
                const bool f = i < n && chk(P.k1(i), P.k2(i), iss, dummy);
                if (i < n) A.inlier[o + i] = f ? 1 : 0;
                c2 += __syncthreads_count(f);
            }
            num = c2;
            if (warp == 0) {
                double sc;
                tv_warp_score<Model>(chk, P, n, iss, lane, &sc);
                if (lane == 0) s_score = sc;
            }
            __syncthreads();
            score = s_score;
        }
    }
    if (t < 9) A.M[9 * (size_t)b + t] = M[t];
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

// One batched solve on the matcher's two-view arenas.  All arrays are host arrays, already validated.
template <int Model>
int two_view_run(ovs_matcher* h, int B, const int32_t* koff_1, const ovs_keypoint* keypts_1, const int32_t* koff_2,
                 const ovs_keypoint* keypts_2, const int32_t* moff, const int32_t* matches_12, float sigma, int max_num_iter, int recompute,
                 const uint64_t* seeds, double* M_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                 uint8_t* inlier_out) {
    const size_t N = (size_t)moff[B], K1 = (size_t)koff_1[B], K2 = (size_t)koff_2[B], NB = (size_t)B, H = (size_t)max_num_iter;
    const size_t in_max = 256 * 6 + 3 * (NB + 1) * 4 + NB * 8 + 2 * N * 4 + 2 * (K1 + K2) * 4;
    const size_t out_max = 256 * 6 + NB * (9 * 8 + 8 + 4 + 4 + 1) + N;
    const size_t hbytes = in_max + out_max;
    const size_t dbytes = hbytes + 256 * 6 + 2 * (K1 + K2) * 4 + NB * 2 * sizeof(ovs::TwoViewNorm) + NB * H * (9 * 8 + 8 + 4) + N * 4 + 4096;
    int rc;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    if ((rc = ovs::grow_dev(&h->d_tv, &h->d_tv_cap, dbytes)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&h->h_tv, &h->h_tv_cap, hbytes)) != OVS_OK) return rc;
    Arena Hh{h->h_tv, 0}, D{h->d_tv, 0};
    // inputs: the same carving sequence in both arenas, so one contiguous copy moves them
    int* hmoff = Hh.take<int>(NB + 1); int* hk1 = Hh.take<int>(NB + 1); int* hk2 = Hh.take<int>(NB + 1);
    uint64_t* hseed = Hh.take<uint64_t>(NB); int* hpairs = Hh.take<int>(2 * N);
    float* hkp1 = Hh.take<float>(2 * K1); float* hkp2 = Hh.take<float>(2 * K2);
    const size_t in_bytes = Hh.off;
    // outputs: one contiguous copy back
    double* hM = Hh.take<double>(9 * NB);
    const size_t out_begin = (size_t)((uint8_t*)hM - h->h_tv);
    double* hscore = Hh.take<double>(NB); int* hnum = Hh.take<int>(NB); int* hbest = Hh.take<int>(NB);
    uint8_t* hvalid = Hh.take<uint8_t>(NB); uint8_t* hflags = Hh.take<uint8_t>(N);
    const size_t out_end = Hh.off;
    TvArgs A;
    A.B = B; A.H = max_num_iter; A.recompute = recompute ? 1 : 0;
    A.inv_sigma_sq = (double)ovs::two_view_inv_sigma_sq(sigma);
    A.moff = D.take<int>(NB + 1); A.koff_1 = D.take<int>(NB + 1); A.koff_2 = D.take<int>(NB + 1);
    A.seed = D.take<uint64_t>(NB); A.pairs = D.take<int>(2 * N);
    A.kp_1 = D.take<float>(2 * K1); A.kp_2 = D.take<float>(2 * K2);
    A.M = D.take<double>(9 * NB); A.score = D.take<double>(NB); A.num_inliers = D.take<int>(NB); A.best_iter = D.take<int>(NB);
    A.valid = D.take<uint8_t>(NB); A.inlier = D.take<uint8_t>(N);
    A.np_1 = D.take<float>(2 * K1); A.np_2 = D.take<float>(2 * K2); A.norm = D.take<ovs::TwoViewNorm>(2 * NB);
    A.hyp = D.take<double>(9 * NB * H); A.hscore = D.take<double>(NB * H); A.hcount = D.take<int>(NB * H); A.cidx = D.take<int>(N);
    memcpy(hmoff, moff, 4 * (NB + 1)); memcpy(hk1, koff_1, 4 * (NB + 1)); memcpy(hk2, koff_2, 4 * (NB + 1));
    memcpy(hseed, seeds, 8 * NB); memcpy(hpairs, matches_12, 8 * N);
    for (size_t i = 0; i < K1; ++i) { hkp1[2 * i] = keypts_1[i].x; hkp1[2 * i + 1] = keypts_1[i].y; }
    for (size_t i = 0; i < K2; ++i) { hkp2[2 * i] = keypts_2[i].x; hkp2[2 * i + 1] = keypts_2[i].y; }
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_tv, h->h_tv, in_bytes, cudaMemcpyHostToDevice, st));
    if (max_num_iter > 0) {
        k_two_view_normalize<<<(2 * B + kTvNormThreads - 1) / kTvNormThreads, kTvNormThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
        const size_t hyp_threads = NB * H;
        k_two_view_hypotheses<Model><<<(unsigned)((hyp_threads + kTvHypThreads - 1) / kTvHypThreads), kTvHypThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
        k_two_view_score<Model><<<dim3((max_num_iter + kTvWarps - 1) / kTvWarps, B), kTvThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
    }
    k_two_view_refine<Model><<<B, kTvRefineThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_tv + out_begin, h->d_tv + out_begin, out_end - out_begin, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(M_21, hM, 9 * 8 * NB); memcpy(best_score, hscore, 8 * NB);
    memcpy(num_inliers, hnum, 4 * NB); memcpy(best_iter, hbest, 4 * NB); memcpy(valid, hvalid, NB);
    if (N) memcpy(inlier_out, hflags, N);
    return OVS_OK;
}

int check_offsets(const int32_t* off, int B, const char* what) {
    OVS_REQUIRE(off[0] == 0, OVS_ERR_INVALID_ARG, "%s[0] must be 0", what);
    for (int b = 0; b < B; ++b)
        OVS_REQUIRE(off[b + 1] >= off[b], OVS_ERR_INVALID_ARG, "%s must be non-decreasing (problem %d)", what, b);
    return OVS_OK;
}

// Validation on the host (nothing is launched for bad input), then the solve.
template <int Model>
int two_view_solve_host(ovs_matcher* h, int B, const int32_t* keypt_offsets_1, const ovs_keypoint* keypts_1, const int32_t* keypt_offsets_2,
                        const ovs_keypoint* keypts_2, const int32_t* match_offsets, const int32_t* matches_12, float sigma, int max_num_iter,
                        int recompute, const uint64_t* seeds, double* M_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter,
                        double* best_score, uint8_t* inlier_out) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(sigma > 0.0f && std::isfinite(sigma), OVS_ERR_INVALID_ARG, "sigma must be positive and finite");
    OVS_REQUIRE(max_num_iter >= 0, OVS_ERR_INVALID_ARG, "max_num_iter must not be negative");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(keypt_offsets_1 && keypt_offsets_2 && match_offsets && seeds && M_21 && valid && num_inliers && best_iter && best_score,
                OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    if ((rc = check_offsets(keypt_offsets_1, B, "keypt_offsets_1")) != OVS_OK) return rc;
    if ((rc = check_offsets(keypt_offsets_2, B, "keypt_offsets_2")) != OVS_OK) return rc;
    if ((rc = check_offsets(match_offsets, B, "match_offsets")) != OVS_OK) return rc;
    const int K1 = keypt_offsets_1[B], K2 = keypt_offsets_2[B], n_all = match_offsets[B];
    OVS_REQUIRE((K1 == 0 || keypts_1) && (K2 == 0 || keypts_2) && (n_all == 0 || (matches_12 && inlier_out)), OVS_ERR_INVALID_ARG,
                "null argument");
    for (int i = 0; i < K1; ++i)
        OVS_REQUIRE(std::isfinite(keypts_1[i].x) && std::isfinite(keypts_1[i].y), OVS_ERR_INVALID_ARG, "keypoint %d of view 1 is not finite", i);
    for (int i = 0; i < K2; ++i)
        OVS_REQUIRE(std::isfinite(keypts_2[i].x) && std::isfinite(keypts_2[i].y), OVS_ERR_INVALID_ARG, "keypoint %d of view 2 is not finite", i);
    for (int b = 0; b < B; ++b) {
        const int n1 = keypt_offsets_1[b + 1] - keypt_offsets_1[b], n2 = keypt_offsets_2[b + 1] - keypt_offsets_2[b];
        for (int m = match_offsets[b]; m < match_offsets[b + 1]; ++m)
            OVS_REQUIRE(matches_12[2 * (size_t)m] >= 0 && matches_12[2 * (size_t)m] < n1 && matches_12[2 * (size_t)m + 1] >= 0 &&
                        matches_12[2 * (size_t)m + 1] < n2, OVS_ERR_INVALID_ARG, "match %d of problem %d indexes no keypoint", m, b);
    }
    if (n_all == 0) {   // no match at all: no hypothesis, invalid
        for (int b = 0; b < B; ++b) {
            for (int k = 0; k < 9; ++k) M_21[9 * (size_t)b + k] = 0.0;
            valid[b] = 0; num_inliers[b] = 0; best_iter[b] = -1; best_score[b] = 0.0;
        }
        return OVS_OK;
    }
    return two_view_run<Model>(h, B, keypt_offsets_1, keypts_1, keypt_offsets_2, keypts_2, match_offsets, matches_12, sigma, max_num_iter,
                               recompute, seeds, M_21, valid, num_inliers, best_iter, best_score, inlier_out);
}

}  // namespace

extern "C" int ovs_homography_solve_ransac_host(ovs_matcher* h, int B, const int32_t* keypt_offsets_1, const ovs_keypoint* keypts_1,
                                                const int32_t* keypt_offsets_2, const ovs_keypoint* keypts_2, const int32_t* match_offsets,
                                                const int32_t* matches_12, float sigma, int max_num_iter, int recompute, const uint64_t* seeds,
                                                double* H_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                                uint8_t* inlier_out) {
    return two_view_solve_host<ovs::kTwoViewH>(h, B, keypt_offsets_1, keypts_1, keypt_offsets_2, keypts_2, match_offsets, matches_12, sigma,
                                               max_num_iter, recompute, seeds, H_21, valid, num_inliers, best_iter, best_score, inlier_out);
}

extern "C" int ovs_fundamental_solve_ransac_host(ovs_matcher* h, int B, const int32_t* keypt_offsets_1, const ovs_keypoint* keypts_1,
                                                 const int32_t* keypt_offsets_2, const ovs_keypoint* keypts_2, const int32_t* match_offsets,
                                                 const int32_t* matches_12, float sigma, int max_num_iter, int recompute, const uint64_t* seeds,
                                                 double* F_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                                 uint8_t* inlier_out) {
    return two_view_solve_host<ovs::kTwoViewF>(h, B, keypt_offsets_1, keypts_1, keypt_offsets_2, keypts_2, match_offsets, matches_12, sigma,
                                               max_num_iter, recompute, seeds, F_21, valid, num_inliers, best_iter, best_score, inlier_out);
}
