// two_view_ransac.cu -- H100 (sm_90a) implementation of the three two-view RANSAC solvers' find_via_ransac, each for a batch of
// independent problems:
//   solve::essential_solver (solve/essential_solver.cc) on bearing pairs, also run by match::robust::match_frame_and_keyframe
//   (match/robust.cc: the brute force of match_bruteforce.cu followed by find_via_ransac(50, false)), the tracker's last fallback;
//   solve::homography_solver and solve::fundamental_solver (solve/{homography,fundamental}_solver.cc) on keypoint matches, the two
//   solvers perspective map initialisation (initialize::perspective::initialize) runs on every frame until the map exists.
// One kernel template per stage, instantiated for each model (EssentialModel, TwoViewModel<kTwoViewH>, TwoViewModel<kTwoViewF>).
//
// Three launches per batch (four for H and F; one with max_num_iter == 0), one copy each way, one host wait:
//   k_two_view_normalize      H and F only, one thread per (problem, view): solve::common's normalize over all of the view's
//                             keypoints
//   k_two_view_hypotheses     one thread per (problem, hypothesis): the counter-based sampler's 8 matches and the minimal solve
//                             (for H and F on their normalised points, then denormalised)
//   k_two_view_score          one warp per hypothesis: check_inliers over the problem's matches (lanes take them with a stride of
//                             32, count by ballot, the 32 partial scores added in lane order) -> score and count per hypothesis
//   k_two_view_refine         one 256-thread CTA per problem: the best hypothesis (first strictly greater score, from 0), its
//                             flags and `valid`; with recompute the model solved again on all inliers (CTA-wide fixed-order sum)
//                             and the flags, count and score re-checked at it
// The arithmetic is essential_math.cuh and two_view_math.cuh (host + device); the conventions are in DESIGN.md section 5.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#include "block_sum.cuh"
#include "essential_math.cuh"
#include "match_common.h"
#include "ransac.cuh"
#include "two_view_math.cuh"
#include "two_view_ransac.h"

namespace {

constexpr int kNormThreads = 64;                     // k_two_view_normalize
constexpr int kHypThreads = 64;                      // k_two_view_hypotheses
constexpr int kScoreWarps = 4;                       // k_two_view_score: hypotheses per CTA, one warp each
constexpr int kScoreThreads = 32 * kScoreWarps;
constexpr int kRefineThreads = ovs::kBlockSumThreads;   // k_two_view_refine: one CTA per problem

// A model policy holds the model's inputs and gives the kernels:
//   kMinSet                   the minimal set (also the fewest inliers of a valid solution)
//   Pairs problem(b, o)       the match view of problem b, whose matches start at o
//   Check check(M)            the per-match test at model M: check(P, i, score) is true for an inlier and adds its terms to score
//   solve(b, P, idx, S, out)  the model (row-major 3 x 3) on the matches idx[0 .. S.n) of P, sums by the policy S

// E_21 on bearing pairs (essential_math.cuh).
struct EssentialModel {
    static constexpr int kMinSet = ovs::kEssMinSet;
    using Pairs = ovs::EssPairs;
    const double* bear_1; const double* bear_2;      // per match, or per keypoint when pairs is set
    const int* pairs;                                // null, or 2 per match (index into bear_1, index into bear_2)
    struct Check {
        double E[9];
        __device__ bool operator()(const Pairs& P, int i, double& score) const { return ovs::essential_check(E, P.b1(i), P.b2(i), score); }
    };
    __device__ Pairs problem(int, int o) const {
        if (pairs) return Pairs{bear_1, bear_2, pairs + 2 * (size_t)o};
        return Pairs{bear_1 + 3 * (size_t)o, bear_2 + 3 * (size_t)o, nullptr};
    }
    __device__ Check check(const double* M) const {
        Check c;
        for (int m = 0; m < 9; ++m) c.E[m] = M[m];
        return c;
    }
    template <class Sum> __device__ void solve(int, const Pairs& P, const int* idx, const Sum& S, double* out) const {
        ovs::essential_from_pairs(P, idx, S, out);
    }
};

// The keypoints of both views and their normalisation (k_two_view_normalize).
struct TwoViewPoints {
    const int* koff_1; const int* koff_2;            // B + 1 keypoint offsets per view
    const float* kp_1; const float* kp_2;            // x, y per keypoint
    float* np_1; float* np_2;                        // normalised x, y per keypoint
    ovs::TwoViewNorm* norm;                          // B x 2 (view 1, view 2)
};

// H_21 or F_21 on keypoint matches (two_view_math.cuh).
template <int Model>
struct TwoViewModel : TwoViewPoints {
    static constexpr int kMinSet = ovs::kTwoViewMinSet;
    using Pairs = ovs::TwoViewPairs;
    const int* pairs;                                // 2 per match: keypoint of view 1, keypoint of view 2 (problem-local)
    double inv_sigma_sq;
    struct Check {
        ovs::TwoViewCheck<Model> chk;
        double iss;
        __device__ bool operator()(const Pairs& P, int i, double& score) const { return chk(P.k1(i), P.k2(i), iss, score); }
    };
    __device__ Pairs problem(int b, int o) const {
        const size_t k1 = 2 * (size_t)koff_1[b], k2 = 2 * (size_t)koff_2[b];
        return Pairs{kp_1 + k1, kp_2 + k2, np_1 + k1, np_2 + k2, pairs + 2 * (size_t)o};
    }
    __device__ Check check(const double* M) const { return Check{ovs::TwoViewCheck<Model>(M), inv_sigma_sq}; }
    template <class Sum> __device__ void solve(int b, const Pairs& P, const int* idx, const Sum& S, double* out) const {
        ovs::two_view_solve<Model>(P, idx, S, norm[2 * b], norm[2 * b + 1], out);
    }
};

template <class Model>
struct Args {
    int B, H, recompute;
    const int* off;                                  // B + 1 match offsets
    const uint64_t* seed;                            // B
    Model model;
    double* hyp;                                     // B x H x 9: every hypothesis's model
    double* hscore; int* hcount;                     // B x H
    int* cidx;                                       // per match: the best hypothesis's inliers, compacted per problem
    double* M; double* score; int* num_inliers; int* best_iter; uint8_t* valid; uint8_t* inlier;   // out
};

__global__ void __launch_bounds__(kNormThreads) k_two_view_normalize(int B, const int* moff, TwoViewPoints V) {
    const int g = blockIdx.x * kNormThreads + threadIdx.x;
    if (g >= 2 * B) return;
    const int b = g >> 1, view = g & 1;
    if (moff[b + 1] - moff[b] < ovs::kTwoViewMinSet) return;   // no hypothesis reads it
    const int* koff = view ? V.koff_2 : V.koff_1;
    const size_t o = 2 * (size_t)koff[b];
    V.norm[g] = ovs::two_view_normalize((view ? V.kp_2 : V.kp_1) + o, koff[b + 1] - koff[b], (view ? V.np_2 : V.np_1) + o);
}

template <class Model>
__global__ void __launch_bounds__(kHypThreads) k_two_view_hypotheses(Args<Model> A) {
    const size_t g = (size_t)blockIdx.x * kHypThreads + threadIdx.x;
    if (g >= (size_t)A.B * (size_t)A.H) return;
    const int b = (int)(g / (size_t)A.H), k = (int)(g % (size_t)A.H);
    const int o = A.off[b], n = A.off[b + 1] - o;
    if (n < Model::kMinSet) return;
    int idx[Model::kMinSet];
    ovs::ransac_sample<Model::kMinSet>(A.seed[b], k, n, idx);
    A.model.solve(b, A.model.problem(b, o), idx, ovs::PnpSeqSum{Model::kMinSet}, A.hyp + 9 * g);
}

// grid (hypothesis blocks, problems), one warp per hypothesis: its score and count.  The selection is the sequential loop's
// rule, applied in k order by k_two_view_refine, so no atomics are needed here.
template <class Model>
__global__ void __launch_bounds__(kScoreThreads) k_two_view_score(Args<Model> A) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const int k = blockIdx.x * kScoreWarps + warp;
    if (n < Model::kMinSet || k >= A.H) return;
    const size_t g = (size_t)b * A.H + k;
    double M[9];
    for (int m = 0; m < 9; ++m) M[m] = A.hyp[9 * g + m];
    const typename Model::Check chk = A.model.check(M);
    const typename Model::Pairs P = A.model.problem(b, o);
    double score;
    const int cnt = ovs::warp_score(n, lane, [=](int i, double& part) { return chk(P, i, part); }, &score);
    if (lane == 0) { A.hscore[g] = score; A.hcount[g] = cnt; }
}

// One CTA per problem: the best hypothesis (the first whose score is strictly greater than the best so far, which starts at 0;
// a NaN score never wins), its flags and `valid` = (best score > 0 and at least kMinSet inliers); with recompute and valid, the
// model solved again on the compacted inliers (index order, CTA-wide sums) and its flags, count and score.
template <class Model>
__global__ void __launch_bounds__(kRefineThreads) k_two_view_refine(Args<Model> A) {
    __shared__ double s_red[ovs::kBlockSumChunk * kRefineThreads];
    __shared__ double s_res[45];
    __shared__ int s_warp[kRefineThreads / 32];
    __shared__ int s_best;
    __shared__ double s_score;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    if (t == 0) {
        int best = -1;
        double bs = 0.0;
        if (n >= Model::kMinSet)
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
    const bool valid = score > 0.0 && cnt >= Model::kMinSet;
    int num = cnt;
    double dummy = 0.0;
    if (best < 0) {
        for (int i = t; i < n; i += kRefineThreads) A.inlier[o + i] = 0;
    } else {
        const typename Model::Pairs P = A.model.problem(b, o);
        {
            const typename Model::Check chk = A.model.check(M);
            for (int i = t; i < n; i += kRefineThreads) A.inlier[o + i] = chk(P, i, dummy) ? 1 : 0;
        }
        if (valid && A.recompute) {
            __syncthreads();   // the flags above are read back below
            ovs::cta_compact<kRefineThreads>(n, A.cidx + o, s_warp, [&](int i) { return A.inlier[o + i] != 0; });
            A.model.solve(b, P, A.cidx + o, ovs::PnpBlockSum{cnt, s_red, s_res}, M);
            const typename Model::Check chk = A.model.check(M);
            int c2 = 0;
            for (int base = 0; base < n; base += kRefineThreads) {
                const int i = base + t;
                const bool f = i < n && chk(P, i, dummy);
                if (i < n) A.inlier[o + i] = f ? 1 : 0;
                c2 += __syncthreads_count(f);
            }
            num = c2;
            if (warp == 0) {
                double sc;
                ovs::warp_score(n, lane, [=](int i, double& part) { return chk(P, i, part); }, &sc);
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

// Point a solve's arguments at its carved outputs and scratch.
template <class Model>
void bind(Args<Model>& A, const ovs::SolveOut& o, const ovs::SolveScratch& s) {
    A.M = o.M; A.score = o.score; A.num_inliers = o.num; A.best_iter = o.best; A.valid = o.valid; A.inlier = o.inlier;
    A.hyp = s.hyp; A.hscore = s.hyp_score; A.hcount = s.hyp_count; A.cidx = s.cidx;
    if constexpr (!std::is_same<Model, EssentialModel>::value) { A.model.np_1 = s.np_1; A.model.np_2 = s.np_2; A.model.norm = s.norm; }
}

// A solve's outputs and scratch, carved after its inputs.
template <class Model>
void carve_results(ovs::Staging& S, Args<Model>& A, ovs::SolveOut& o, size_t N, size_t K1, size_t K2) {
    ovs::SolveScratch s;
    ovs::carve_solve_out(S, o, (size_t)A.B, N);
    ovs::carve_solve_scratch(S, s, (size_t)A.B, (size_t)A.H, N, K1, K2);
    bind(A, o, s);
}

// The launches of a staged solve.
template <class Model>
int enqueue(cudaStream_t st, const Args<Model>& A) {
    if (A.H > 0) {
        if constexpr (!std::is_same<Model, EssentialModel>::value) {
            k_two_view_normalize<<<(2 * A.B + kNormThreads - 1) / kNormThreads, kNormThreads, 0, st>>>(A.B, A.off, A.model);
            OVS_LAUNCH_CHECK();
        }
        const size_t hyp_threads = (size_t)A.B * (size_t)A.H;
        k_two_view_hypotheses<Model><<<(unsigned)((hyp_threads + kHypThreads - 1) / kHypThreads), kHypThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
        k_two_view_score<Model><<<dim3((A.H + kScoreWarps - 1) / kScoreWarps, A.B), kScoreThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
    }
    k_two_view_refine<Model><<<A.B, kRefineThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    return OVS_OK;
}

// A staged solve: the upload, the launches, the copy back and the host outputs (M_21 ... per problem, inlier_out per match).
template <class Model>
int launch_and_fetch(cudaStream_t st, const ovs::Staging& S, const Args<Model>& A, const ovs::SolveOut& o, size_t N, double* M_21,
                     uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score, uint8_t* inlier_out) {
    const size_t NB = (size_t)A.B;
    OVS_CUDA_CHECK(S.upload(st));
    int rc = enqueue(st, A);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(M_21, o.hM, 9 * 8 * NB); memcpy(best_score, o.hscore, 8 * NB);
    memcpy(num_inliers, o.hnum, 4 * NB); memcpy(best_iter, o.hbest, 4 * NB); memcpy(valid, o.hvalid, NB);
    if (N) memcpy(inlier_out, o.hinlier, N);
    return OVS_OK;
}

// The bearings of an essential solve: host arrays (uploaded with the other inputs) or device arrays (read in place).
struct EssBearings {
    const double* b1; size_t n1;
    const double* b2; size_t n2;
    bool on_device;
};

// One batched essential solve on the matcher's essential arenas.  off: host, B + 1 offsets of N = off[B] matches; pairs: host,
// 2 per match or null; outputs: host.  E / score / num_inliers / best_iter / valid per problem, inlier_out per match.
int essential_run(ovs_matcher* h, int B, const int32_t* off, const int32_t* pairs, const EssBearings& bear, int max_num_iter,
                  int recompute, const uint64_t* seeds, double* E_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter,
                  double* best_score, uint8_t* inlier_out) {
    const size_t N = (size_t)off[B], NB = (size_t)B;
    const size_t np = pairs ? 2 * N : 0;
    Args<EssentialModel> A{};
    A.B = B; A.H = max_num_iter; A.recompute = recompute ? 1 : 0;
    int* hoff; uint64_t* hseed; int* hpairs = nullptr; double* hb1 = nullptr; double* hb2 = nullptr;
    ovs::SolveOut r;
    ovs::Staging S;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = ovs::stage(S, h->h_ess, h->h_ess_cap, h->d_ess, h->d_ess_cap, [&](ovs::Staging& S) {
        A.off = S.in(hoff, NB + 1); A.seed = S.in(hseed, NB);
        A.model.pairs = pairs ? S.in(hpairs, np) : nullptr;
        if (bear.on_device) { A.model.bear_1 = bear.b1; A.model.bear_2 = bear.b2; }
        else { A.model.bear_1 = S.in(hb1, 3 * bear.n1); A.model.bear_2 = S.in(hb2, 3 * bear.n2); }
        carve_results(S, A, r, N, 0, 0);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hoff, off, 4 * (NB + 1)); memcpy(hseed, seeds, 8 * NB);
    if (pairs) memcpy(hpairs, pairs, 4 * np);
    if (!bear.on_device) {
        if (bear.n1) memcpy(hb1, bear.b1, 24 * bear.n1);
        if (bear.n2) memcpy(hb2, bear.b2, 24 * bear.n2);
    }
    return launch_and_fetch(h->stream, S, A, r, N, E_21, valid, num_inliers, best_iter, best_score, inlier_out);
}

// One batched homography or fundamental-matrix solve on the matcher's two-view arenas.  All arrays are host arrays, already
// validated.
template <int Model>
int two_view_run(ovs_matcher* h, int B, const int32_t* koff_1, const ovs_keypoint* keypts_1, const int32_t* koff_2,
                 const ovs_keypoint* keypts_2, const int32_t* moff, const int32_t* matches_12, float sigma, int max_num_iter, int recompute,
                 const uint64_t* seeds, double* M_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                 uint8_t* inlier_out) {
    const size_t N = (size_t)moff[B], K1 = (size_t)koff_1[B], K2 = (size_t)koff_2[B], NB = (size_t)B;
    Args<TwoViewModel<Model>> A{};
    A.B = B; A.H = max_num_iter; A.recompute = recompute ? 1 : 0;
    A.model.inv_sigma_sq = (double)ovs::two_view_inv_sigma_sq(sigma);
    int *hmoff, *hk1, *hk2, *hpairs; uint64_t* hseed; float *hkp1, *hkp2;
    ovs::SolveOut r;
    ovs::Staging S;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = ovs::stage(S, h->h_tv, h->h_tv_cap, h->d_tv, h->d_tv_cap, [&](ovs::Staging& S) {
        TwoViewModel<Model>& m = A.model;
        A.off = S.in(hmoff, NB + 1); m.koff_1 = S.in(hk1, NB + 1); m.koff_2 = S.in(hk2, NB + 1);
        A.seed = S.in(hseed, NB); m.pairs = S.in(hpairs, 2 * N);
        m.kp_1 = S.in(hkp1, 2 * K1); m.kp_2 = S.in(hkp2, 2 * K2);
        carve_results(S, A, r, N, K1, K2);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hmoff, moff, 4 * (NB + 1)); memcpy(hk1, koff_1, 4 * (NB + 1)); memcpy(hk2, koff_2, 4 * (NB + 1));
    memcpy(hseed, seeds, 8 * NB); memcpy(hpairs, matches_12, 8 * N);
    for (size_t i = 0; i < K1; ++i) { hkp1[2 * i] = keypts_1[i].x; hkp1[2 * i + 1] = keypts_1[i].y; }
    for (size_t i = 0; i < K2; ++i) { hkp2[2 * i] = keypts_2[i].x; hkp2[2 * i + 1] = keypts_2[i].y; }
    return launch_and_fetch(h->stream, S, A, r, N, M_21, valid, num_inliers, best_iter, best_score, inlier_out);
}

// A batch without any match: no hypothesis, every problem invalid.
void no_match_results(int B, double* M_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score) {
    for (int b = 0; b < B; ++b) {
        for (int k = 0; k < 9; ++k) M_21[9 * (size_t)b + k] = 0.0;
        valid[b] = 0; num_inliers[b] = 0; best_iter[b] = -1; best_score[b] = 0.0;
    }
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
    if ((rc = ovs::check_offsets(keypt_offsets_1, B, "keypt_offsets_1")) != OVS_OK) return rc;
    if ((rc = ovs::check_offsets(keypt_offsets_2, B, "keypt_offsets_2")) != OVS_OK) return rc;
    if ((rc = ovs::check_offsets(match_offsets, B, "match_offsets")) != OVS_OK) return rc;
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
    if (n_all == 0) {
        no_match_results(B, M_21, valid, num_inliers, best_iter, best_score);
        return OVS_OK;
    }
    return two_view_run<Model>(h, B, keypt_offsets_1, keypts_1, keypt_offsets_2, keypts_2, match_offsets, matches_12, sigma, max_num_iter,
                               recompute, seeds, M_21, valid, num_inliers, best_iter, best_score, inlier_out);
}

}  // namespace

namespace ovs {

void carve_solve_out(Staging& S, SolveOut& o, size_t NB, size_t N) {
    o.M = S.out(o.hM, 9 * NB); o.score = S.out(o.hscore, NB); o.num = S.out(o.hnum, NB); o.best = S.out(o.hbest, NB);
    o.valid = S.out(o.hvalid, NB); o.inlier = S.out(o.hinlier, N);
}

void carve_solve_scratch(Staging& S, SolveScratch& s, size_t NB, size_t H, size_t N, size_t K1, size_t K2) {
    s.hyp = S.dev<double>(9 * NB * H); s.hyp_score = S.dev<double>(NB * H); s.hyp_count = S.dev<int>(NB * H); s.cidx = S.dev<int>(N);
    s.np_1 = s.np_2 = nullptr; s.norm = nullptr;
    if (K1 + K2) { s.np_1 = S.dev<float>(2 * K1); s.np_2 = S.dev<float>(2 * K2); s.norm = S.dev<TwoViewNorm>(2 * NB); }
}

namespace {
template <int Model>
int enqueue_keypoint_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s, float sigma) {
    Args<TwoViewModel<Model>> A{};
    A.B = in.B; A.H = in.H; A.recompute = in.recompute; A.off = in.off; A.seed = in.seed;
    TwoViewModel<Model>& m = A.model;
    m.koff_1 = in.koff_1; m.koff_2 = in.koff_2; m.kp_1 = in.kp_1; m.kp_2 = in.kp_2; m.pairs = in.pairs;
    m.inv_sigma_sq = (double)two_view_inv_sigma_sq(sigma);
    bind(A, o, s);
    return enqueue(st, A);
}
}  // namespace

int enqueue_homography_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s, float sigma) {
    return enqueue_keypoint_solve<kTwoViewH>(st, in, o, s, sigma);
}

int enqueue_fundamental_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s, float sigma) {
    return enqueue_keypoint_solve<kTwoViewF>(st, in, o, s, sigma);
}

int enqueue_essential_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s) {
    Args<EssentialModel> A{};
    A.B = in.B; A.H = in.H; A.recompute = in.recompute; A.off = in.off; A.seed = in.seed;
    A.model.bear_1 = in.bear_1; A.model.bear_2 = in.bear_2; A.model.pairs = nullptr;
    bind(A, o, s);
    return enqueue(st, A);
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

}  // namespace ovs

extern "C" int ovs_essential_solve_ransac_host(ovs_matcher* h, int B, const int32_t* match_offsets, const double* bearings_1,
                                               const double* bearings_2, int max_num_iter, int recompute, const uint64_t* seeds,
                                               double* E_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                               uint8_t* inlier_out) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(max_num_iter >= 0, OVS_ERR_INVALID_ARG, "max_num_iter must not be negative");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(match_offsets && seeds && E_21 && valid && num_inliers && best_iter && best_score, OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    if ((rc = ovs::check_offsets(match_offsets, B, "match_offsets")) != OVS_OK) return rc;
    const int n_all = match_offsets[B];
    OVS_REQUIRE(n_all == 0 || (bearings_1 && bearings_2 && inlier_out), OVS_ERR_INVALID_ARG, "null argument");
    if ((rc = ovs::check_bearings(bearings_1, n_all, "bearings_1 of match")) != OVS_OK) return rc;
    if ((rc = ovs::check_bearings(bearings_2, n_all, "bearings_2 of match")) != OVS_OK) return rc;
    if (n_all == 0) {
        no_match_results(B, E_21, valid, num_inliers, best_iter, best_score);
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
    if ((rc = ovs::check_bearings(bearings_frm, n1, "bearing of frame keypoint")) != OVS_OK) return rc;
    if ((rc = ovs::check_bearings(bearings_keyfrm, n2, "bearing of keyframe keypoint")) != OVS_OK) return rc;
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
