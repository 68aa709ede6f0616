// initializer.cu -- monocular map initialisation on the device: initialize::perspective::initialize (H and F) and
// initialize::bearing_vector::initialize (E), each for a batch of independent problems, from the matches to the triangulated
// points in one call.  The solves are two_view_ransac.cu's, enqueued on this call's buffers (two_view_ransac.h); the arithmetic
// after them is initializer_math.cuh.  Five launches after the solves, whatever B and whichever model each problem takes:
//   k_init_setup    one thread per problem: the model choice, the decomposition into the hypothesis table (8 or 4 (R, t))
//   k_init_check    one thread per (match, hypothesis, problem): check_pose's test of one inlier match -> the order-preserving
//                   key of its cos_parallax, or kInitNoKey when it is not valid
//   k_init_select   one CTA per (hypothesis, problem): the valid count n and the min(50, n - 1)-th smallest key by an exact
//                   4-pass radix select (8 bits a pass, shared-memory integer histograms)
//   k_init_choose   one thread per problem: find_most_plausible_pose, the status and the chosen (R, t)
//   k_init_points   one thread per reference keypoint: the chosen hypothesis's point, recomputed by the same function
//                   (the same bits), or zeros; every entry is written
// No float atomics: the results do not depend on the schedule.
#include <cmath>
#include <cstring>
#include <vector>

#include "initializer_math.cuh"
#include "match_common.h"
#include "ransac.cuh"
#include "two_view_ransac.h"

namespace {

constexpr int kProbThreads = 64;                     // k_init_setup, k_init_choose
constexpr int kCheckThreads = 128;                   // k_init_check
constexpr int kSelectThreads = 256;                  // k_init_select
constexpr int kPointThreads = 128;                   // k_init_points
constexpr int kStatusPending = -1;                   // a problem with hypotheses, before k_init_choose
constexpr int kMaxItems = (1 << 28) - 1;             // keypoints per side and matches per call: 8 keys per match fit an int

struct InitArgs {
    int B, perspective, min_num_triangulated;
    double cos_thr, reproj_err_thr_sq;
    const int* moff;                                 // B + 1 match offsets
    const int* roff;                                 // B + 1 reference keypoint offsets
    const ovs::CameraD* cam;                         // 2 per problem: reference, current
    const double* bear_ref; const double* bear_cur;  // 3 per match
    const float* kpm;                                // 4 per match: reference x, y, current x, y
    const int* ref_match;                            // per reference keypoint: its match (call-wide index) or -1
    ovs::SolveOut s0, s1;                            // perspective: H, F; bearing_vector: E, unused
    double* hyp_R; double* hyp_t;                    // B x 8 x 9, B x 8 x 3
    unsigned* keys;                                  // 8 per match: problem o's keys at 8 o + h n + i
    ovs_init_result* res;                            // per problem
    uint8_t* flag; double* pts;                      // per reference keypoint
};

__device__ const uint8_t* inlier_flags(const InitArgs& A, int model) { return model == OVS_INIT_MODEL_F ? A.s1.inlier : A.s0.inlier; }

__device__ void load_hyp(const InitArgs& A, int b, int h, double* Rt) {
    const size_t g = (size_t)b * ovs::kInitMaxHyp + h;
    for (int k = 0; k < 9; ++k) Rt[k] = A.hyp_R[9 * g + k];
    for (int k = 0; k < 3; ++k) Rt[9 + k] = A.hyp_t[3 * g + k];
}

__device__ int check_match(const InitArgs& A, int b, const double* Rt, int m, double* p, float* cp) {
    return ovs::init_check_match(Rt, A.cam[2 * b], A.cam[2 * b + 1], A.bear_ref + 3 * (size_t)m, A.bear_cur + 3 * (size_t)m,
                                 A.kpm + 4 * (size_t)m, A.kpm + 4 * (size_t)m + 2, A.reproj_err_thr_sq, A.perspective != 0, p, cp);
}

__global__ void __launch_bounds__(kProbThreads) k_init_setup(InitArgs A) {
    const int b = blockIdx.x * kProbThreads + threadIdx.x;
    if (b >= A.B) return;
    int model = OVS_INIT_MODEL_NONE;
    if (A.perspective) {
        const double sH = A.s0.score[b], sF = A.s1.score[b];
        if (ovs::kInitRelScoreH < sH / (sH + sF) && A.s0.valid[b]) model = OVS_INIT_MODEL_H;
        else if (A.s1.valid[b]) model = OVS_INIT_MODEL_F;
    } else if (A.s0.valid[b]) {
        model = OVS_INIT_MODEL_E;
    }
    int nh = 0, status = OVS_INIT_NO_VALID_MODEL;
    double* R = A.hyp_R + 9 * (size_t)b * ovs::kInitMaxHyp;
    double* t = A.hyp_t + 3 * (size_t)b * ovs::kInitMaxHyp;
    if (model == OVS_INIT_MODEL_H) {
        const bool ok = ovs::decompose_homography(A.s0.M + 9 * (size_t)b, A.cam[2 * b], A.cam[2 * b + 1], R, t, nullptr);
        nh = ok ? 8 : 0;
        status = ok ? kStatusPending : OVS_INIT_DECOMPOSITION_REFUSED;
    } else if (model == OVS_INIT_MODEL_F) {
        ovs::decompose_fundamental(A.s1.M + 9 * (size_t)b, A.cam[2 * b], A.cam[2 * b + 1], R, t);
        nh = 4; status = kStatusPending;
    } else if (model == OVS_INIT_MODEL_E) {
        ovs::decompose_essential(A.s0.M + 9 * (size_t)b, R, t);
        nh = 4; status = kStatusPending;
    }
    ovs_init_result& r = A.res[b];
    r.status = status; r.model = model; r.num_hypotheses = nh;
}

// grid (match blocks, 8, B)
__global__ void __launch_bounds__(kCheckThreads) k_init_check(InitArgs A) {
    const int b = blockIdx.z, h = blockIdx.y, i = blockIdx.x * kCheckThreads + threadIdx.x;
    const int o = A.moff[b], n = A.moff[b + 1] - o;
    if (i >= n) return;
    unsigned key = ovs::kInitNoKey;
    const ovs_init_result& r = A.res[b];
    if (h < r.num_hypotheses && inlier_flags(A, r.model)[o + i]) {
        double Rt[12], p[3];
        float cp;
        load_hyp(A, b, h, Rt);
        const int code = check_match(A, b, Rt, o + i, p, &cp);
        if (code == ovs::kInitValid || code == ovs::kInitValidSmall) key = ovs::init_key(cp);
    }
    A.keys[8 * (size_t)o + (size_t)h * n + i] = key;
}

// grid (8, B): the count of valid keys and the key of rank min(50, n - 1) among them.  Every valid key is below kInitNoKey and
// the rank is below the count, so the select runs over all n keys of the hypothesis.
__global__ void __launch_bounds__(kSelectThreads) k_init_select(InitArgs A) {
    __shared__ int s_hist[256];
    __shared__ int s_digit, s_rank;
    const int b = blockIdx.y, h = blockIdx.x, t = threadIdx.x;
    const int o = A.moff[b], n = A.moff[b + 1] - o;
    ovs_init_result& r = A.res[b];
    const unsigned* keys = A.keys + 8 * (size_t)o + (size_t)h * n;
    int cnt = 0;
    if (h < r.num_hypotheses)
        for (int base = 0; base < n; base += kSelectThreads) {
            const int i = base + t;
            cnt += __syncthreads_count(i < n && keys[i] != ovs::kInitNoKey);
        }
    if (cnt == 0) {
        if (t == 0) { r.num_valid[h] = 0; r.cos_parallax[h] = 1.0f; }
        return;
    }
    int rank = ovs::init_parallax_rank(cnt);
    unsigned prefix = 0, mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        s_hist[t] = 0;
        __syncthreads();
        for (int i = t; i < n; i += kSelectThreads) {
            const unsigned k = keys[i];
            if ((k & mask) == prefix) atomicAdd(&s_hist[(k >> shift) & 255u], 1);
        }
        __syncthreads();
        if (t == 0) {
            int c = 0;
            while (rank >= s_hist[c]) rank -= s_hist[c++];
            s_digit = c; s_rank = rank;
        }
        __syncthreads();
        prefix |= (unsigned)s_digit << shift;
        mask |= 255u << shift;
        rank = s_rank;
        __syncthreads();
    }
    if (t == 0) { r.num_valid[h] = cnt; r.cos_parallax[h] = ovs::init_key_value(prefix); }
}

__global__ void __launch_bounds__(kProbThreads) k_init_choose(InitArgs A) {
    const int b = blockIdx.x * kProbThreads + threadIdx.x;
    if (b >= A.B) return;
    ovs_init_result& r = A.res[b];
    int best = -1;
    if (r.status == kStatusPending) r.status = ovs::init_choose(r.num_hypotheses, r.num_valid, r.cos_parallax, A.min_num_triangulated, A.cos_thr, &best);
    r.chosen = best;
    double Rt[12];
    if (r.status == OVS_INIT_OK) load_hyp(A, b, best, Rt);
    for (int k = 0; k < 9; ++k) r.rot_ref_to_cur[k] = r.status == OVS_INIT_OK ? Rt[k] : 0.0;
    for (int k = 0; k < 3; ++k) r.trans_ref_to_cur[k] = r.status == OVS_INIT_OK ? Rt[9 + k] : 0.0;
}

__global__ void __launch_bounds__(kPointThreads) k_init_points(InitArgs A, int K) {
    const int g = blockIdx.x * kPointThreads + threadIdx.x;
    if (g >= K) return;
    int lo = 0, hi = A.B;                            // the problem b with roff[b] <= g < roff[b + 1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) / 2;
        if (A.roff[mid] <= g) lo = mid; else hi = mid;
    }
    const int b = lo, m = A.ref_match[g];
    const ovs_init_result& r = A.res[b];
    double p[3] = {0.0, 0.0, 0.0};
    bool tri = false;
    if (r.status == OVS_INIT_OK && m >= 0 && inlier_flags(A, r.model)[m]) {
        double Rt[12];
        float cp;
        load_hyp(A, b, r.chosen, Rt);
        tri = check_match(A, b, Rt, m, p, &cp) == ovs::kInitValid;
    }
    A.flag[g] = tri ? 1 : 0;
    for (int k = 0; k < 3; ++k) A.pts[3 * (size_t)g + k] = tri ? p[k] : 0.0;
}

ovs::CameraD camera_d(const ovs_camera& c) {
    return ovs::CameraD{c.model, c.fx, c.fy, c.cx, c.cy, c.focal_x_baseline, c.cols, c.rows};
}

int check_view(const ovs_init_view& v, bool perspective, const char* what, int b) {
    const ovs_camera& c = v.camera;
    if (perspective)
        OVS_REQUIRE(c.model == OVS_CAMERA_PERSPECTIVE && std::isfinite(c.fx) && c.fx > 0.0 && std::isfinite(c.fy) && c.fy > 0.0 &&
                    std::isfinite(c.cx) && std::isfinite(c.cy), OVS_ERR_INVALID_ARG,
                    "%s view of problem %d: a perspective camera with positive finite fx, fy and finite cx, cy is required", what, b);
    else
        OVS_REQUIRE(c.model == OVS_CAMERA_EQUIRECTANGULAR && std::isfinite(c.cols) && c.cols > 0.0 && std::isfinite(c.rows) && c.rows > 0.0,
                    OVS_ERR_INVALID_ARG, "%s view of problem %d: an equirectangular camera with positive finite cols, rows is required", what, b);
    OVS_REQUIRE(v.num_keypts >= 0, OVS_ERR_INVALID_ARG, "%s view of problem %d: negative num_keypts", what, b);
    if (v.num_keypts == 0) return OVS_OK;
    OVS_REQUIRE(v.undist_keypts && v.bearings, OVS_ERR_INVALID_ARG, "%s view of problem %d: null keypoint or bearing array", what, b);
    for (int i = 0; i < v.num_keypts; ++i)
        OVS_REQUIRE(std::isfinite(v.undist_keypts[i].x) && std::isfinite(v.undist_keypts[i].y), OVS_ERR_INVALID_ARG,
                    "keypoint %d of the %s view of problem %d is not finite", i, what, b);
    return ovs::check_bearings(v.bearings, v.num_keypts, what[0] == 'r' ? "bearing of a reference keypoint" : "bearing of a current keypoint");
}

// The call with no launch (B == 0 or no match): every problem without a valid model.
void no_match_results(int B, ovs_init_result* results, size_t K1, uint8_t* is_triangulated, double* triangulated_pts) {
    for (int b = 0; b < B; ++b) {
        ovs_init_result& r = results[b];
        memset(&r, 0, sizeof(r));
        r.status = OVS_INIT_NO_VALID_MODEL; r.model = OVS_INIT_MODEL_NONE; r.chosen = -1;
        for (int h = 0; h < ovs::kInitMaxHyp; ++h) r.cos_parallax[h] = 1.0f;
    }
    if (K1) { memset(is_triangulated, 0, K1); memset(triangulated_pts, 0, 24 * K1); }
}

int initialize(ovs_matcher* h, bool perspective, int B, const ovs_init_view* ref_views, const ovs_init_view* cur_views,
               const int32_t* ref_matches_with_cur, int num_ransac_iters, int min_num_triangulated, float parallax_deg_thr,
               float reproj_err_thr_sq, const uint64_t* seeds, ovs_init_result* results, uint8_t* is_triangulated,
               double* triangulated_pts) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(num_ransac_iters >= 0 && min_num_triangulated >= 0, OVS_ERR_INVALID_ARG,
                "num_ransac_iters and min_num_triangulated must not be negative");
    OVS_REQUIRE(parallax_deg_thr >= 0.0f && parallax_deg_thr <= 180.0f, OVS_ERR_INVALID_ARG, "parallax_deg_thr must be in 0 .. 180");
    OVS_REQUIRE(std::isfinite(reproj_err_thr_sq) && reproj_err_thr_sq >= 0.0f, OVS_ERR_INVALID_ARG,
                "reproj_err_thr_sq must be finite and not negative");
    OVS_REQUIRE((size_t)B * (size_t)num_ransac_iters <= (size_t)INT32_MAX, OVS_ERR_UNSUPPORTED,
                "B x num_ransac_iters above 2^31 - 1");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(ref_views && cur_views && seeds && results, OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    size_t K1 = 0, K2 = 0, N = 0;
    for (int b = 0; b < B; ++b) {
        if ((rc = check_view(ref_views[b], perspective, "reference", b)) != OVS_OK) return rc;
        if ((rc = check_view(cur_views[b], perspective, "current", b)) != OVS_OK) return rc;
        K1 += (size_t)ref_views[b].num_keypts; K2 += (size_t)cur_views[b].num_keypts;
    }
    OVS_REQUIRE(K1 <= (size_t)kMaxItems && K2 <= (size_t)kMaxItems, OVS_ERR_UNSUPPORTED, "2^28 or more keypoints of one side in one call");
    OVS_REQUIRE(K1 == 0 || (ref_matches_with_cur && is_triangulated && triangulated_pts), OVS_ERR_INVALID_ARG, "null argument");
    {
        size_t g = 0;
        for (int b = 0; b < B; ++b)
            for (int r = 0; r < ref_views[b].num_keypts; ++r, ++g) {
                const int c = ref_matches_with_cur[g];
                OVS_REQUIRE(c >= -1 && c < cur_views[b].num_keypts, OVS_ERR_INVALID_ARG,
                            "ref_matches_with_cur[%d] of problem %d is %d: not -1 or a keypoint of the current view", r, b, c);
                N += c >= 0 ? 1 : 0;
            }
    }
    OVS_REQUIRE(N <= (size_t)kMaxItems, OVS_ERR_UNSUPPORTED, "2^28 or more matches in one call");
    if (N == 0) {
        no_match_results(B, results, K1, is_triangulated, triangulated_pts);
        return OVS_OK;
    }
    const double cos_thr = std::cos((double)parallax_deg_thr / 180.0 * M_PI);
    const size_t NB = (size_t)B, H = (size_t)num_ransac_iters;

    ovs::SolveInputs in{};
    in.B = B; in.H = num_ransac_iters; in.recompute = 1;
    InitArgs A{};
    A.B = B; A.perspective = perspective ? 1 : 0; A.min_num_triangulated = min_num_triangulated;
    A.cos_thr = cos_thr; A.reproj_err_thr_sq = (double)reproj_err_thr_sq;
    int *hmoff, *hroff, *hrm, *hk1 = nullptr, *hk2 = nullptr, *hpairs = nullptr;
    uint64_t* hseed; ovs::CameraD* hcam; double *hb1, *hb2; float *hkpm, *hkp1 = nullptr, *hkp2 = nullptr;
    ovs_init_result* hres; uint8_t* hflag; double* hpts;
    ovs::SolveScratch sc0, sc1;
    ovs::Staging S;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    rc = ovs::stage(S, h->h_init, h->h_init_cap, h->d_init, h->d_init_cap, [&](ovs::Staging& S) {
        A.moff = in.off = S.in(hmoff, NB + 1); in.seed = S.in(hseed, NB);
        A.roff = S.in(hroff, NB + 1); A.ref_match = S.in(hrm, K1); A.cam = S.in(hcam, 2 * NB);
        A.bear_ref = in.bear_1 = S.in(hb1, 3 * N); A.bear_cur = in.bear_2 = S.in(hb2, 3 * N); A.kpm = S.in(hkpm, 4 * N);
        if (perspective) {
            in.koff_1 = S.in(hk1, NB + 1); in.koff_2 = S.in(hk2, NB + 1); in.pairs = S.in(hpairs, 2 * N);
            in.kp_1 = S.in(hkp1, 2 * K1); in.kp_2 = S.in(hkp2, 2 * K2);
        }
        ovs::carve_solve_out(S, A.s0, NB, N);
        if (perspective) ovs::carve_solve_out(S, A.s1, NB, N);
        A.res = S.out(hres, NB); A.flag = S.out(hflag, K1); A.pts = S.out(hpts, 3 * K1);
        ovs::carve_solve_scratch(S, sc0, NB, H, N, perspective ? K1 : 0, perspective ? K2 : 0);
        if (perspective) ovs::carve_solve_scratch(S, sc1, NB, H, N, K1, K2);
        A.hyp_R = S.dev<double>(9 * ovs::kInitMaxHyp * NB); A.hyp_t = S.dev<double>(3 * ovs::kInitMaxHyp * NB);
        A.keys = S.dev<unsigned>(ovs::kInitMaxHyp * N);
    });
    if (rc != OVS_OK) return rc;

    // the matches in reference-index order, and what every stage reads of them
    int m = 0;
    size_t g1 = 0, g2 = 0;
    hmoff[0] = 0; hroff[0] = 0;
    if (perspective) { hk1[0] = 0; hk2[0] = 0; }
    for (int b = 0; b < B; ++b) {
        const ovs_init_view& R = ref_views[b];
        const ovs_init_view& Cv = cur_views[b];
        hcam[2 * b] = camera_d(R.camera); hcam[2 * b + 1] = camera_d(Cv.camera);
        hseed[b] = seeds[b];
        for (int r = 0; r < R.num_keypts; ++r) {
            const int c = ref_matches_with_cur[g1 + r];
            hrm[g1 + r] = c >= 0 ? m : -1;
            if (c < 0) continue;
            for (int k = 0; k < 3; ++k) { hb1[3 * (size_t)m + k] = R.bearings[3 * (size_t)r + k]; hb2[3 * (size_t)m + k] = Cv.bearings[3 * (size_t)c + k]; }
            hkpm[4 * (size_t)m] = R.undist_keypts[r].x; hkpm[4 * (size_t)m + 1] = R.undist_keypts[r].y;
            hkpm[4 * (size_t)m + 2] = Cv.undist_keypts[c].x; hkpm[4 * (size_t)m + 3] = Cv.undist_keypts[c].y;
            if (perspective) { hpairs[2 * (size_t)m] = r; hpairs[2 * (size_t)m + 1] = c; }
            ++m;
        }
        if (perspective) {
            for (int i = 0; i < R.num_keypts; ++i) { hkp1[2 * (g1 + i)] = R.undist_keypts[i].x; hkp1[2 * (g1 + i) + 1] = R.undist_keypts[i].y; }
            for (int i = 0; i < Cv.num_keypts; ++i) { hkp2[2 * (g2 + i)] = Cv.undist_keypts[i].x; hkp2[2 * (g2 + i) + 1] = Cv.undist_keypts[i].y; }
        }
        g1 += (size_t)R.num_keypts; g2 += (size_t)Cv.num_keypts;
        hmoff[b + 1] = m; hroff[b + 1] = (int)g1;
        if (perspective) { hk1[b + 1] = (int)g1; hk2[b + 1] = (int)g2; }
    }

    int max_n = 0;
    for (int b = 0; b < B; ++b) max_n = std::max(max_n, hmoff[b + 1] - hmoff[b]);
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    if (perspective) {
        if ((rc = ovs::enqueue_homography_solve(st, in, A.s0, sc0, 1.0f)) != OVS_OK) return rc;
        if ((rc = ovs::enqueue_fundamental_solve(st, in, A.s1, sc1, 1.0f)) != OVS_OK) return rc;
    } else {
        if ((rc = ovs::enqueue_essential_solve(st, in, A.s0, sc0)) != OVS_OK) return rc;
    }
    const unsigned pb = (unsigned)((B + kProbThreads - 1) / kProbThreads);
    k_init_setup<<<pb, kProbThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    k_init_check<<<dim3((max_n + kCheckThreads - 1) / kCheckThreads, ovs::kInitMaxHyp, B), kCheckThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    k_init_select<<<dim3(ovs::kInitMaxHyp, B), kSelectThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    k_init_choose<<<pb, kProbThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    k_init_points<<<(unsigned)((K1 + kPointThreads - 1) / kPointThreads), kPointThreads, 0, st>>>(A, (int)K1);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));

    memcpy(results, hres, sizeof(ovs_init_result) * NB);
    for (int b = 0; b < B; ++b) {
        ovs_init_result& r = results[b];
        const ovs::SolveOut* so[2] = {&A.s0, &A.s1};
        for (int s = 0; s < 2; ++s) {
            const bool has = s == 0 || perspective;
            for (int k = 0; k < 9; ++k) r.solver_M[s][k] = has ? so[s]->hM[9 * (size_t)b + k] : 0.0;
            r.solver_score[s] = has ? so[s]->hscore[b] : 0.0;
            r.solver_num_inliers[s] = has ? so[s]->hnum[b] : 0;
            r.solver_valid[s] = has ? so[s]->hvalid[b] : 0;
        }
        memset(r.reserved, 0, sizeof(r.reserved));
    }
    memcpy(is_triangulated, hflag, K1);
    memcpy(triangulated_pts, hpts, 24 * K1);
    return OVS_OK;
}

}  // namespace

extern "C" int ovs_initialize_perspective_host(ovs_matcher* h, int B, const ovs_init_view* ref_views, const ovs_init_view* cur_views,
                                               const int32_t* ref_matches_with_cur, int num_ransac_iters, int min_num_triangulated,
                                               float parallax_deg_thr, float reproj_err_thr_sq, const uint64_t* seeds,
                                               ovs_init_result* results, uint8_t* is_triangulated, double* triangulated_pts) {
    return initialize(h, true, B, ref_views, cur_views, ref_matches_with_cur, num_ransac_iters, min_num_triangulated, parallax_deg_thr,
                      reproj_err_thr_sq, seeds, results, is_triangulated, triangulated_pts);
}

extern "C" int ovs_initialize_bearing_vector_host(ovs_matcher* h, int B, const ovs_init_view* ref_views, const ovs_init_view* cur_views,
                                                  const int32_t* ref_matches_with_cur, int num_ransac_iters, int min_num_triangulated,
                                                  float parallax_deg_thr, float reproj_err_thr_sq, const uint64_t* seeds,
                                                  ovs_init_result* results, uint8_t* is_triangulated, double* triangulated_pts) {
    return initialize(h, false, B, ref_views, cur_views, ref_matches_with_cur, num_ransac_iters, min_num_triangulated, parallax_deg_thr,
                      reproj_err_thr_sq, seeds, results, is_triangulated, triangulated_pts);
}
