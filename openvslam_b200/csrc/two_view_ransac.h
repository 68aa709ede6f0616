// two_view_ransac.h -- the two-view RANSAC solves (two_view_ransac.cu) as pieces a composed call stages and enqueues itself:
// map initialisation (initializer.cu) carves the solves' buffers into its own staging and enqueues its kernels after them, so
// they read the solutions on the device, with one copy each way and one wait for the whole call.
#pragma once
#include "match_common.h"
#include "two_view_math.cuh"

namespace ovs {

// One batched solve's outputs: device buffers and their host copies (carved together, filled by the caller's download).
struct SolveOut {
    double* M; double* score; int* num; int* best; uint8_t* valid; uint8_t* inlier;            // device
    double* hM; double* hscore; int* hnum; int* hbest; uint8_t* hvalid; uint8_t* hinlier;      // host
};

// One batched solve's device scratch.  np_1, np_2 and norm are used by the keypoint solves (H, F) only.
struct SolveScratch {
    double* hyp; double* hyp_score; int* hyp_count; int* cidx;
    float* np_1; float* np_2; TwoViewNorm* norm;
};

// The staged inputs of a batch of B problems (device pointers).  H and F read the keypoints (koff_*, kp_*: x, y per keypoint) and
// pairs (2 per match, problem-local keypoint indices); E reads one bearing per match and view (bear_*: 3 per match).
struct SolveInputs {
    int B, H, recompute;                             // problems, hypotheses per problem (max_num_iter), recompute
    const int* off; const uint64_t* seed;            // B + 1 match offsets, B seeds
    const int* koff_1; const int* koff_2; const float* kp_1; const float* kp_2; const int* pairs;
    const double* bear_1; const double* bear_2;
};

// Carve one solve's outputs (S.out: after the caller's inputs) and, separately, its scratch (S.dev: after every output).  N
// matches; K1, K2 keypoints per view (0 for E).
void carve_solve_out(Staging& S, SolveOut& o, size_t NB, size_t N);
void carve_solve_scratch(Staging& S, SolveScratch& s, size_t NB, size_t H, size_t N, size_t K1, size_t K2);

// Enqueue the solve's kernels on st (no copy, no wait): the launches the solver's entry point states.
int enqueue_homography_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s, float sigma);
int enqueue_fundamental_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s, float sigma);
int enqueue_essential_solve(cudaStream_t st, const SolveInputs& in, const SolveOut& o, const SolveScratch& s);

// OVS_ERR_INVALID_ARG unless each of the n bearings b[3 i ..] is a finite unit vector (|b.b - 1| <= 1e-6).
int check_bearings(const double* b, int n, const char* what);

}  // namespace ovs
