// Test shim: the homography / fundamental-matrix solvers' device arithmetic (openvslam_b200/csrc/two_view_math.cuh) compiled for
// the host, so that tests/test_two_view_solvers_oracle.py can compare it with the oracle (oracle/two_view_solver_oracle.c)
// without a GPU.  Built by that test with g++ -ffp-contract=off (the oracle is built the same way).  model: 0 = H, 1 = F.
#include "../../openvslam_b200/csrc/two_view_math.cuh"

namespace {
ovs::TwoViewNorm norm_of(const float* T4) { return ovs::TwoViewNorm{T4[0], T4[1], T4[2], T4[3]}; }
}  // namespace

extern "C" {
void tvc_normalize(int n, const float* xy, float* norm, float* T4) {
    const ovs::TwoViewNorm N = ovs::two_view_normalize(xy, n, norm);
    T4[0] = N.mean_x; T4[1] = N.mean_y; T4[2] = N.inv_x; T4[3] = N.inv_y;
}
// the model on n matches (idx may be null) with the sequential fixed-order sums
void tvc_compute(int model, int n, const float* norm_1, const float* norm_2, const int* pairs, const int* idx, const float* T4_1,
                 const float* T4_2, double* M) {
    const ovs::TwoViewPairs P{nullptr, nullptr, norm_1, norm_2, pairs};
    if (model == ovs::kTwoViewH)
        ovs::two_view_solve<ovs::kTwoViewH>(P, idx, ovs::PnpSeqSum{n}, norm_of(T4_1), norm_of(T4_2), M);
    else
        ovs::two_view_solve<ovs::kTwoViewF>(P, idx, ovs::PnpSeqSum{n}, norm_of(T4_1), norm_of(T4_2), M);
}
int tvc_check_inliers(int model, const double* M, int n, const float* xy_1, const float* xy_2, const int* pairs, float sigma,
                      unsigned char* flags, double* score) {
    const ovs::TwoViewPairs P{xy_1, xy_2, nullptr, nullptr, pairs};
    const double iss = (double)ovs::two_view_inv_sigma_sq(sigma);
    if (model == ovs::kTwoViewH) return ovs::two_view_score_seq<ovs::kTwoViewH>(M, P, n, iss, flags, score);
    return ovs::two_view_score_seq<ovs::kTwoViewF>(M, P, n, iss, flags, score);
}
}
