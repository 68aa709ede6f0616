// Test shim: the PnP RANSAC solver's device arithmetic (openvslam_b200/csrc/pnp_math.cuh) compiled for the host, so that
// tests/test_pnp_solver_oracle.py can compare it with the oracle (oracle/pnp_solver_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).
#include "../../openvslam_b200/csrc/pnp_math.cuh"

extern "C" {
void psc_sample6(uint64_t seed, int k, int n, int* idx) { ovs::ransac_sample<6>(seed, k, n, idx); }
double psc_max_cos(float scale_factor) { return ovs::pnp_max_cos(scale_factor); }
// EPnP on n correspondences (idx may be null) with the sequential fixed-order sums
void psc_epnp(int n, const double* bearings, const double* pos_w, const int* idx, double* pose) {
    const ovs::PnpPoints P{pos_w, bearings, idx, n};
    ovs::epnp_pose(P, ovs::PnpSeqSum{n}, pose);
}
int psc_check_inliers(int n, const double* bearings, const double* pos_w, const float* scale_factor, const double* pose,
                      unsigned char* flags) {
    int count = 0;
    for (int i = 0; i < n; ++i) {
        const bool in = ovs::pnp_is_inlier(pose, pos_w + 3 * i, bearings + 3 * i, ovs::pnp_max_cos(scale_factor[i]));
        if (flags) flags[i] = in ? 1 : 0;
        count += in ? 1 : 0;
    }
    return count;
}
}
