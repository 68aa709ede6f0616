// Test shim: the Sim3 RANSAC solver's device arithmetic (openvslam_b200/csrc/sim3_math.cuh) compiled for the host, so that
// tests/test_sim3_solver_oracle.py can compare it with the oracle (oracle/sim3_solver_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).
#include "../../openvslam_b200/csrc/sim3_math.cuh"

extern "C" {
uint64_t ssc_splitmix64_mix(uint64_t z) { return ovs::splitmix64_mix(z); }
void ssc_ransac_triple(uint64_t seed, int k, int n, int* idx) { ovs::sim3_ransac_triple(seed, k, n, idx); }
void ssc_jacobi4(double* A, double* V) { ovs::jacobi4(A, V); }
void ssc_horn(const double* p1, const double* p2, int fix_scale, double* S12, double* S21) { ovs::sim3_horn(p1, p2, fix_scale != 0, S12, S21); }
int ssc_reproject(const ovs::CameraD* cam, const double* rot, const double* trans, const double* p, double* uv) {
    return ovs::ransac_reproject(*cam, rot, trans, p, uv) ? 1 : 0;
}
// count_inliers of one hypothesis over n pairs given in keyframe camera frames, as the kernel evaluates it (own reprojections and
// bounds as k_sim3_ransac_prep forms them); flags may be null
int ssc_count_inliers(const ovs::CameraD* cam1, const ovs::CameraD* cam2, const double* S12, const double* S21, int n, const double* pc1,
                      const double* pc2, const float* sigma_sq_1, const float* sigma_sq_2, unsigned char* flags) {
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
    double sR12[9], sR21[9];
    ovs::sim3_scaled_rotation(S12, sR12);
    ovs::sim3_scaled_rotation(S21, sR21);
    int count = 0;
    for (int i = 0; i < n; ++i) {
        double r1[2] = {0, 0}, r2[2] = {0, 0};
        const bool ok1 = ovs::ransac_reproject(*cam1, I, zero, pc1 + 3 * i, r1);
        const bool ok2 = ovs::ransac_reproject(*cam2, I, zero, pc2 + 3 * i, r2);
        const bool in = ovs::ransac_is_inlier(*cam1, *cam2, sR12, S12 + 9, sR21, S21 + 9, pc1 + 3 * i, pc2 + 3 * i, r1, r2,
                                              ovs::ransac_bound(sigma_sq_1[i], ok1), ovs::ransac_bound(sigma_sq_2[i], ok2));
        if (flags) flags[i] = in ? 1 : 0;
        count += in ? 1 : 0;
    }
    return count;
}
}
