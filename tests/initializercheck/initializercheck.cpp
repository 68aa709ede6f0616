// Test shim: map initialisation's device arithmetic (openvslam_b200/csrc/initializer_math.cuh) compiled for the host, so that
// tests/test_initializer_oracle.py can compare it with the oracle (oracle/initializer_oracle.c) without a GPU.  Built by that test
// with g++ -ffp-contract=off (the oracle is built the same way).  Cameras have the layout of ovs_camera.
#include "../../openvslam_b200/csrc/initializer_math.cuh"
#include "../../include/ovs_b200.h"

namespace {
ovs::CameraD cam_of(const ovs_camera& c) { return ovs::CameraD{c.model, c.fx, c.fy, c.cx, c.cy, c.focal_x_baseline, c.cols, c.rows}; }
}  // namespace

extern "C" void ic_svd3(const double* A, int third_by_cross, double* U, double* d, double* V) { ovs::svd3(A, third_by_cross != 0, U, d, V); }

extern "C" int ic_decompose_homography(const double* H, const ovs_camera* c1, const ovs_camera* c2, double* R, double* t, double* n) {
    return ovs::decompose_homography(H, cam_of(*c1), cam_of(*c2), R, t, n) ? 1 : 0;
}

extern "C" void ic_decompose_essential(const double* E, double* R, double* t) { ovs::decompose_essential(E, R, t); }

extern "C" void ic_decompose_fundamental(const double* F, const ovs_camera* c1, const ovs_camera* c2, double* R, double* t) {
    ovs::decompose_fundamental(F, cam_of(*c1), cam_of(*c2), R, t);
}

// check_pose's test of m matches (bearings 3 and keypoints 2 per match) under one hypothesis Rt[12]
extern "C" void ic_check_matches(const double* Rt, const ovs_camera* cr, const ovs_camera* cc, int m, const double* b_ref, const double* b_cur,
                                 const float* kp_ref, const float* kp_cur, double thr_sq, int depth_is_positive, int* code, double* p, float* cos_par) {
    const ovs::CameraD c1 = cam_of(*cr), c2 = cam_of(*cc);
    for (int i = 0; i < m; ++i) {
        double q[3] = {0.0, 0.0, 0.0};
        float c = 0.0f;
        code[i] = ovs::init_check_match(Rt, c1, c2, b_ref + 3 * i, b_cur + 3 * i, kp_ref + 2 * i, kp_cur + 2 * i, thr_sq, depth_is_positive != 0, q, &c);
        for (int k = 0; k < 3; ++k) p[3 * i + k] = q[k];
        cos_par[i] = c;
    }
}

extern "C" int ic_choose(int nh, const int* count, const float* cos_par, int min_num, double cos_thr, int* best) {
    return ovs::init_choose(nh, count, cos_par, min_num, cos_thr, best);
}

extern "C" unsigned ic_key(float f) { return ovs::init_key(f); }
extern "C" float ic_key_value(unsigned k) { return ovs::init_key_value(k); }
