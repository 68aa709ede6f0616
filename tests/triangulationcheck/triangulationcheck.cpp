// Test shim: the two-view triangulator's device arithmetic (openvslam_b200/csrc/triangulation_math.cuh) compiled for the host, so
// that tests/test_two_view_triangulator_oracle.py can compare it with the oracle (oracle/triangulation_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).  The keyframe arguments have the layout of
// ovs_keyframe_view.
#include "../../openvslam_b200/csrc/triangulation_math.cuh"
#include "../../include/ovs_b200.h"

namespace {
ovs::TriCam cam_of(const ovs_keyframe_view& k) {
    ovs::TriCam c;
    for (int i = 0; i < 12; ++i) c.pose[i] = k.pose_cw[i];
    c.cam = ovs::CameraD{k.camera.model, k.camera.fx, k.camera.fy, k.camera.cx, k.camera.cy, k.camera.focal_x_baseline, k.camera.cols,
                         k.camera.rows};
    c.true_baseline = k.true_baseline;
    return c;
}
ovs::TriKeypt keypt_of(const ovs_keyframe_view& k, int i) {
    ovs::TriKeypt r;
    for (int c = 0; c < 3; ++c) r.bearing[c] = k.bearings[3 * i + c];
    r.x = k.undist_keypts[i].x; r.y = k.undist_keypts[i].y;
    r.x_right = k.stereo_x_right ? k.stereo_x_right[i] : -1.0f;
    r.depth = k.depths ? k.depths[i] : -1.0f;
    r.sigma_sq = k.level_sigma_sq[k.undist_keypts[i].octave];
    r.scale_factor = k.scale_factors[k.undist_keypts[i].octave];
    return r;
}
}  // namespace

extern "C" void tc_two_view_triangulate(const ovs_keyframe_view* k1, const ovs_keyframe_view* k2, int m, const int* pairs, double cos_thr,
                                        double* pos_w, int* reason, int* branch) {
    const ovs::TriCam c1 = cam_of(*k1), c2 = cam_of(*k2);
    for (int i = 0; i < m; ++i) {
        double p[3] = {0.0, 0.0, 0.0};
        reason[i] = ovs::tri_two_view(c1, c2, keypt_of(*k1, pairs[2 * i]), keypt_of(*k2, pairs[2 * i + 1]), cos_thr, 1.5f * k1->scale_factor,
                                      p, &branch[i]);
        for (int c = 0; c < 3; ++c) pos_w[3 * i + c] = reason[i] == ovs::kTriOk ? p[c] : 0.0;
    }
}
