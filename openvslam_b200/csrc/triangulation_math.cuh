// triangulation_math.cuh -- FP64 arithmetic of the two-view triangulator of local mapping (module::two_view_triangulator,
// solve::triangulator, keyframe::triangulate_stereo; names as recalled, DESIGN.md section 5).
// __host__ __device__ so tests/triangulationcheck can compare the same code with the oracle (oracle/triangulation_oracle.c) on
// the CPU.  Only + - * / sqrt and fabs are used, except the equirectangular reprojection's atan2 / asin (ransac_reproject, as in
// sim3_math.cuh), so with contraction off the host and the device give the same bits.
//
// Pose = {R row-major (9), t (3)} of cam_pose_cw: p_c = R p_w + t.  Camera centre c = -(R^T t).
#pragma once
#include "pnp_math.cuh"

namespace ovs {

// What the triangulator reads of one keyframe (besides its keypoints).
struct TriCam {
    double pose[12];
    CameraD cam;
    double true_baseline;
};

// What the triangulator reads of one keypoint: bearings_[idx], undist_keypts_[idx].pt, stereo_x_right_[idx] (< 0: monocular),
// depths_[idx], level_sigma_sq_[octave] and scale_factors_[octave].
struct TriKeypt {
    double bearing[3];
    float x, y, x_right, depth, sigma_sq, scale_factor;
};

// The outcome of one pair, in the order the reference tests it.  Only kTriOk creates a landmark.
enum : int {
    kTriOk = 0,
    kTriNoBranch = 1,          // neither enough parallax for two cameras nor a stereo keypoint with the smaller stereo parallax
    kTriNonFinite = 2,         // the two-camera solution is not finite (v[3] == 0)
    kTriCheirality1 = 3, kTriCheirality2 = 4,
    kTriReproj1 = 5, kTriReproj2 = 6,
    kTriScale = 7,
};
// The branch that produced pos_w: two-camera triangulation, or the stereo back-projection of keyframe 1 or 2 (-1: none).
enum : int { kTriBranchNone = -1, kTriBranchTwoCameras = 0, kTriBranchStereo1 = 1, kTriBranchStereo2 = 2 };

OVS_BA_HD void tri_cam_center(const double* pose, double* c) {
    for (int i = 0; i < 3; ++i) c[i] = -(pose[i] * pose[9] + pose[3 + i] * pose[10] + pose[6 + i] * pose[11]);
}

// cos(2 atan2(h, d)) = (d^2 - h^2) / (d^2 + h^2), h = true_baseline / 2, d = depth; 2.0 for a monocular keypoint.
OVS_BA_HD double tri_cos_stereo(const TriCam& c, const TriKeypt& k) {
    if (!(0.0f <= k.x_right)) return 2.0;
    const double h = c.true_baseline / 2.0, d = (double)k.depth;
    return (d * d - h * h) / (d * d + h * h);
}

// solve::triangulator::triangulate(b_1, b_2, P_1, P_2): rows b_x P_r3 - b_z P_r1, b_y P_r3 - b_z P_r2 of each view (P = [R | t]),
// v = the eigenvector of A^T A's smallest eigenvalue (jacobi_sym<4>, eig_order ties to the lowest index, eig_column's sign),
// pos_w = v[0:3] / v[3].  A^T A is summed over the rows in order 0..3.  Forming A^T A squares A's condition number: the
// eigenvector's error is about eps (s_1 / s_3)^2 where the reference's SVD has eps s_1 / s_3 (DESIGN.md section 5).
OVS_BA_HD void tri_two_cameras(const double* b1, const double* b2, const double* P1, const double* P2, double* pos_w) {
    double A[16];
    for (int c = 0; c < 4; ++c) {   // column c of [R | t]
        const double p1r1 = c < 3 ? P1[c] : P1[9], p1r2 = c < 3 ? P1[3 + c] : P1[10], p1r3 = c < 3 ? P1[6 + c] : P1[11];
        const double p2r1 = c < 3 ? P2[c] : P2[9], p2r2 = c < 3 ? P2[3 + c] : P2[10], p2r3 = c < 3 ? P2[6 + c] : P2[11];
        A[c] = b1[0] * p1r3 - b1[2] * p1r1;
        A[4 + c] = b1[1] * p1r3 - b1[2] * p1r2;
        A[8 + c] = b2[0] * p2r3 - b2[2] * p2r1;
        A[12 + c] = b2[1] * p2r3 - b2[2] * p2r2;
    }
    double M[16], V[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) M[4 * i + j] = ((A[i] * A[j] + A[4 + i] * A[4 + j]) + A[8 + i] * A[8 + j]) + A[12 + i] * A[12 + j];
    jacobi_sym<4>(M, V);
    int order[4];
    eig_order<4>(M, false, order);
    double v[4];
    eig_column<4>(V, order[0], v);
    for (int k = 0; k < 3; ++k) pos_w[k] = v[k] / v[3];
}

// keyframe::triangulate_stereo(idx), perspective: unproj = (float)((pt - c) * depth * (1 / f)), p_w = R^T p_c + centre; a
// depth <= 0 gives the zero vector.
OVS_BA_HD void tri_stereo(const TriCam& c, const TriKeypt& k, double* pos_w) {
    if (!(0.0f < k.depth)) { pos_w[0] = pos_w[1] = pos_w[2] = 0.0; return; }
    const double fx_inv = 1.0 / c.cam.fx, fy_inv = 1.0 / c.cam.fy;
    const float ux = (float)(((double)k.x - c.cam.cx) * (double)k.depth * fx_inv);
    const float uy = (float)(((double)k.y - c.cam.cy) * (double)k.depth * fy_inv);
    const double pc[3] = {(double)ux, (double)uy, (double)k.depth};
    double ctr[3];
    tri_cam_center(c.pose, ctr);
    for (int i = 0; i < 3; ++i) pos_w[i] = (c.pose[i] * pc[0] + c.pose[3 + i] * pc[1] + c.pose[6 + i] * pc[2]) + ctr[i];
}

// check_depth_is_positive: the camera-frame z, stored as a float, must be > 0 (perspective); equirectangular always passes.
OVS_BA_HD bool tri_depth_positive(const TriCam& c, const double* p) {
    if (c.cam.model == kCamEquirectangular) return true;
    const float z = (float)((c.pose[6] * p[0] + c.pose[7] * p[1] + c.pose[8] * p[2]) + c.pose[11]);
    return 0.0f < z;
}

// check_reprojection_error: chi-square 5.99146f (mono) or 7.81473f (stereo, with the float x_right term) times sigma^2, in float,
// against the squared error in double.  x_right of the reprojection = (float)(u - focal_x_baseline / z).
OVS_BA_HD bool tri_reproj_ok(const TriCam& c, const TriKeypt& k, const double* p) {
    double uv[2];
    if (!ransac_reproject(c.cam, c.pose, c.pose + 9, p, uv)) return false;
    const double ex = uv[0] - (double)k.x, ey = uv[1] - (double)k.y;
    const double e2 = ex * ex + ey * ey;
    if (0.0f <= k.x_right) {
        const double z = (c.pose[6] * p[0] + c.pose[7] * p[1] + c.pose[8] * p[2]) + c.pose[11];
        const float xr = (float)(uv[0] - c.cam.fb * (1.0 / z));
        const float exr = xr - k.x_right;
        return !((double)(7.81473f * k.sigma_sq) < e2 + (double)(exr * exr));
    }
    return !((double)(5.99146f * k.sigma_sq) < e2);
}

// check_scale_factors: d_k = |p - c_k|, ratio_dists = d_2 / d_1, ratio_octave = sf_1 / sf_2 (float); rejected when either
// distance is 0, ratio_dists * f < ratio_octave or ratio_octave * f < ratio_dists, f = 1.5f * keyfrm_1 scale_factor_ (float).
OVS_BA_HD bool tri_scale_ok(const TriCam& c1, const TriCam& c2, float sf_1, float sf_2, float ratio_factor, const double* p) {
    double c[3], d[2];
    const TriCam* cs[2] = {&c1, &c2};
    for (int v = 0; v < 2; ++v) {
        tri_cam_center(cs[v]->pose, c);
        const double x = p[0] - c[0], y = p[1] - c[1], z = p[2] - c[2];
        d[v] = sqrt(x * x + y * y + z * z);
    }
    if (d[0] == 0.0 || d[1] == 0.0) return false;
    const double ratio_dists = d[1] / d[0];
    const float ratio_octave = sf_1 / sf_2;
    return !(ratio_dists * (double)ratio_factor < (double)ratio_octave || (double)(ratio_octave * ratio_factor) < ratio_dists);
}

// two_view_triangulator::triangulate(idx_1, idx_2, pos_w) for one pair.  cos_thr = cos(rays_parallax_deg_thr * pi / 180),
// computed once by the caller.  Returns kTriOk or the first failed test; *branch = the branch taken.  pos_w is written whenever a
// branch was taken.
OVS_BA_HD int tri_two_view(const TriCam& c1, const TriCam& c2, const TriKeypt& k1, const TriKeypt& k2, double cos_thr, float ratio_factor,
                           double* pos_w, int* branch) {
    const bool st1 = 0.0f <= k1.x_right, st2 = 0.0f <= k2.x_right;
    double r1[3], r2[3];
    for (int i = 0; i < 3; ++i) {
        r1[i] = c1.pose[i] * k1.bearing[0] + c1.pose[3 + i] * k1.bearing[1] + c1.pose[6 + i] * k1.bearing[2];
        r2[i] = c2.pose[i] * k2.bearing[0] + c2.pose[3 + i] * k2.bearing[1] + c2.pose[6 + i] * k2.bearing[2];
    }
    const double n1 = sqrt(r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2]), n2 = sqrt(r2[0] * r2[0] + r2[1] * r2[1] + r2[2] * r2[2]);
    const double cos_rays = (r1[0] * r2[0] + r1[1] * r2[1] + r1[2] * r2[2]) / (n1 * n2);
    const double cs1 = tri_cos_stereo(c1, k1), cs2 = tri_cos_stereo(c2, k2);
    const double cs = cs1 < cs2 ? cs1 : cs2;
    const bool two = ((!st1 && !st2) && 0.0 < cos_rays && cos_rays < cos_thr) || ((st1 || st2) && 0.0 < cos_rays && cos_rays < cs);
    if (two) {
        *branch = kTriBranchTwoCameras;
        tri_two_cameras(k1.bearing, k2.bearing, c1.pose, c2.pose, pos_w);
        if (!(isfinite(pos_w[0]) && isfinite(pos_w[1]) && isfinite(pos_w[2]))) return kTriNonFinite;
    } else if (st1 && cs1 < cs2) {
        *branch = kTriBranchStereo1;
        tri_stereo(c1, k1, pos_w);
    } else if (st2 && cs2 < cs1) {
        *branch = kTriBranchStereo2;
        tri_stereo(c2, k2, pos_w);
    } else {
        *branch = kTriBranchNone;
        return kTriNoBranch;
    }
    if (!tri_depth_positive(c1, pos_w)) return kTriCheirality1;
    if (!tri_depth_positive(c2, pos_w)) return kTriCheirality2;
    if (!tri_reproj_ok(c1, k1, pos_w)) return kTriReproj1;
    if (!tri_reproj_ok(c2, k2, pos_w)) return kTriReproj2;
    if (!tri_scale_ok(c1, c2, k1.scale_factor, k2.scale_factor, ratio_factor, pos_w)) return kTriScale;
    return kTriOk;
}

}  // namespace ovs
