// tracking_math.cuh -- FP64 geometry the tracker computes per landmark before its two projection searches
// (camera::base::reproject_to_image, data::frame::can_observe, data::landmark::predict_scale_level and the motion-model
// direction of match::projection::match_current_and_last_frames; names as recalled, DESIGN.md section 5).
// __host__ __device__ so the C ABI can evaluate the motion direction on the host with the same code the kernel runs.
// Only + - * /, sqrt and the log of the predicted level are used, except the equirectangular reprojection's atan2 / asin
// (ransac_reproject, as in sim3_math.cuh).  The oracle (oracle/tracking_oracle.c) restates every function independently.
//
// Pose = {R row-major (9), t (3)} of cam_pose_cw: p_c = R p_w + t.
#pragma once
#include "sim3_math.cuh"

namespace ovs {

// camera::base::img_bounds_
struct ImgBounds {
    float min_x, max_x, min_y, max_y;
};

// The predicted level's logarithm on both sides: the double log of the float argument, rounded to float once.  CUDA's logf and
// glibc's logf each stay within about an ulp of the true value but do not always agree, and a quotient next to an integer then
// flips the ceil.
OVS_BA_HD float log_f(float x) { return (float)log((double)x); }

// camera::reproject_to_image(rot_cw, trans_cw, pos_w, reproj, x_right).  Perspective (fisheye and radial division on undistorted
// keypoints alike): false behind the camera (z <= 0, so z = -0.0 too), else the pinhole reprojection in double, x_right =
// reproj(0) - focal_x_baseline * z_inv in double rounded to float once, and the in-image test of the double reprojection against
// the float bounds with < / >.  Equirectangular: always in the image, x_right = -1.  A NaN coordinate fails no comparison.
OVS_BA_HD bool reproject_to_image(const CameraD& cam, const ImgBounds& b, const double* rot_cw, const double* trans_cw, const double* pos_w,
                                  double* uv, float* x_right) {
    if (!ransac_reproject(cam, rot_cw, trans_cw, pos_w, uv)) return false;
    if (cam.model == kCamEquirectangular) {
        *x_right = -1.0f;
        return true;
    }
    // z of the same p_c ransac_reproject formed: (R row 2 . p, summed x, y, z) + t_z
    const double z = rot_cw[6] * pos_w[0] + rot_cw[7] * pos_w[1] + rot_cw[8] * pos_w[2] + trans_cw[2];
    const double z_inv = 1.0 / z;
    *x_right = (float)(uv[0] - cam.fb * z_inv);
    if (uv[0] < b.min_x || uv[0] > b.max_x) return false;
    if (uv[1] < b.min_y || uv[1] > b.max_y) return false;
    return true;
}

// landmark::predict_scale_level(dist_f, frm): ratio = max_valid_dist_ / dist_f in float, ceil(log_f(ratio) / log_scale_factor) in
// float, clamped to [0, num_levels - 1].  The clamp compares the float quotient before the cast to int, so that an infinite
// quotient (dist_f = 0) takes the last level and a NaN one level 0.
OVS_BA_HD int predict_scale_level(float dist_f, float max_valid_dist, float log_scale_factor, int num_levels) {
    const float ratio = max_valid_dist / dist_f;
    const float q = ceilf(log_f(ratio) / log_scale_factor);
    if (!(q >= 0.0f)) return 0;
    if ((float)num_levels <= q) return num_levels - 1;
    return (int)q;
}

// frame::can_observe(lm, ray_cos_thr, reproj, x_right, pred_scale_level): the in-image test, then the ORB scale range of
// (float)dist against (float)(0.7 * min_valid_dist_) and (float)(1.3 * max_valid_dist_) (landmark::is_inside_in_orb_scale), then
// the ray test dot(cam_to_lm_vec, mean_normal) / dist < ray_cos_thr -> reject in double, then the predicted level.
// cam_to_lm_vec = pos_w - cam_center, dist = sqrt((x^2 + y^2) + z^2), the dot summed x, y, z.
OVS_BA_HD bool can_observe(const CameraD& cam, const ImgBounds& b, const double* rot_cw, const double* trans_cw, const double* cam_center,
                           const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist, float ray_cos_thr,
                           float log_scale_factor, int num_levels, double* uv, float* x_right, int* pred_level) {
    if (!reproject_to_image(cam, b, rot_cw, trans_cw, pos_w, uv, x_right)) return false;
    const double v[3] = {pos_w[0] - cam_center[0], pos_w[1] - cam_center[1], pos_w[2] - cam_center[2]};
    const double dist = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float dist_f = (float)dist;
    const float min_dist = (float)(0.7 * (double)min_valid_dist), max_dist = (float)(1.3 * (double)max_valid_dist);
    if (!(min_dist <= dist_f && dist_f <= max_dist)) return false;
    const double ray_cos = (v[0] * mean_normal[0] + v[1] * mean_normal[1] + v[2] * mean_normal[2]) / dist;
    if (ray_cos < (double)ray_cos_thr) return false;
    *pred_level = predict_scale_level(dist_f, max_valid_dist, log_scale_factor, num_levels);
    return true;
}

// match::fuse::replace_duplication's per-landmark geometry (fuse_observe(...) in DESIGN.md section 5): the in-image test, then the
// valid-distance range and the ray test as that loop writes them -- both in double, unlike can_observe: dist < (double)(float)(0.7 *
// min_valid_dist_) or (double)(float)(1.3 * max_valid_dist_) < dist rejects, and dot(cam_to_lm_vec, mean_normal) < 0.5 * dist
// rejects, with no division -- then the predicted level of (float)dist.  dist and the dot are summed as in can_observe.  A position
// or a reprojection that is not finite is rejected first: those gates let a NaN through, and the reference is undefined there.
OVS_BA_HD bool fuse_observe(const CameraD& cam, const ImgBounds& b, const double* rot_cw, const double* trans_cw, const double* cam_center,
                            const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist, float log_scale_factor,
                            int num_levels, double* uv, float* x_right, int* pred_level) {
    if (!(isfinite(pos_w[0]) && isfinite(pos_w[1]) && isfinite(pos_w[2]))) return false;
    if (!reproject_to_image(cam, b, rot_cw, trans_cw, pos_w, uv, x_right)) return false;
    if (!(isfinite(uv[0]) && isfinite(uv[1]))) return false;
    const double v[3] = {pos_w[0] - cam_center[0], pos_w[1] - cam_center[1], pos_w[2] - cam_center[2]};
    const double dist = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float min_dist = (float)(0.7 * (double)min_valid_dist), max_dist = (float)(1.3 * (double)max_valid_dist);
    if (dist < (double)min_dist || (double)max_dist < dist) return false;
    if (v[0] * mean_normal[0] + v[1] * mean_normal[1] + v[2] * mean_normal[2] < 0.5 * dist) return false;
    *pred_level = predict_scale_level((float)dist, max_valid_dist, log_scale_factor, num_levels);
    return true;
}

// The motion model's direction (match::projection::match_current_and_last_frames): trans_wc = -R_cw^T t_cw, trans_lc = R_lw trans_wc
// + t_lw, each row summed x, y, z; forward when trans_lc.z > true_baseline, backward when -trans_lc.z > true_baseline; monocular
// gives neither.
OVS_BA_HD void motion_direction(const double* pose_cw_curr, const double* pose_cw_last, bool is_monocular, double true_baseline, bool* forward,
                                bool* backward) {
    *forward = *backward = false;
    if (is_monocular) return;
    const double* R = pose_cw_curr;
    const double* t = pose_cw_curr + 9;
    double wc[3];
    for (int i = 0; i < 3; ++i) wc[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
    const double* L = pose_cw_last;
    const double z = L[6] * wc[0] + L[7] * wc[1] + L[8] * wc[2] + L[11];
    *forward = z > true_baseline;
    *backward = -z > true_baseline;
}

}  // namespace ovs
