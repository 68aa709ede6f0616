// tracking_search.cu -- the tracker's per-landmark geometry on the device (frame::can_observe, landmark::predict_scale_level,
// camera::reproject_to_image): k_track_geometry, one FP64 thread per landmark, on the arithmetic of tracking_math.cuh.
// The composed entries feed its outputs to the existing projection matchers through their C ABI
// (ovs_projection_match_frame_and_landmarks_host, ovs_projection_match_current_and_last_host): one matcher, one replay.
#include <cmath>
#include <cstring>
#include <vector>

#include "match_common.h"
#include "tracking_math.cuh"

namespace ovs {

namespace {

struct TrackArgs {
    CameraD cam;
    ImgBounds b;
    double rot[9], trans[3], center[3];
    float ray_cos_thr, log_scale_factor;
    int num_levels, n;
    const uint8_t* usable;
    const double* pos;
    const double* normal;            // nullptr: reprojection only (the motion model)
    const float* min_dist;
    const float* max_dist;
    uint8_t* ok;
    float2* uv;
    float* xr;
    int* level;
};

__global__ void __launch_bounds__(128) k_track_geometry(TrackArgs A) {
    const int l = blockIdx.x * 128 + threadIdx.x;
    if (l >= A.n) return;
    double p[3], uv[2] = {0.0, 0.0};
    for (int k = 0; k < 3; ++k) p[k] = A.pos[3 * (size_t)l + k];
    float xr = 0.0f;
    int level = 0;
    bool ok = false;
    if (A.usable[l]) {
        if (A.normal) {
            double nrm[3];
            for (int k = 0; k < 3; ++k) nrm[k] = A.normal[3 * (size_t)l + k];
            ok = can_observe(A.cam, A.b, A.rot, A.trans, A.center, p, nrm, A.min_dist[l], A.max_dist[l], A.ray_cos_thr, A.log_scale_factor,
                             A.num_levels, uv, &xr, &level);
        } else {
            ok = reproject_to_image(A.cam, A.b, A.rot, A.trans, p, uv, &xr);
        }
    }
    A.ok[l] = ok ? 1 : 0;
    A.uv[l] = ok ? make_float2((float)uv[0], (float)uv[1]) : make_float2(0.0f, 0.0f);
    A.xr[l] = ok ? xr : 0.0f;
    if (A.level) A.level[l] = ok ? level : 0;
}

TrackArgs track_args(const ovs_frame_geometry& g) {
    TrackArgs A{};
    const ovs_camera& c = g.camera;
    A.cam.model = c.model == OVS_CAMERA_EQUIRECTANGULAR ? kCamEquirectangular : kCamPerspective;
    A.cam.fx = c.fx; A.cam.fy = c.fy; A.cam.cx = c.cx; A.cam.cy = c.cy; A.cam.fb = c.focal_x_baseline; A.cam.cols = c.cols; A.cam.rows = c.rows;
    A.b = ImgBounds{g.min_x, g.max_x, g.min_y, g.max_y};
    for (int k = 0; k < 9; ++k) A.rot[k] = g.rot_cw[k];
    for (int k = 0; k < 3; ++k) { A.trans[k] = g.trans_cw[k]; A.center[k] = g.cam_center[k]; }
    A.log_scale_factor = g.log_scale_factor;
    A.num_levels = g.num_scale_levels;
    return A;
}

// One launch over n > 0 landmarks on the handle's own arenas: inputs up in one copy, outputs back in one, one wait.
// mean_normal == nullptr: reprojection only (pred_scale_level is not written).
int run_track_geometry(ovs_matcher* m, const ovs_frame_geometry& g, int n, const uint8_t* usable, const double* pos_w, const double* mean_normal,
                       const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr, uint8_t* ok, float* uv, float* xr,
                       int32_t* level) {
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    const size_t N = (size_t)n;
    const bool full = mean_normal != nullptr;
    TrackArgs A = track_args(g);
    A.n = n; A.ray_cos_thr = ray_cos_thr;
    uint8_t* hu; double* hpos; double* hnrm = nullptr; float* hmin = nullptr; float* hmax = nullptr;
    uint8_t* hok; float2* huv; float* hxr; int* hlevel = nullptr;
    Staging S;
    int rc = stage(S, m->h_trk, m->h_trk_cap, m->d_trk, m->d_trk_cap, [&](Staging& S) {
        A.usable = S.in(hu, N); A.pos = S.in(hpos, 3 * N);
        if (full) { A.normal = S.in(hnrm, 3 * N); A.min_dist = S.in(hmin, N); A.max_dist = S.in(hmax, N); }
        A.ok = S.out(hok, N); A.uv = S.out(huv, N); A.xr = S.out(hxr, N);
        A.level = full ? S.out(hlevel, N) : nullptr;
    });
    if (rc != OVS_OK) return rc;
    if (usable) memcpy(hu, usable, N);
    else memset(hu, 1, N);
    memcpy(hpos, pos_w, 24 * N);
    if (full) { memcpy(hnrm, mean_normal, 24 * N); memcpy(hmin, min_valid_dist, 4 * N); memcpy(hmax, max_valid_dist, 4 * N); }
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_track_geometry<<<(n + 127) / 128, 128, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    memcpy(ok, hok, N);
    memcpy(uv, huv, 8 * N);
    memcpy(xr, hxr, 4 * N);
    if (full) memcpy(level, hlevel, 4 * N);
    return OVS_OK;
}

int check_can_observe_args(const ovs_frame_geometry* g, int nlm, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                           const float* max_valid_dist, const uint8_t* observable, const float* reproj_xy, const float* x_right,
                           const int32_t* pred_scale_level) {
    OVS_REQUIRE(nlm >= 0, OVS_ERR_INVALID_ARG, "nlm must be >= 0");
    int rc;
    if ((rc = check_geometry(g)) != OVS_OK) return rc;
    OVS_REQUIRE(nlm == 0 || (pos_w && mean_normal && min_valid_dist && max_valid_dist && observable && reproj_xy && x_right && pred_scale_level),
                OVS_ERR_INVALID_ARG, "null argument");
    return OVS_OK;
}

}  // namespace

int check_geometry(const ovs_frame_geometry* g) {
    OVS_REQUIRE(g, OVS_ERR_INVALID_ARG, "null frame geometry");
    const int model = g->camera.model;
    OVS_REQUIRE(model == OVS_CAMERA_PERSPECTIVE || model == OVS_CAMERA_EQUIRECTANGULAR || model == OVS_CAMERA_FISHEYE ||
                model == OVS_CAMERA_RADIAL_DIVISION, OVS_ERR_INVALID_ARG, "unknown camera model %d", model);
    OVS_REQUIRE(g->num_scale_levels >= 1 && g->num_scale_levels <= 16, OVS_ERR_INVALID_ARG, "num_scale_levels %d outside 1 .. 16",
                g->num_scale_levels);
    OVS_REQUIRE(std::isfinite(g->log_scale_factor) && g->log_scale_factor > 0.0f, OVS_ERR_INVALID_ARG,
                "log_scale_factor must be positive and finite");
    bool finite = true;
    for (int k = 0; k < 9; ++k) finite = finite && std::isfinite(g->rot_cw[k]);
    for (int k = 0; k < 3; ++k) finite = finite && std::isfinite(g->trans_cw[k]) && std::isfinite(g->cam_center[k]);
    OVS_REQUIRE(finite, OVS_ERR_INVALID_ARG, "the frame's pose or camera centre is not finite");
    return OVS_OK;
}

}  // namespace ovs

extern "C" int ovs_frame_can_observe_host(ovs_matcher* m, const ovs_frame_geometry* geometry, int nlm, const uint8_t* usable, const double* pos_w,
                                          const double* mean_normal, const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr,
                                          uint8_t* observable, float* reproj_xy, float* x_right, int32_t* pred_scale_level) {
    OVS_REQUIRE(m, OVS_ERR_INVALID_ARG, "null matcher");
    int rc = ovs::check_can_observe_args(geometry, nlm, pos_w, mean_normal, min_valid_dist, max_valid_dist, observable, reproj_xy, x_right,
                                         pred_scale_level);
    if (rc != OVS_OK || nlm == 0) return rc;
    return ovs::run_track_geometry(m, *geometry, nlm, usable, pos_w, mean_normal, min_valid_dist, max_valid_dist, ray_cos_thr, observable,
                                   reproj_xy, x_right, pred_scale_level);
}

extern "C" int ovs_projection_search_local_landmarks_host(ovs_frame_index* f, const ovs_frame_geometry* geometry, const float* scale_factors, int nlm,
                                                          const uint8_t* usable, const double* pos_w, const double* mean_normal,
                                                          const float* min_valid_dist, const float* max_valid_dist, const uint8_t* lm_desc,
                                                          const uint8_t* kp_has_observed_lm, float ray_cos_thr, float margin, float lowe_ratio,
                                                          uint8_t* observable, float* reproj_xy, float* x_right, int32_t* pred_scale_level,
                                                          int32_t* matched_lm_of_kp, int* num_matches) {
    OVS_REQUIRE(f && scale_factors && matched_lm_of_kp && num_matches, OVS_ERR_INVALID_ARG, "bad argument");
    int rc = ovs::check_can_observe_args(geometry, nlm, pos_w, mean_normal, min_valid_dist, max_valid_dist, observable, reproj_xy, x_right,
                                         pred_scale_level);
    if (rc != OVS_OK) return rc;
    OVS_REQUIRE(nlm == 0 || lm_desc, OVS_ERR_INVALID_ARG, "null argument");
    if (nlm > 0 && (rc = ovs::run_track_geometry(ovs::frame_index_matcher(f), *geometry, nlm, usable, pos_w, mean_normal, min_valid_dist,
                                                 max_valid_dist, ray_cos_thr, observable, reproj_xy, x_right, pred_scale_level)) != OVS_OK)
        return rc;
    return ovs_projection_match_frame_and_landmarks_host(f, scale_factors, geometry->num_scale_levels, nlm, observable, reproj_xy, x_right,
                                                         pred_scale_level, lm_desc, kp_has_observed_lm, margin, lowe_ratio, matched_lm_of_kp,
                                                         num_matches);
}

extern "C" int ovs_projection_match_current_and_last_reproject_host(ovs_frame_index* curr, const ovs_frame_geometry* geometry, int is_monocular,
                                                                    double true_baseline, const double* last_pose_cw, const float* scale_factors,
                                                                    int n_last, const uint8_t* last_usable, const double* pos_w,
                                                                    const int32_t* last_octave, const float* last_angle, const uint8_t* lm_desc,
                                                                    const uint8_t* kp_has_observed_lm, float margin, int check_orientation,
                                                                    int32_t* matched_last_of_kp, int* num_matches, uint8_t* in_image_out,
                                                                    float* reproj_xy_out) {
    OVS_REQUIRE(curr && scale_factors && matched_last_of_kp && num_matches && last_pose_cw && n_last >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE((in_image_out == nullptr) == (reproj_xy_out == nullptr), OVS_ERR_INVALID_ARG, "in_image_out and reproj_xy_out come together");
    int rc;
    if ((rc = ovs::check_geometry(geometry)) != OVS_OK) return rc;
    bool finite = std::isfinite(true_baseline);
    for (int k = 0; k < 12; ++k) finite = finite && std::isfinite(last_pose_cw[k]);
    OVS_REQUIRE(finite, OVS_ERR_INVALID_ARG, "the last frame's pose or true_baseline is not finite");
    OVS_REQUIRE(n_last == 0 || (pos_w && last_octave && lm_desc && (!check_orientation || last_angle)), OVS_ERR_INVALID_ARG, "null argument");
    const int L = geometry->num_scale_levels;
    for (int i = 0; i < n_last; ++i)
        OVS_REQUIRE((last_usable && !last_usable[i]) || (last_octave[i] >= 0 && last_octave[i] < L), OVS_ERR_INVALID_ARG,
                    "octave %d of last-frame keypoint %d outside the scale table (%d levels)", last_octave[i], i, L);
    bool forward, backward;
    double pose_cw[12];
    for (int k = 0; k < 9; ++k) pose_cw[k] = geometry->rot_cw[k];
    for (int k = 0; k < 3; ++k) pose_cw[9 + k] = geometry->trans_cw[k];
    ovs::motion_direction(pose_cw, last_pose_cw, is_monocular != 0, true_baseline, &forward, &backward);
    const size_t N = (size_t)std::max(n_last, 1);
    std::vector<uint8_t> in_image(N, 0);
    std::vector<float> uv(2 * N, 0.0f), xr(N, 0.0f);
    if (n_last > 0 && (rc = ovs::run_track_geometry(ovs::frame_index_matcher(curr), *geometry, n_last, last_usable, pos_w, nullptr, nullptr, nullptr,
                                                    0.0f, in_image.data(), uv.data(), xr.data(), nullptr)) != OVS_OK)
        return rc;
    if (in_image_out) {
        memcpy(in_image_out, in_image.data(), (size_t)n_last);
        memcpy(reproj_xy_out, uv.data(), 8 * (size_t)n_last);
    }
    return ovs_projection_match_current_and_last_host(curr, scale_factors, L, n_last, in_image.data(), uv.data(), xr.data(), last_octave, last_angle,
                                                      lm_desc, kp_has_observed_lm, margin, forward ? 1 : 0, backward ? 1 : 0, check_orientation,
                                                      matched_last_of_kp, num_matches);
}
