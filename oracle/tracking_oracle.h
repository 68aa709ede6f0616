/* tracking_oracle.h -- the tracker's per-landmark geometry (camera::reproject_to_image, frame::can_observe,
 * landmark::predict_scale_level, the motion model's direction), restated on the CPU for the tests.  ott_geometry has the layout of
 * ovs_frame_geometry (include/ovs_b200.h). */
#ifndef TRACKING_ORACLE_H
#define TRACKING_ORACLE_H
#include <stdint.h>

typedef struct {
    int32_t model;                     /* 1 = equirectangular, anything else reprojects with the pinhole formula */
    double fx, fy, cx, cy, focal_x_baseline, cols, rows;
} ott_camera;

typedef struct {
    ott_camera camera;
    float min_x, max_x, min_y, max_y;
    double rot_cw[9], trans_cw[3], cam_center[3];
    int32_t num_scale_levels;
    float log_scale_factor;
} ott_geometry;

/* camera::reproject_to_image: 1 = in the image; uv and x_right are written whenever the reprojection exists */
int ott_reproject_to_image(const ott_geometry* g, const double* pos_w, double* uv, float* x_right);
int ott_predict_scale_level(float dist_f, float max_valid_dist, float log_scale_factor, int num_levels);
/* frame::can_observe: 1 = observable (then uv, x_right, pred_level are written) */
int ott_can_observe(const ott_geometry* g, const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist,
                    float ray_cos_thr, double* uv, float* x_right, int* pred_level);
void ott_motion_direction(const double* pose_cw_curr, const double* pose_cw_last, int is_monocular, double true_baseline, int* forward,
                          int* backward);

/* The tracker's loops, one landmark after the other, with the outputs of ovs_frame_can_observe_host /
 * ovs_projection_match_current_and_last_reproject_host (usable may be NULL; 0 outputs where not observable / not in the image). */
void ott_can_observe_all(const ott_geometry* g, int n, const uint8_t* usable, const double* pos_w, const double* mean_normal,
                         const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr, uint8_t* observable, float* reproj_xy,
                         float* x_right, int32_t* pred_level);
void ott_reproject_all(const ott_geometry* g, int n, const uint8_t* usable, const double* pos_w, uint8_t* in_image, float* reproj_xy,
                       float* x_right);
#endif
