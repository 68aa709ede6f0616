/* tracking_oracle.c -- camera::{perspective,equirectangular}::reproject_to_image, frame::can_observe,
 * landmark::predict_scale_level and the direction of match::projection::match_current_and_last_frames, as recalled (DESIGN.md
 * section 5).  Built with -ffp-contract=off: every product and sum is rounded on its own, in the order written. */
#include "tracking_oracle.h"

#include <math.h>

#define OTT_PI 3.14159265358979323846

int ott_reproject_to_image(const ott_geometry* g, const double* pos_w, double* uv, float* x_right) {
    const double* R = g->rot_cw;
    double pc[3];
    for (int r = 0; r < 3; ++r) pc[r] = R[3 * r] * pos_w[0] + R[3 * r + 1] * pos_w[1] + R[3 * r + 2] * pos_w[2] + g->trans_cw[r];
    const ott_camera* c = &g->camera;
    if (c->model == 1) {
        /* longitude / latitude of the unit bearing */
        const double n = sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
        const double bx = pc[0] / n, by = pc[1] / n, bz = pc[2] / n;
        const double latitude = -asin(by), longitude = atan2(bx, bz);
        uv[0] = c->cols * (0.5 + longitude / (2.0 * OTT_PI));
        uv[1] = c->rows * (0.5 - latitude / OTT_PI);
        *x_right = -1.0f;
        return 1;
    }
    if (pc[2] <= 0.0) return 0;
    const double z_inv = 1.0 / pc[2];
    uv[0] = c->fx * pc[0] * z_inv + c->cx;
    uv[1] = c->fy * pc[1] * z_inv + c->cy;
    *x_right = (float)(uv[0] - c->focal_x_baseline * z_inv);
    if (uv[0] < g->min_x || uv[0] > g->max_x) return 0;
    if (uv[1] < g->min_y || uv[1] > g->max_y) return 0;
    return 1;
}

int ott_predict_scale_level(float dist_f, float max_valid_dist, float log_scale_factor, int num_levels) {
    const float ratio = max_valid_dist / dist_f;
    const float lg = (float)log((double)ratio);
    const float level = ceilf(lg / log_scale_factor);
    /* compared as a float before the cast: +inf takes the last level, NaN level 0 */
    if (level >= 0.0f) {
        if (level >= (float)num_levels) return num_levels - 1;
        return (int)level;
    }
    return 0;
}

int ott_can_observe(const ott_geometry* g, const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist,
                    float ray_cos_thr, double* uv, float* x_right, int* pred_level) {
    if (!ott_reproject_to_image(g, pos_w, uv, x_right)) return 0;
    double v[3];
    for (int k = 0; k < 3; ++k) v[k] = pos_w[k] - g->cam_center[k];
    const double dist = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float d = (float)dist;
    const float lo = (float)(0.7 * min_valid_dist), hi = (float)(1.3 * max_valid_dist);
    if (!(lo <= d && d <= hi)) return 0;
    const double dot = v[0] * mean_normal[0] + v[1] * mean_normal[1] + v[2] * mean_normal[2];
    if (dot / dist < ray_cos_thr) return 0;
    *pred_level = ott_predict_scale_level(d, max_valid_dist, g->log_scale_factor, g->num_scale_levels);
    return 1;
}

void ott_motion_direction(const double* pose_cw_curr, const double* pose_cw_last, int is_monocular, double true_baseline, int* forward,
                          int* backward) {
    *forward = *backward = 0;
    if (is_monocular) return;
    double trans_wc[3];
    for (int i = 0; i < 3; ++i)
        trans_wc[i] = -(pose_cw_curr[i] * pose_cw_curr[9] + pose_cw_curr[3 + i] * pose_cw_curr[10] + pose_cw_curr[6 + i] * pose_cw_curr[11]);
    const double z = pose_cw_last[6] * trans_wc[0] + pose_cw_last[7] * trans_wc[1] + pose_cw_last[8] * trans_wc[2] + pose_cw_last[11];
    *forward = z > true_baseline;
    *backward = -z > true_baseline;
}

void ott_can_observe_all(const ott_geometry* g, int n, const uint8_t* usable, const double* pos_w, const double* mean_normal,
                         const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr, uint8_t* observable, float* reproj_xy,
                         float* x_right, int32_t* pred_level) {
    for (int l = 0; l < n; ++l) {
        double uv[2];
        float xr = 0.0f;
        int level = 0;
        const int ok = (!usable || usable[l]) && ott_can_observe(g, pos_w + 3 * (long)l, mean_normal + 3 * (long)l, min_valid_dist[l],
                                                                 max_valid_dist[l], ray_cos_thr, uv, &xr, &level);
        observable[l] = (uint8_t)ok;
        reproj_xy[2 * l] = ok ? (float)uv[0] : 0.0f;
        reproj_xy[2 * l + 1] = ok ? (float)uv[1] : 0.0f;
        x_right[l] = ok ? xr : 0.0f;
        pred_level[l] = ok ? level : 0;
    }
}

void ott_reproject_all(const ott_geometry* g, int n, const uint8_t* usable, const double* pos_w, uint8_t* in_image, float* reproj_xy,
                       float* x_right) {
    for (int l = 0; l < n; ++l) {
        double uv[2];
        float xr = 0.0f;
        const int ok = (!usable || usable[l]) && ott_reproject_to_image(g, pos_w + 3 * (long)l, uv, &xr);
        in_image[l] = (uint8_t)ok;
        reproj_xy[2 * l] = ok ? (float)uv[0] : 0.0f;
        reproj_xy[2 * l + 1] = ok ? (float)uv[1] : 0.0f;
        x_right[l] = ok ? xr : 0.0f;
    }
}
