/* fuse_oracle.c -- the geometry and search of match::fuse::replace_duplication, as recalled (DESIGN.md section 5).  Built with
 * -ffp-contract=off: every product and sum is rounded on its own, in the order written. */
#include "fuse_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

int ott_fuse_observe(const ott_geometry* g, const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist,
                     double* uv, float* x_right, int* pred_level) {
    /* not in the reference: the gates below let a NaN through, and it would then reach the cell range */
    if (!isfinite(pos_w[0]) || !isfinite(pos_w[1]) || !isfinite(pos_w[2])) return 0;
    if (!ott_reproject_to_image(g, pos_w, uv, x_right)) return 0;
    if (!isfinite(uv[0]) || !isfinite(uv[1])) return 0;
    double v[3];
    for (int k = 0; k < 3; ++k) v[k] = pos_w[k] - g->cam_center[k];
    const double dist = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    /* landmark::get_min_valid_distance / get_max_valid_distance return float; the loop compares them with the double distance */
    const float lo = (float)(0.7 * min_valid_dist), hi = (float)(1.3 * max_valid_dist);
    if (dist < lo || hi < dist) return 0;
    const double dot = v[0] * mean_normal[0] + v[1] * mean_normal[1] + v[2] * mean_normal[2];
    if (dot < 0.5 * dist) return 0;
    *pred_level = ott_predict_scale_level((float)dist, max_valid_dist, g->log_scale_factor, g->num_scale_levels);
    return 1;
}

int ott_fuse_replace_duplication_all(const ott_geometry* g, const om_frame* f, const float* scale_factors, const float* inv_level_sigma_sq,
                                     int nq, const int32_t* q_lm, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                                     const float* max_valid_dist, const uint8_t* lm_desc, float margin, int32_t* best_idx, uint8_t* passed,
                                     float* reproj_xy, float* x_right, int32_t* pred_level) {
    const int n1 = nq > 0 ? nq : 1;
    int* lvl = (int*)calloc((size_t)n1, sizeof(int));
    uint8_t* desc = (uint8_t*)calloc((size_t)n1, 32);
    for (int q = 0; q < nq; ++q) {
        const long l = q_lm[q];
        double uv[2];
        float xr = 0.0f;
        int level = 0;
        const int ok = l >= 0 && ott_fuse_observe(g, pos_w + 3 * l, mean_normal + 3 * l, min_valid_dist[l], max_valid_dist[l], uv, &xr, &level);
        passed[q] = (uint8_t)ok;
        reproj_xy[2 * q] = ok ? (float)uv[0] : 0.0f;
        reproj_xy[2 * q + 1] = ok ? (float)uv[1] : 0.0f;
        x_right[q] = ok ? xr : 0.0f;
        pred_level[q] = ok ? level : 0;
        lvl[q] = pred_level[q];
        if (ok) memcpy(desc + 32 * (size_t)q, lm_desc + 32 * l, 32);
    }
    const int num = om_fuse_best_keypoints(f, nq, passed, reproj_xy, x_right, lvl, desc, scale_factors, inv_level_sigma_sq, margin, best_idx);
    free(lvl);
    free(desc);
    return num;
}
