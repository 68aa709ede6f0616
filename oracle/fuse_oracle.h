/* fuse_oracle.h -- match::fuse::replace_duplication's per-landmark geometry and search (match/fuse.cc, as recalled; DESIGN.md
 * section 5), restated on the CPU for the tests, on the tracker's reprojection (tracking_oracle.h) and the fuse matching core
 * (match_oracle.h). */
#ifndef FUSE_ORACLE_H
#define FUSE_ORACLE_H
#include <stdint.h>

#include "match_oracle.h"
#include "tracking_oracle.h"

/* The geometry of one landmark in one keyframe: 1 = it passes (then uv, x_right, pred_level are written).  Rejected: a position or
 * a reprojection that is not finite, not in the image, dist < (double)(float)(0.7 min) or (double)(float)(1.3 max) < dist,
 * v . n < 0.5 dist; pred_level = predict_scale_level((float)dist). */
int ott_fuse_observe(const ott_geometry* g, const double* pos_w, const double* mean_normal, float min_valid_dist, float max_valid_dist,
                     double* uv, float* x_right, int* pred_level);

/* One target keyframe and nq queries, one after the other: q_lm[q] = landmark row or -1 (skip); the geometry, then
 * om_fuse_best_keypoints' search over the ones that passed.  Outputs as ovs_fuse_replace_duplication_host (0 where not passed);
 * returns the number of queries with a best_idx. */
int ott_fuse_replace_duplication_all(const ott_geometry* g, const om_frame* f, const float* scale_factors, const float* inv_level_sigma_sq,
                                     int nq, const int32_t* q_lm, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                                     const float* max_valid_dist, const uint8_t* lm_desc, float margin, int32_t* best_idx, uint8_t* passed,
                                     float* reproj_xy, float* x_right, int32_t* pred_level);
#endif
