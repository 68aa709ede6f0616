/* triangulation_oracle.h -- module::two_view_triangulator and the compute step of mapping_module::create_new_landmarks (local
 * mapping), restated on the CPU for the tests.  otr_keyframe has the layout of ovs_keyframe_view (include/ovs_b200.h). */
#ifndef TRIANGULATION_ORACLE_H
#define TRIANGULATION_ORACLE_H
#include <stdint.h>

#include "ba_oracle.h"

typedef struct {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} otr_keypoint;

typedef struct {
    double pose_cw[12];
    ob_camera camera;
    double true_baseline;
    float scale_factor;
    int32_t num_scale_levels;
    const float* scale_factors;
    const float* level_sigma_sq;
    int32_t num_keypts;
    const otr_keypoint* undist_keypts;
    const double* bearings;
    const float* stereo_x_right;
    const float* depths;
    const uint8_t* descriptors;
    const uint8_t* has_landmark;
    const int32_t* bow_node;
} otr_keyframe;

/* reasons: 0 landmark, 1 no branch, 2 non-finite, 3 / 4 cheirality of view 1 / 2, 5 / 6 reprojection of view 1 / 2, 7 scale;
 * branch: 0 two cameras, 1 stereo of keyframe 1, 2 stereo of keyframe 2, -1 none */
int otr_triangulate(const otr_keyframe* k1, const otr_keyframe* k2, int idx_1, int idx_2, double cos_thr, double* pos_w, int* branch);
/* m pairs (idx_1, idx_2): valid, pos_w (zero where invalid), reason and branch per pair */
void otr_two_view_triangulate(const otr_keyframe* k1, const otr_keyframe* k2, int m, const int* pairs, double deg_thr, uint8_t* valid,
                              double* pos_w, int* reason, int* branch);
/* the sequential loop over the B neighbours; records (neighbour, idx_1, idx_2) in rec[3 * r], points in pos[3 * r]; returns the count */
int otr_create_new_landmarks(const otr_keyframe* k1, int B, const otr_keyframe* k2, const double* E_12, const double* epipole_in_2,
                             int check_orientation, double deg_thr, int* rec, double* pos);
#endif
