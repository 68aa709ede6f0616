/* oracle/initializer_oracle.h -- CPU oracle for monocular map initialisation (initialize::perspective / bearing_vector::initialize
 * with homography_solver / fundamental_solver / essential_solver::decompose, check_pose and find_most_plausible_pose; test
 * infrastructure only).  A hypothesis is {R row-major (9), t (3)}: p_cur = R p_ref + t. */
#ifndef INITIALIZER_ORACLE_H
#define INITIALIZER_ORACLE_H
#include <stdint.h>

#include "ba_oracle.h"

/* The outcome of one problem, field for field ovs_init_result of include/ovs_b200.h. */
typedef struct {
    int32_t status, model, chosen, num_hypotheses;
    int32_t num_valid[8];
    float cos_parallax[8];
    double rot_ref_to_cur[9], trans_ref_to_cur[3];
    double solver_M[2][9];
    double solver_score[2];
    int32_t solver_num_inliers[2];
    uint8_t solver_valid[2];
    uint8_t reserved[6];
} oi_result;

/* A = U diag(d) V^T by the Jacobi eigen-decomposition of A^T A; the third column of U is u1 x u2 when third_by_cross */
void oi_svd3(const double* A, int third_by_cross, double* U, double* d, double* V);
/* homography_solver::decompose: 1 with 8 hypotheses (R 9, t 3, n 3 each), 0 when refused */
int oi_decompose_homography(const double* H, const ob_camera* cam_1, const ob_camera* cam_2, double* R, double* t, double* n);
/* essential_solver::decompose: 4 hypotheses */
void oi_decompose_essential(const double* E, double* R, double* t);
/* fundamental_solver::decompose: E = K_2^T F K_1, then the essential decomposition */
void oi_decompose_fundamental(const double* F, const ob_camera* cam_1, const ob_camera* cam_2, double* R, double* t);
/* check_pose's test of one match: 0 valid, 1 valid with a small parallax, 2 non-finite, 3 / 4 depth (reference / current),
 * 5 / 6 reprojection (reference / current); p and *cos_par as formed */
int oi_check_match(const double* Rt, const ob_camera* cam_ref, const ob_camera* cam_cur, const double* b_ref, const double* b_cur,
                   const float* kp_ref, const float* kp_cur, double reproj_err_thr_sq, int depth_is_positive, double* p, float* cos_par);
/* find_most_plausible_pose's decision over nh hypotheses -> status (0 ok, 3 too few, 4 ambiguous, 5 small parallax) and *best */
int oi_choose(int nh, const int* count, const float* cos_par, int min_num_triangulated, double cos_thr, int* best);
/* initialize() on one problem.  kp_*: x, y per keypoint; bear_*: 3 per keypoint.  hyp_R[72], hyp_t[24] and reason[8 * m] (per
 * hypothesis, per match in reference-index order: check_pose's code, 7 for a match that is not a solver inlier, -1 for an
 * unused hypothesis) may be NULL.  is_triangulated[n_ref] and pts[n_ref * 3] are always written. */
void oi_initialize(int perspective, const ob_camera* cam_ref, const ob_camera* cam_cur, int n_ref, const float* kp_ref,
                   const double* bear_ref, int n_cur, const float* kp_cur, const double* bear_cur, const int* ref_matches_with_cur,
                   int num_ransac_iters, int min_num_triangulated, float parallax_deg_thr, float reproj_err_thr_sq, uint64_t seed,
                   oi_result* res, double* hyp_R, double* hyp_t, int* reason, uint8_t* is_triangulated, double* pts);

#endif
