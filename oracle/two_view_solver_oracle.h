/* oracle/two_view_solver_oracle.h -- CPU oracle for solve::homography_solver and solve::fundamental_solver ::find_via_ransac
 * (perspective map initialisation; test infrastructure only).  Keypoints are x, y floats (2 per keypoint); a match is
 * (idx_1, idx_2) into them; model 0 is H_21 (p2 ~ H_21 p1), model 1 is F_21 (p2^T F_21 p1 = 0), row-major. */
#ifndef TWO_VIEW_SOLVER_ORACLE_H
#define TWO_VIEW_SOLVER_ORACLE_H
#include <stdint.h>

#define OT_MODEL_H 0
#define OT_MODEL_F 1

/* solve::common's normalize over n keypoints: norm (2 per keypoint) and T4 = {mean_x, mean_y, inv_x, inv_y} */
void ot_normalize(int n, const float* xy, float* norm, float* T4);
/* the model on the matches idx[0 .. n) (idx NULL: 0 .. n) of pairs, from normalised points and both views' T4, denormalised */
void ot_compute(int model, int n, const float* norm_1, const float* norm_2, const int* pairs, const int* idx, const float* T4_1,
                const float* T4_2, double* M);
/* check_inliers of M over n matches: the count, the flags (may be NULL) and the score in its fixed order */
int ot_check_inliers(int model, const double* M, int n, const float* xy_1, const float* xy_2, const int* pairs, float sigma,
                     uint8_t* flags, double* score);
/* find_via_ransac on one problem; hyp_idx[max_num_iter * 8], hyp_M[max_num_iter * 9], hyp_score[max_num_iter] and
 * hyp_count[max_num_iter] may be NULL */
void ot_solve_ransac(int model, int n1, const float* xy_1, int n2, const float* xy_2, int n, const int* pairs, float sigma,
                     int max_num_iter, int recompute, uint64_t seed, double* M, int* valid, int* num_inliers, int* best_iter,
                     double* best_score, uint8_t* inlier_out, int* hyp_idx, double* hyp_M, double* hyp_score, int* hyp_count);

#endif
