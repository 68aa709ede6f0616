/* oracle/sim3_oracle.h -- CPU oracle for optimize::transform_optimizer (Sim3 refinement of a loop candidate; test
 * infrastructure only).  sim3 = {R row-major (9), t (3), s}, S p = s R p + t; update = [omega, upsilon, sigma]. */
#ifndef SIM3_ORACLE_H
#define SIM3_ORACLE_H
#include <stdint.h>
#include "ba_oracle.h"

void ob_sim3_exp(const double* u, double* S);
void ob_sim3_oplus(const double* S, const double* u, int fix_scale, double* out);
/* e (2) and J (2 x 7, may be NULL) of the forward edge (obs_1 - pi_1(S pc2)) and of the backward edge (obs_2 - pi_2(S^-1 pc1)) */
void ob_sim3_edge_forward(const ob_camera* cam1, const double* S, const double* pc2, const double* obs, double* e, double* J);
void ob_sim3_edge_backward(const ob_camera* cam2, const double* S, const double* pc1, const double* obs, double* e, double* J);
/* transform_optimizer::optimize(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, g2o_Sim3_12, chi_sq) on n correspondences.
 * Returns the inlier count (0 on the early exit, sim3_12 then unchanged); inlier_out[i] = 1 while pair i stays matched. */
int ob_transform_optimize(const ob_camera* cam_1, const ob_camera* cam_2, const double* pose_1w, const double* pose_2w, int n,
                          const double* pos_w_1, const float* obs_xy_1, const float* inv_sigma_sq_1, const double* pos_w_2,
                          const float* obs_xy_2, const float* inv_sigma_sq_2, int fix_scale, float chi_sq, int num_first_iter,
                          int num_iter, double* sim3_12, uint8_t* inlier_out, ob_stats* st);
#endif
