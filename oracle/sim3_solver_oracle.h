/* oracle/sim3_solver_oracle.h -- CPU oracle for solve::sim3_solver::find_via_ransac (loop detection; test infrastructure only).
 * sim3 = {R row-major (9), t (3), s}, S p = s R p + t; S_12 maps keyframe 2's camera frame into keyframe 1's. */
#ifndef SIM3_SOLVER_ORACLE_H
#define SIM3_SOLVER_ORACLE_H
#include <stdint.h>
#include "ba_oracle.h"

uint64_t os_splitmix64_mix(uint64_t z);
/* the three distinct pair indices of hypothesis k (n >= 3) */
void os_ransac_triple(uint64_t seed, int k, int n, int* idx);
/* cyclic Jacobi of a symmetric 4 x 4 (row-major): eigenvalues (the final diagonal) and eigenvectors (columns of V) */
void os_jacobi4(const double* A, double* evals, double* V);
/* Horn's closed form on three pairs (p[3 * j + c]): S_12 and its inverse S_21 */
void os_horn(const double* p1, const double* p2, int fix_scale, double* S12, double* S21);
/* camera::reproject_to_image(rot_cw, trans_cw, p): returns 0 when a perspective point is not in front of the camera */
int os_reproject(const ob_camera* cam, const double* rot, const double* trans, const double* p, double* uv);
/* find_via_ransac on one problem of n pairs.  hyp_idx (3 * max_num_iter) / hyp_count (max_num_iter) may be NULL; when given they
 * receive every hypothesis's triple and inlier count (all -1 / 0 when no hypothesis runs). */
void os_sim3_solve_ransac(const ob_camera* cam_1, const ob_camera* cam_2, const double* pose_1w, const double* pose_2w, int n,
                          const double* pos_w_1, const float* sigma_sq_1, const double* pos_w_2, const float* sigma_sq_2, int fix_scale,
                          int min_num_inliers, int max_num_iter, uint64_t seed, double* sim3_12, int* valid, int* num_inliers,
                          int* best_iter, uint8_t* inlier_out, int* hyp_idx, int* hyp_count);
#endif
