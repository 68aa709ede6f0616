/* oracle/pnp_solver_oracle.h -- CPU oracle for solve::pnp_solver::find_via_ransac (relocalisation; test infrastructure only).
 * pose = {R row-major (9), t (3)} of cam_pose_cw: p_c = R p_w + t. */
#ifndef PNP_SOLVER_ORACLE_H
#define PNP_SOLVER_ORACLE_H
#include <stdint.h>

/* the sampler: m distinct indices of hypothesis k of n entries */
void op_ransac_sample(uint64_t seed, int k, int n, int m, int* idx);
/* cyclic Jacobi on a symmetric N x N A (N <= 12): the final diagonal and the eigenvectors as columns of V */
void op_jacobi(int N, const double* A, double* evals, double* V);
/* cos(pi / 180 * scale_factor) as the solver forms it */
double op_max_cos(float scale_factor);
/* EPnP on n >= 4 correspondences (bearings and world points, 3 per entry) */
void op_epnp(int n, const double* bearings, const double* pos_w, double* pose);
/* find_via_ransac on one problem; hyp_idx[max_num_iter * 6], hyp_pose[max_num_iter * 12], hyp_count[max_num_iter] may be NULL */
void op_pnp_solve_ransac(int n, const double* bearings, const double* pos_w, const float* scale_factor, int min_num_inliers,
                         int max_num_iter, int recompute, uint64_t seed, double* pose, int* valid, int* num_inliers, int* best_iter,
                         uint8_t* inlier_out, int* hyp_idx, double* hyp_pose, int* hyp_count);

#endif
