/* oracle/essential_solver_oracle.h -- CPU oracle for solve::essential_solver::find_via_ransac (tracking's robust match, map
 * initialisation; test infrastructure only).  A match is a pair of unit bearings (b1 in camera 1, b2 in camera 2);
 * E_21 row-major with b2^T E_21 b1 = 0. */
#ifndef ESSENTIAL_SOLVER_ORACLE_H
#define ESSENTIAL_SOLVER_ORACLE_H
#include <stdint.h>

/* the eight-point E_21 on the matches idx[0 .. n) (idx NULL: 0 .. n) of the per-match bearing arrays */
void oe_compute_E(int n, const double* b1, const double* b2, const int* idx, double* E);
/* check_inliers of E over n matches: the count, the flags (may be NULL) and the score in its fixed order */
int oe_check_inliers(const double* E, int n, const double* b1, const double* b2, uint8_t* flags, double* score);
/* find_via_ransac on one problem; hyp_idx[max_num_iter * 8], hyp_E[max_num_iter * 9], hyp_score[max_num_iter] and
 * hyp_count[max_num_iter] may be NULL */
void oe_essential_solve_ransac(int n, const double* b1, const double* b2, int max_num_iter, int recompute, uint64_t seed, double* E,
                               int* valid, int* num_inliers, int* best_iter, double* best_score, uint8_t* inlier_out, int* hyp_idx,
                               double* hyp_E, double* hyp_score, int* hyp_count);

#endif
