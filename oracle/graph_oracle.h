/* oracle/graph_oracle.h -- CPU oracle for optimize::graph_optimizer (loop closure pose graph over Sim3 vertices; test
 * infrastructure only).  sim3 = {R row-major (9), t (3), s}, S p = s R p + t; update = [omega, upsilon, sigma], S <- exp(d) S. */
#ifndef GRAPH_ORACLE_H
#define GRAPH_ORACLE_H
#include <stdint.h>
#include "ba_oracle.h"

void ob_sim3_inverse(const double* S, double* out);
void ob_sim3_compose(const double* A, const double* B, double* out);
void ob_sim3_log(const double* S, double* xi);
void ob_sim3_adjoint(const double* S, double* Ad);
void ob_sim3_ad(const double* xi, double* ad);
void ob_sim3_phi7(const double* A, double* F);
/* e = log(S_ji S_i S_j^-1) (7) and J = [J_i | J_j] (7 x 14 row-major, may be NULL) */
void ob_graph_edge(const double* S_ji, const double* S_i, const double* S_j, double* e, double* J);
/* graph_optimizer::optimize on K vertices (sim3_cw in / out), E edges, L landmarks (lm_pos_w in / out through lm_ref, -1 =
 * unchanged); pose_cw_out (K x 12) may be NULL.  Returns 0, or -1 for more free vertices than the dense solve takes. */
int ob_graph_optimize(int K, double* sim3_cw, const uint8_t* fixed, int E, const int32_t* edge_i, const int32_t* edge_j,
                      const double* meas_ji, int fix_scale, int num_iter, int L, double* lm_pos_w, const int32_t* lm_ref,
                      double* pose_cw_out, ob_stats* st);
#endif
