/*
 * oracle/graph_oracle.c -- CPU restatement (FP64) of OpenVSLAM's optimize::graph_optimizer::optimize (loop closure: the loop
 * correction spread over the keyframes' Sim3 poses, then every landmark moved with its reference keyframe) together with the g2o
 * parts it drives: OptimizationAlgorithmLevenberg with setUserLambdaInit(1e-16) over one Sim3 vertex per keyframe and EdgeSim3
 * (identity information, no robust kernel), as recalled.
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes (the same as openvslam_b200/csrc/sim3_math.cuh, restated operation for operation):
 *  - log is the exact inverse of ob_sim3_exp; the rotation angle is atan2(|vee(R - R')| / 2, (tr R - 1) / 2);
 *  - the Jacobians are analytic: J_i = J_l^-1(e) Ad(S_ji), J_j = -J_l^-1(e) Ad(E), J_l = phi(ad e) by scaling and squaring;
 *  - the system is dense (7 x free vertices), summed edge by edge in edge order; a free vertex without an edge stays out.
 * Checks: tests/test_graph_oracle.py (logm, expm, finite differences, scipy least_squares, an independent numpy step).
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "graph_oracle.h"
#include "sim3_oracle.h"

static void g_mat3_vec(const double* R, const double* v, double* o) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
static void g_mat3_mat3(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

void ob_sim3_inverse(const double* S, double* out) {
    const double is = 1.0 / S[12];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) out[3 * i + j] = S[3 * j + i];
    for (int k = 0; k < 3; ++k) out[9 + k] = -(S[k] * S[9] + S[3 + k] * S[10] + S[6 + k] * S[11]) * is;
    out[12] = is;
}

void ob_sim3_compose(const double* A, const double* B, double* out) {
    double q[3];
    g_mat3_mat3(A, B, out);
    g_mat3_vec(A, B + 9, q);
    for (int k = 0; k < 3; ++k) out[9 + k] = A[12] * q[k] + A[9 + k];
    out[12] = A[12] * B[12];
}

void ob_sim3_log(const double* S, double* xi) {
    const double* R = S;
    const double v[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    const double sn = 0.5 * sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
    const double theta = atan2(sn, c);
    if (c > -0.5) {
        const double f = theta < 1e-5 ? 0.5 : 0.5 * theta / sn;
        for (int k = 0; k < 3; ++k) xi[k] = f * v[k];
    } else {
        const double oc = 1.0 - c;
        const double B[9] = {R[0] - c, 0.5 * (R[1] + R[3]), 0.5 * (R[2] + R[6]),
                             0.5 * (R[3] + R[1]), R[4] - c, 0.5 * (R[5] + R[7]),
                             0.5 * (R[6] + R[2]), 0.5 * (R[7] + R[5]), R[8] - c};
        int k = 0;
        if (B[4] > B[0]) k = 1;
        if (B[8] > B[4 * k]) k = 2;
        const double ak = sqrt(B[4 * k] / oc);
        double a[3];
        for (int m = 0; m < 3; ++m) a[m] = (m == k) ? ak : B[3 * k + m] / (oc * ak);
        const double sg = (a[0] * v[0] + a[1] * v[1] + a[2] * v[2]) < 0.0 ? -1.0 : 1.0;
        for (int m = 0; m < 3; ++m) xi[m] = sg * theta * a[m];
    }
    xi[6] = log(S[12]);
    double W[9];
    for (int col = 0; col < 3; ++col) {
        double u[7] = {xi[0], xi[1], xi[2], 0.0, 0.0, 0.0, xi[6]}, E[13];
        u[3 + col] = 1.0;
        ob_sim3_exp(u, E);
        for (int r = 0; r < 3; ++r) W[3 * r + col] = E[9 + r];
    }
    const double c00 = W[4] * W[8] - W[5] * W[7], c01 = W[5] * W[6] - W[3] * W[8], c02 = W[3] * W[7] - W[4] * W[6];
    const double c10 = W[2] * W[7] - W[1] * W[8], c11 = W[0] * W[8] - W[2] * W[6], c12 = W[1] * W[6] - W[0] * W[7];
    const double c20 = W[1] * W[5] - W[2] * W[4], c21 = W[2] * W[3] - W[0] * W[5], c22 = W[0] * W[4] - W[1] * W[3];
    const double id = 1.0 / (W[0] * c00 + W[1] * c01 + W[2] * c02);
    const double* t = S + 9;
    xi[3] = (c00 * t[0] + c10 * t[1] + c20 * t[2]) * id;
    xi[4] = (c01 * t[0] + c11 * t[1] + c21 * t[2]) * id;
    xi[5] = (c02 * t[0] + c12 * t[1] + c22 * t[2]) * id;
}

void ob_sim3_adjoint(const double* S, double* Ad) {
    for (int k = 0; k < 49; ++k) Ad[k] = 0.0;
    const double* t = S + 9;
    const double T[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    double TR[9];
    g_mat3_mat3(T, S, TR);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            Ad[7 * i + j] = S[3 * i + j];
            Ad[7 * (3 + i) + j] = TR[3 * i + j];
            Ad[7 * (3 + i) + 3 + j] = S[12] * S[3 * i + j];
        }
        Ad[7 * (3 + i) + 6] = -t[i];
    }
    Ad[48] = 1.0;
}

void ob_sim3_ad(const double* xi, double* ad) {
    for (int k = 0; k < 49; ++k) ad[k] = 0.0;
    const double W[9] = {0, -xi[2], xi[1], xi[2], 0, -xi[0], -xi[1], xi[0], 0};
    const double U[9] = {0, -xi[5], xi[4], xi[5], 0, -xi[3], -xi[4], xi[3], 0};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            ad[7 * i + j] = W[3 * i + j];
            ad[7 * (3 + i) + j] = U[3 * i + j];
            ad[7 * (3 + i) + 3 + j] = W[3 * i + j] + (i == j ? xi[6] : 0.0);
        }
        ad[7 * (3 + i) + 6] = -xi[3 + i];
    }
}

static void g_mat7_mul(const double* A, const double* B, double* C) {
    for (int i = 0; i < 7; ++i)
        for (int j = 0; j < 7; ++j) {
            double s = 0.0;
            for (int k = 0; k < 7; ++k) s += A[7 * i + k] * B[7 * k + j];
            C[7 * i + j] = s;
        }
}

void ob_sim3_phi7(const double* A, double* F) {
    double nrm = 0.0;
    for (int i = 0; i < 7; ++i) {
        double r = 0.0;
        for (int j = 0; j < 7; ++j) r += fabs(A[7 * i + j]);
        nrm = fmax(nrm, r);
    }
    int sq = 0;
    double scale = 1.0;
    while (nrm * scale > 0.5 && sq < 64) { scale *= 0.5; ++sq; }
    double X[49], T[49];
    for (int k = 0; k < 49; ++k) X[k] = A[k] * scale;
    double inv_fact[13];
    inv_fact[0] = 1.0;
    for (int k = 1; k < 13; ++k) inv_fact[k] = inv_fact[k - 1] / (double)(k + 1);
    for (int k = 0; k < 49; ++k) F[k] = (k % 8 == 0) ? inv_fact[12] : 0.0;
    for (int k = 11; k >= 0; --k) {
        g_mat7_mul(X, F, T);
        for (int m = 0; m < 49; ++m) F[m] = T[m] + ((m % 8 == 0) ? inv_fact[k] : 0.0);
    }
    for (int s = 0; s < sq; ++s) {
        g_mat7_mul(X, F, T);
        for (int m = 0; m < 49; ++m) T[m] = 0.5 * T[m] + ((m % 8 == 0) ? 1.0 : 0.0);
        double Fn[49];
        g_mat7_mul(F, T, Fn);
        for (int m = 0; m < 49; ++m) { F[m] = Fn[m]; X[m] = 2.0 * X[m]; }
    }
}

static int g_solve7_general(double* M, double* B, int nrhs) {
    for (int c = 0; c < 7; ++c) {
        int p = c;
        for (int r = c + 1; r < 7; ++r)
            if (fabs(M[7 * r + c]) > fabs(M[7 * p + c])) p = r;
        if (!(fabs(M[7 * p + c]) > 0.0)) return 0;
        if (p != c) {
            for (int k = 0; k < 7; ++k) { const double tmp = M[7 * c + k]; M[7 * c + k] = M[7 * p + k]; M[7 * p + k] = tmp; }
            for (int k = 0; k < nrhs; ++k) { const double tmp = B[nrhs * c + k]; B[nrhs * c + k] = B[nrhs * p + k]; B[nrhs * p + k] = tmp; }
        }
        const double ip = 1.0 / M[8 * c];
        for (int r = c + 1; r < 7; ++r) {
            const double f = M[7 * r + c] * ip;
            if (f == 0.0) continue;
            for (int k = c; k < 7; ++k) M[7 * r + k] -= f * M[7 * c + k];
            for (int k = 0; k < nrhs; ++k) B[nrhs * r + k] -= f * B[nrhs * c + k];
        }
    }
    for (int c = 6; c >= 0; --c) {
        const double ip = 1.0 / M[8 * c];
        for (int k = 0; k < nrhs; ++k) {
            double s = B[nrhs * c + k];
            for (int m = c + 1; m < 7; ++m) s -= M[7 * c + m] * B[nrhs * m + k];
            B[nrhs * c + k] = s * ip;
        }
    }
    return 1;
}

void ob_graph_edge(const double* S_ji, const double* S_i, const double* S_j, double* e, double* J) {
    double Sji_i[13], Sj_inv[13], E[13];
    ob_sim3_compose(S_ji, S_i, Sji_i);
    ob_sim3_inverse(S_j, Sj_inv);
    ob_sim3_compose(Sji_i, Sj_inv, E);
    ob_sim3_log(E, e);
    if (!J) return;
    double Jl[49], ad[49], Ad1[49], Ad2[49];
    ob_sim3_ad(e, ad);
    ob_sim3_phi7(ad, Jl);
    ob_sim3_adjoint(S_ji, Ad1);
    ob_sim3_adjoint(E, Ad2);
    for (int r = 0; r < 7; ++r)
        for (int k = 0; k < 7; ++k) { J[14 * r + k] = Ad1[7 * r + k]; J[14 * r + 7 + k] = -Ad2[7 * r + k]; }
    if (!g_solve7_general(Jl, J, 14))
        for (int k = 0; k < 98; ++k) J[k] = 0.0;
}

typedef struct {
    int K, E, nfree, n, fix_scale;
    const int32_t *ei, *ej; const double* meas; const int* fidx;
} og_problem;

static double g_chi2(const og_problem* P, const double* S) {
    double total = 0.0;
    for (int e = 0; e < P->E; ++e) {
        double err[7], c = 0.0;
        ob_graph_edge(P->meas + 13 * (size_t)e, S + 13 * (size_t)P->ei[e], S + 13 * (size_t)P->ej[e], err, NULL);
        for (int k = 0; k < 7; ++k) c += err[k] * err[k];
        total += c;
    }
    return total;
}

/* H (n x n, full) and b = -J' e, summed edge by edge */
static void g_build(const og_problem* P, const double* S, double* H, double* b) {
    const size_t n = (size_t)P->n;
    memset(H, 0, n * n * sizeof(double));
    memset(b, 0, n * sizeof(double));
    for (int e = 0; e < P->E; ++e) {
        const int a = P->fidx[P->ei[e]], c = P->fidx[P->ej[e]];
        if (a < 0 && c < 0) continue;
        double err[7], J[98];
        ob_graph_edge(P->meas + 13 * (size_t)e, S + 13 * (size_t)P->ei[e], S + 13 * (size_t)P->ej[e], err, J);
        const int blk[2] = {a, c};
        for (int u = 0; u < 2; ++u) {
            if (blk[u] < 0) continue;
            for (int w = 0; w < 2; ++w) {
                if (blk[w] < 0) continue;
                for (int r = 0; r < 7; ++r)
                    for (int q = 0; q < 7; ++q) {
                        double h = 0.0;
                        for (int k = 0; k < 7; ++k) h += J[14 * k + 7 * u + r] * J[14 * k + 7 * w + q];
                        H[(7 * (size_t)blk[u] + r) * n + 7 * (size_t)blk[w] + q] += h;
                    }
            }
            for (int r = 0; r < 7; ++r) {
                double g = 0.0;
                for (int k = 0; k < 7; ++k) g += J[14 * k + 7 * u + r] * err[k];
                b[7 * (size_t)blk[u] + r] += -g;
            }
        }
    }
}

/* (H + lambda I) x = b by a dense Cholesky; -1 if not positive definite */
static int g_solve(const double* H, int n, double lambda, const double* b, double* x, double* Lm) {
    const size_t N = (size_t)n;
    for (size_t j = 0; j < N; ++j) {
        double d = H[j * N + j] + lambda;
        for (size_t k = 0; k < j; ++k) d -= Lm[j * N + k] * Lm[j * N + k];
        if (!(d > 0.0) || !isfinite(d)) return -1;
        d = sqrt(d);
        Lm[j * N + j] = d;
        for (size_t i = j + 1; i < N; ++i) {
            double s = H[i * N + j];
            for (size_t k = 0; k < j; ++k) s -= Lm[i * N + k] * Lm[j * N + k];
            Lm[i * N + j] = s / d;
        }
    }
    for (size_t i = 0; i < N; ++i) {
        double s = b[i];
        for (size_t k = 0; k < i; ++k) s -= Lm[i * N + k] * x[k];
        x[i] = s / Lm[i * N + i];
    }
    for (size_t ii = N; ii-- > 0;) {
        double s = x[ii];
        for (size_t k = ii + 1; k < N; ++k) s -= Lm[k * N + ii] * x[k];
        x[ii] = s / Lm[ii * N + ii];
    }
    return 0;
}

int ob_graph_optimize(int K, double* sim3_cw, const uint8_t* fixed, int E, const int32_t* edge_i, const int32_t* edge_j,
                      const double* meas_ji, int fix_scale, int num_iter, int L, double* lm_pos_w, const int32_t* lm_ref,
                      double* pose_cw_out, ob_stats* st) {
    if (st) memset(st, 0, sizeof(*st));
    int* fidx = (int*)malloc(sizeof(int) * (size_t)(K > 0 ? K : 1));
    uint8_t* used = (uint8_t*)calloc((size_t)(K > 0 ? K : 1), 1);
    for (int e = 0; e < E; ++e) { used[edge_i[e]] = 1; used[edge_j[e]] = 1; }
    int nfree = 0;
    for (int k = 0; k < K; ++k) fidx[k] = (used[k] && !fixed[k]) ? nfree++ : -1;
    free(used);
    if (7 * nfree > 6000) { free(fidx); return -1; }
    og_problem P = {K, E, nfree, 7 * nfree, fix_scale, edge_i, edge_j, meas_ji, fidx};
    const size_t sK = (size_t)K, n = (size_t)P.n;
    double* init = (double*)malloc(sizeof(double) * 13 * sK);
    memcpy(init, sim3_cw, sizeof(double) * 13 * sK);
    double* S = sim3_cw;
    if (nfree > 0 && num_iter > 0) {
        double* H = (double*)malloc(sizeof(double) * n * n);
        double* Lm = (double*)malloc(sizeof(double) * n * n);
        double* b = (double*)malloc(sizeof(double) * n);
        double* x = (double*)malloc(sizeof(double) * n);
        double* bak = (double*)malloc(sizeof(double) * 13 * sK);
        double lambda = 0, ni = 2;
        int it = 0, ok = 1;
        double currentChi = g_chi2(&P, S);
        for (; it < num_iter && ok; ++it) {
            g_build(&P, S, H, b);
            if (it == 0) {
                lambda = 1e-16;                 /* setUserLambdaInit */
                ni = 2;
                if (st) st->lambda_init[0] = lambda;
            }
            double rho = 0;
            int qmax = 0;
            do {
                memcpy(bak, S, sizeof(double) * 13 * sK);
                const int ok2 = g_solve(H, P.n, lambda, b, x, Lm) == 0;
                if (ok2)
                    for (int k = 0; k < K; ++k) {
                        if (fidx[k] < 0) continue;
                        double Sn[13];
                        ob_sim3_oplus(S + 13 * (size_t)k, x + 7 * (size_t)fidx[k], fix_scale, Sn);
                        memcpy(S + 13 * (size_t)k, Sn, sizeof(Sn));
                    }
                double tempChi = g_chi2(&P, S);
                if (!ok2) tempChi = DBL_MAX;
                rho = currentChi - tempChi;
                double scale = 0;
                if (ok2) for (size_t d = 0; d < n; ++d) scale += x[d] * (lambda * x[d] + b[d]);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && isfinite(tempChi)) {
                    double alpha = 1. - pow((2 * rho - 1), 3);
                    alpha = fmin(alpha, 2. / 3.);
                    lambda *= fmax(1. / 3., alpha);
                    ni = 2;
                    currentChi = tempChi;
                } else {
                    lambda *= ni;
                    ni *= 2;
                    memcpy(S, bak, sizeof(double) * 13 * sK);
                }
                qmax++;
                if (st) st->num_trials++;
            } while (rho < 0 && qmax < 10);
            if (st) { st->last_chi2 = currentChi; st->last_lambda = lambda; }
            if (qmax == 10 || rho == 0) ok = 0;
        }
        if (st) { st->num_iterations = it; st->round_iterations[0] = it; st->num_rounds = 1; st->final_chi2 = currentChi; }
        free(H); free(Lm); free(b); free(x); free(bak);
    }
    for (int l = 0; l < L; ++l) {
        const int r = lm_ref[l];
        if (r < 0) continue;
        double Si[13], q0[3], q1[3], pc[3];
        const double* S0 = init + 13 * (size_t)r;
        const double* p = lm_pos_w + 3 * (size_t)l;
        ob_sim3_inverse(S + 13 * (size_t)r, Si);
        g_mat3_vec(S0, p, q0);
        for (int q = 0; q < 3; ++q) pc[q] = S0[12] * q0[q] + S0[9 + q];
        g_mat3_vec(Si, pc, q1);
        for (int q = 0; q < 3; ++q) lm_pos_w[3 * (size_t)l + q] = Si[12] * q1[q] + Si[9 + q];
    }
    if (pose_cw_out)
        for (int k = 0; k < K; ++k) {
            for (int q = 0; q < 9; ++q) pose_cw_out[12 * (size_t)k + q] = S[13 * (size_t)k + q];
            for (int q = 0; q < 3; ++q) pose_cw_out[12 * (size_t)k + 9 + q] = S[13 * (size_t)k + 9 + q] / S[13 * (size_t)k + 12];
        }
    free(init); free(fidx);
    return 0;
}
