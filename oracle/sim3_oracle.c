/*
 * oracle/sim3_oracle.c -- CPU restatement (FP64) of OpenVSLAM's optimize::transform_optimizer::optimize (loop closure:
 * the Sim3 between the current keyframe and a loop candidate, refined on their mutual landmark matches) together with the
 * g2o parts it drives: OptimizationAlgorithmLevenberg (one vertex, so the 7 x 7 system is solved densely), RobustKernelHuber,
 * g2o::Sim3's exponential and the forward / backward reprojection edges (optimize/g2o/sim3/, as recalled).
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes:
 *  - the exponential follows the series of the true matrix exponential in its small-angle / small-scale branches;
 *  - the Jacobians are analytic (2 x 7, the sigma column included also with a fixed scale, so the damped system stays
 *    7 x 7 and fix_scale only zeroes update[6] inside oplus);
 *  - the outlier tests read the errors of the last evaluated trial, as g2o leaves them stored.
 * Checks: tests/test_transform_oracle.py (expm, finite differences, scipy least_squares, an independent numpy step).
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "sim3_oracle.h"

static void s3_mat3_vec(const double* R, const double* v, double* o) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
static void s3_mat3_mat3(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

/* g2o::Sim3(update): s = e^sigma, R = exp([omega]x), t = W upsilon, W = int_0^1 e^(sigma u) exp(u [omega]x) du
 * = C I + A O + B O^2.  Small branches: leading terms of the same series. */
void ob_sim3_exp(const double* u, double* S) {
    const double wx = u[0], wy = u[1], wz = u[2], sigma = u[6];
    const double theta = sqrt(wx * wx + wy * wy + wz * wz);
    const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    double O2[9];
    s3_mat3_mat3(O, O, O2);
    const double es = exp(sigma);
    double C;
    if (fabs(sigma) < 1e-5) C = 1.0 + sigma * (0.5 + sigma * (1.0 / 6.0));
    else C = expm1(sigma) / sigma;
    double ra, rb, A, B;
    if (theta < 1e-5) {
        ra = 1.0; rb = 0.5;
        if (fabs(sigma) < 1e-2) {
            A = 0.5 + sigma * (1.0 / 3.0 + sigma * (1.0 / 8.0 + sigma * (1.0 / 30.0 + sigma * (1.0 / 144.0))));
            B = 0.5 * (1.0 / 3.0 + sigma * (1.0 / 4.0 + sigma * (1.0 / 10.0 + sigma * (1.0 / 36.0 + sigma * (1.0 / 168.0)))));
        } else {
            A = (es * (sigma - 1.0) + 1.0) / (sigma * sigma);
            B = 0.5 * (es * (sigma * sigma - 2.0 * sigma + 2.0) - 2.0) / (sigma * sigma * sigma);
        }
    } else {
        const double st = sin(theta), ct = cos(theta);
        ra = st / theta;
        rb = (1.0 - ct) / (theta * theta);
        const double a = es * st, b = es * ct, c = theta * theta + sigma * sigma;
        A = (a * sigma + (1.0 - b) * theta) / (theta * c);
        B = (C - ((b - 1.0) * sigma + a * theta) / c) / (theta * theta);
    }
    double W[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i == 0 || i == 4 || i == 8) ? 1.0 : 0.0;
        S[i] = I + ra * O[i] + rb * O2[i];
        W[i] = C * I + A * O[i] + B * O2[i];
    }
    s3_mat3_vec(W, u + 3, S + 9);
    S[12] = es;
}

/* transform_vertex::oplusImpl: S <- exp(update) S, update[6] = 0 with a fixed scale */
void ob_sim3_oplus(const double* S, const double* xi, int fix_scale, double* out) {
    double u[7];
    for (int k = 0; k < 7; ++k) u[k] = xi[k];
    if (fix_scale) u[6] = 0.0;
    double E[13], Rn[9], q[3];
    ob_sim3_exp(u, E);
    s3_mat3_mat3(E, S, Rn);
    s3_mat3_vec(E, S + 9, q);
    for (int k = 0; k < 9; ++k) out[k] = Rn[k];
    for (int k = 0; k < 3; ++k) out[9 + k] = E[12] * q[k] + E[9 + k];
    out[12] = E[12] * S[12];
}

static void s3_project(const ob_camera* cam, const double* p, double* uv, double* P) {
    const double x = p[0], y = p[1], z = p[2];
    if (cam->model == OB_CAM_EQUIRECTANGULAR) {
        const double L = sqrt(x * x + y * y + z * z);
        const double theta = atan2(x, z);
        const double phi = -asin(y / L);
        uv[0] = cam->cols * (0.5 + theta / (2 * M_PI));
        uv[1] = cam->rows * (0.5 - phi / M_PI);
        if (P) {
            const double xz2 = x * x + z * z;
            const double c0 = (cam->cols / (2 * M_PI)) / xz2;
            const double c1 = (cam->rows / M_PI) / (L * sqrt(xz2));
            P[0] = c0 * z; P[1] = 0.0; P[2] = -c0 * x;
            P[3] = -c1 * (y * x / L); P[4] = c1 * (L - y * y / L); P[5] = -c1 * (y * z / L);
        }
        return;
    }
    uv[0] = cam->fx * x / z + cam->cx;
    uv[1] = cam->fy * y / z + cam->cy;
    if (P) {
        const double z_sq = z * z;
        P[0] = cam->fx / z; P[1] = 0.0; P[2] = -cam->fx * x / z_sq;
        P[3] = 0.0; P[4] = cam->fy / z; P[5] = -cam->fy * y / z_sq;
    }
}

static void s3_chain(const double* P, const double* D, double* J) {
    for (int r = 0; r < 2; ++r)
        for (int k = 0; k < 7; ++k) J[7 * r + k] = -(P[3 * r] * D[k] + P[3 * r + 1] * D[7 + k] + P[3 * r + 2] * D[14 + k]);
}

void ob_sim3_edge_forward(const ob_camera* cam1, const double* S, const double* pc2, const double* obs, double* e, double* J) {
    double q[3], p[3], uv[2], P[6];
    s3_mat3_vec(S, pc2, q);
    for (int k = 0; k < 3; ++k) p[k] = S[12] * q[k] + S[9 + k];
    s3_project(cam1, p, uv, J ? P : NULL);
    e[0] = obs[0] - uv[0];
    e[1] = obs[1] - uv[1];
    if (J) {
        const double x = p[0], y = p[1], z = p[2];
        const double D[21] = {0, z, -y, 1, 0, 0, x,
                              -z, 0, x, 0, 1, 0, y,
                              y, -x, 0, 0, 0, 1, z};
        s3_chain(P, D, J);
    }
}

void ob_sim3_edge_backward(const ob_camera* cam2, const double* S, const double* pc1, const double* obs, double* e, double* J) {
    const double is = 1.0 / S[12];
    const double d[3] = {pc1[0] - S[9], pc1[1] - S[10], pc1[2] - S[11]};
    double p[3], uv[2], P[6];
    for (int k = 0; k < 3; ++k) p[k] = (S[k] * d[0] + S[3 + k] * d[1] + S[6 + k] * d[2]) * is;
    s3_project(cam2, p, uv, J ? P : NULL);
    e[0] = obs[0] - uv[0];
    e[1] = obs[1] - uv[1];
    if (J) {
        const double x = pc1[0], y = pc1[1], z = pc1[2];
        const double M[21] = {0, -z, y, -1, 0, 0, -x,
                              z, 0, -x, 0, -1, 0, -y,
                              -y, x, 0, 0, 0, -1, -z};
        double D[21];
        for (int m = 0; m < 3; ++m)
            for (int k = 0; k < 7; ++k) D[7 * m + k] = (S[m] * M[k] + S[3 + m] * M[7 + k] + S[6 + m] * M[14 + k]) * is;
        s3_chain(P, D, J);
    }
}

/* ------------------------------------------------------------------------------- the optimiser */
typedef struct {
    const ob_camera *cam1, *cam2;
    const double *pose1, *pose2;
    int n;
    const double *pw1, *pw2;
    const float *xy1, *xy2, *w1, *w2;
    uint8_t* level;           /* per pair: 0 = both edges active, 1 = both at level 1 */
    double* err;              /* n x 4: e12 (2), e21 (2) as of the last evaluation */
    double delta;
    int fix_scale;
} os_problem;

static void s3_cam_point(const double* pose, const double* pw, double* pc) {
    s3_mat3_vec(pose, pw, pc);
    pc[0] += pose[9]; pc[1] += pose[10]; pc[2] += pose[11];
}
static void s3_obs(const float* xy, int i, double* o) { o[0] = (double)xy[2 * i]; o[1] = (double)xy[2 * i + 1]; }

static double s3_huber_rho(double e2, double delta, double* rho1) {
    const double dsqr = delta * delta;
    if (e2 <= dsqr) { *rho1 = 1.0; return e2; }
    const double sqrte = sqrt(e2);
    *rho1 = delta / sqrte;
    return 2 * sqrte * delta - dsqr;
}

/* computeActiveErrors + activeRobustChi2; with H / b: buildSystem at the same state */
static double s3_evaluate(os_problem* P, const double* S, double* H, double* b) {
    double total = 0;
    if (H) { memset(H, 0, 49 * sizeof(double)); memset(b, 0, 7 * sizeof(double)); }
    for (int i = 0; i < P->n; ++i) {
        if (P->level[i]) continue;
        double pc1[3], pc2[3], o1[2], o2[2], J[2][14];
        s3_cam_point(P->pose1, P->pw1 + 3 * (size_t)i, pc1);
        s3_cam_point(P->pose2, P->pw2 + 3 * (size_t)i, pc2);
        s3_obs(P->xy1, i, o1); s3_obs(P->xy2, i, o2);
        double* e = P->err + 4 * (size_t)i;
        ob_sim3_edge_forward(P->cam1, S, pc2, o1, e, H ? J[0] : NULL);
        ob_sim3_edge_backward(P->cam2, S, pc1, o2, e + 2, H ? J[1] : NULL);
        for (int k = 0; k < 2; ++k) {
            const double w = (double)(k == 0 ? P->w1[i] : P->w2[i]);
            const double* ek = e + 2 * k;
            const double chi = w * (ek[0] * ek[0] + ek[1] * ek[1]);
            double rho1;
            total += s3_huber_rho(chi, P->delta, &rho1);
            if (!H) continue;
            const double ww = rho1 * w;
            const double* Jk = J[k];
            for (int a = 0; a < 7; ++a) {
                b[a] -= Jk[a] * ww * ek[0] + Jk[7 + a] * ww * ek[1];
                for (int c = 0; c < 7; ++c) H[7 * a + c] += Jk[a] * ww * Jk[c] + Jk[7 + a] * ww * Jk[7 + c];
            }
        }
    }
    return total;
}

/* (H + lambda I) x = b by Cholesky; -1 if not positive definite */
static int s3_solve7(const double* H, double lambda, const double* b, double* x) {
    double L[49], y[7];
    for (int j = 0; j < 7; ++j) {
        double d = H[8 * j] + lambda;
        for (int k = 0; k < j; ++k) d -= L[7 * j + k] * L[7 * j + k];
        if (!(d > 0.0) || !isfinite(d)) return -1;
        d = sqrt(d);
        L[8 * j] = d;
        for (int i = j + 1; i < 7; ++i) {
            double s = H[7 * i + j];
            for (int k = 0; k < j; ++k) s -= L[7 * i + k] * L[7 * j + k];
            L[7 * i + j] = s / d;
        }
    }
    for (int i = 0; i < 7; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= L[7 * i + k] * y[k];
        y[i] = s / L[8 * i];
    }
    for (int i = 6; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < 7; ++k) s -= L[7 * k + i] * x[k];
        x[i] = s / L[8 * i];
    }
    return 0;
}

/* SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg on the one Sim3 vertex */
static int s3_lm(os_problem* P, double* S, int iterations, ob_stats* st) {
    double lambda = 0, ni = 2;
    double H[49], b[7];
    int it = 0, ok = 1;
    for (; it < iterations && ok; ++it) {
        double currentChi = s3_evaluate(P, S, H, b);
        if (it == 0) {
            double maxd = 0;
            for (int d = 0; d < 7; ++d) maxd = fmax(fabs(H[8 * d]), maxd);
            lambda = 1e-5 * maxd;
            ni = 2;
            if (st && st->num_rounds < OB_MAX_ROUNDS) st->lambda_init[st->num_rounds] = lambda;
        }
        double rho = 0;
        int qmax = 0;
        do {
            double bak[13], x[7];
            memcpy(bak, S, sizeof(bak));
            const int ok2 = s3_solve7(H, lambda, b, x) == 0;
            if (ok2) { double Sn[13]; ob_sim3_oplus(S, x, P->fix_scale, Sn); memcpy(S, Sn, sizeof(Sn)); }
            double tempChi = s3_evaluate(P, S, NULL, NULL);
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0;
            if (ok2) for (int d = 0; d < 7; ++d) scale += x[d] * (lambda * x[d] + b[d]);   /* all seven, fixed scale or not */
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
                memcpy(S, bak, sizeof(bak));
            }
            qmax++;
            if (st) st->num_trials++;
        } while (rho < 0 && qmax < 10);
        if (st) { st->last_chi2 = currentChi; st->last_lambda = lambda; }
        if (qmax == 10 || rho == 0) ok = 0;
    }
    if (st) { st->num_iterations += it; if (st->num_rounds < OB_MAX_ROUNDS) st->round_iterations[st->num_rounds] = it; st->num_rounds++; }
    return it;
}

/* chi_sq < e12' W e12 || chi_sq < e21' W e21 on the stored errors */
static int s3_pair_is_outlier(const os_problem* P, int i, double chi_sq) {
    const double* e = P->err + 4 * (size_t)i;
    const double c12 = (double)P->w1[i] * (e[0] * e[0] + e[1] * e[1]);
    const double c21 = (double)P->w2[i] * (e[2] * e[2] + e[3] * e[3]);
    return chi_sq < c12 || chi_sq < c21;
}

int ob_transform_optimize(const ob_camera* cam_1, const ob_camera* cam_2, const double* pose_1w, const double* pose_2w, int n,
                          const double* pos_w_1, const float* obs_xy_1, const float* inv_sigma_sq_1, const double* pos_w_2,
                          const float* obs_xy_2, const float* inv_sigma_sq_2, int fix_scale, float chi_sq, int num_first_iter,
                          int num_iter, double* sim3_12, uint8_t* inlier_out, ob_stats* st) {
    if (st) memset(st, 0, sizeof(*st));
    if (n <= 0) return 0;
    os_problem P;
    P.cam1 = cam_1; P.cam2 = cam_2; P.pose1 = pose_1w; P.pose2 = pose_2w; P.n = n;
    P.pw1 = pos_w_1; P.pw2 = pos_w_2; P.xy1 = obs_xy_1; P.xy2 = obs_xy_2; P.w1 = inv_sigma_sq_1; P.w2 = inv_sigma_sq_2;
    P.level = (uint8_t*)calloc((size_t)n, 1);
    P.err = (double*)calloc(4 * (size_t)n, sizeof(double));
    P.delta = (double)sqrtf(chi_sq);
    P.fix_scale = fix_scale;
    const double thr = (double)chi_sq;
    double S[13];
    memcpy(S, sim3_12, sizeof(S));

    s3_lm(&P, S, num_first_iter, st);
    int num_outliers = 0;
    for (int i = 0; i < n; ++i)
        if (s3_pair_is_outlier(&P, i, thr)) { P.level[i] = 1; ++num_outliers; }
    int num_inliers = 0;
    if (n - num_outliers >= 10) {
        s3_lm(&P, S, num_iter, st);
        for (int i = 0; i < n; ++i) {
            if (P.level[i]) continue;
            if (s3_pair_is_outlier(&P, i, thr)) P.level[i] = 1;
            else ++num_inliers;
        }
        memcpy(sim3_12, S, sizeof(S));
    }
    for (int i = 0; i < n; ++i) inlier_out[i] = P.level[i] ? 0 : 1;
    if (st) {
        st->final_chi2 = 0;
        for (int i = 0; i < n; ++i) {
            if (P.level[i]) continue;
            const double* e = P.err + 4 * (size_t)i;
            st->final_chi2 += (double)P.w1[i] * (e[0] * e[0] + e[1] * e[1]) + (double)P.w2[i] * (e[2] * e[2] + e[3] * e[3]);
        }
    }
    free(P.level); free(P.err);
    return num_inliers;
}
