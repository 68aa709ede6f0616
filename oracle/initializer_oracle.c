/* initializer_oracle.c -- monocular map initialisation as recalled (DESIGN.md section 5): perspective::initialize (the homography
 * and fundamental-matrix solvers, the model choice S_H / (S_H + S_F) > 0.40), bearing_vector::initialize (the essential solver),
 * the three decompositions, check_pose and find_most_plausible_pose, one problem at a time.  The 3 x 3 SVD and the two-camera
 * triangulation take their eigenvectors from the oracle's cyclic Jacobi (op_jacobi). */
#include "initializer_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "essential_solver_oracle.h"
#include "pnp_solver_oracle.h"
#include "sim3_solver_oracle.h"
#include "two_view_solver_oracle.h"

#define OI_RANK_RATIO 1.00001
#define OI_SMALL_PARALLAX_COS 0.99998
#define OI_PARALLAX_RANK 50
#define OI_AMBIGUITY 0.8
#define OI_REL_SCORE_H 0.40

static void oi_mul(const double* A, const double* B, double* C) {   /* C = A B */
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

static void oi_mul_t(const double* A, const double* B, double* C) {   /* C = A B^T */
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}

static void oi_mv(const double* A, const double* v, double* o) {
    for (int i = 0; i < 3; ++i) o[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}

static double oi_det(const double* M) {
    return M[0] * (M[4] * M[8] - M[5] * M[7]) + M[1] * (M[5] * M[6] - M[3] * M[8]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

static void oi_unit(double* t) {
    const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    for (int r = 0; r < 3; ++r) t[r] /= n;
}

/* the Jacobi eigenvector of rank `rank` (descending or ascending, lowest index on ties), largest-magnitude entry positive */
static void oi_eigvec(int N, const double* ev, const double* V, int descending, int rank, double* v) {
    int used[4] = {0, 0, 0, 0}, m = -1;
    for (int r = 0; r <= rank; ++r) {
        m = -1;
        for (int k = 0; k < N; ++k) {
            if (used[k]) continue;
            if (m < 0 || (descending ? ev[k] > ev[m] : ev[k] < ev[m])) m = k;
        }
        used[m] = 1;
    }
    int a = 0;
    for (int r = 1; r < N; ++r) if (fabs(V[N * r + m]) > fabs(V[N * a + m])) a = r;
    const double sg = V[N * a + m] < 0.0 ? -1.0 : 1.0;
    for (int r = 0; r < N; ++r) v[r] = sg * V[N * r + m];
}

static double oi_eigval(int N, const double* ev, int descending, int rank) {
    int used[4] = {0, 0, 0, 0}, m = -1;
    for (int r = 0; r <= rank; ++r) {
        m = -1;
        for (int k = 0; k < N; ++k) {
            if (used[k]) continue;
            if (m < 0 || (descending ? ev[k] > ev[m] : ev[k] < ev[m])) m = k;
        }
        used[m] = 1;
    }
    return ev[m];
}

void oi_svd3(const double* A, int third_by_cross, double* U, double* d, double* V) {
    double G[9], ev[3], W[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) G[3 * i + j] = A[i] * A[j] + A[3 + i] * A[3 + j] + A[6 + i] * A[6 + j];
    op_jacobi(3, G, ev, W);
    for (int k = 0; k < 3; ++k) {
        double v[3];
        oi_eigvec(3, ev, W, 1, k, v);
        for (int r = 0; r < 3; ++r) V[3 * r + k] = v[r];
        const double l = oi_eigval(3, ev, 1, k);
        d[k] = l > 0.0 ? sqrt(l) : 0.0;
    }
    for (int k = 0; k < (third_by_cross ? 2 : 3); ++k) {
        const double v[3] = {V[k], V[3 + k], V[6 + k]};
        double a[3];
        oi_mv(A, v, a);
        for (int r = 0; r < 3; ++r) U[3 * r + k] = a[r] / d[k];
    }
    if (third_by_cross) {   /* u1 x u2 */
        U[2] = U[3] * U[7] - U[6] * U[4];
        U[5] = U[6] * U[1] - U[0] * U[7];
        U[8] = U[0] * U[4] - U[3] * U[1];
    }
}

static void oi_K(const ob_camera* c, double* K) {
    const double k[9] = {c->fx, 0.0, c->cx, 0.0, c->fy, c->cy, 0.0, 0.0, 1.0};
    memcpy(K, k, sizeof(k));
}

int oi_decompose_homography(const double* H, const ob_camera* cam_1, const ob_camera* cam_2, double* R, double* t, double* n) {
    const double K2i[9] = {1.0 / cam_2->fx, 0.0, -cam_2->cx / cam_2->fx, 0.0, 1.0 / cam_2->fy, -cam_2->cy / cam_2->fy, 0.0, 0.0, 1.0};
    double K1[9], T[9], A[9], U[9], d[3], V[9];
    oi_K(cam_1, K1);
    oi_mul(K2i, H, T);
    oi_mul(T, K1, A);
    oi_svd3(A, 0, U, d, V);
    const double d1 = d[0], d2 = d[1], d3 = d[2];
    if (d1 / d2 < OI_RANK_RATIO || d2 / d3 < OI_RANK_RATIO || isnan(d1 / d2) || isnan(d2 / d3)) return 0;
    const double s = oi_det(U) * oi_det(V);
    const double x1v = sqrt((d1 * d1 - d2 * d2) / (d1 * d1 - d3 * d3)), x3v = sqrt((d2 * d2 - d3 * d3) / (d1 * d1 - d3 * d3));
    const double x1[4] = {x1v, x1v, -x1v, -x1v}, x3[4] = {x3v, -x3v, x3v, -x3v};
    const double root = sqrt((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3));
    /* d' = d2 */
    const double sin_theta = root / ((d1 + d3) * d2), cos_theta = (d2 * d2 + d1 * d3) / ((d1 + d3) * d2);
    /* d' = -d2 */
    const double sin_phi = root / ((d1 - d3) * d2), cos_phi = (d1 * d3 - d2 * d2) / ((d1 - d3) * d2);
    for (int h = 0; h < 8; ++h) {
        const int i = h & 3, neg = h >> 2;
        const double sn = neg ? sin_phi : sin_theta;
        const double si = (i == 0 || i == 3) ? sn : -sn;
        double Rp[9] = {0};
        if (!neg) { Rp[0] = cos_theta; Rp[2] = -si; Rp[4] = 1.0; Rp[6] = si; Rp[8] = cos_theta; }
        else { Rp[0] = cos_phi; Rp[2] = si; Rp[4] = -1.0; Rp[6] = si; Rp[8] = -cos_phi; }
        double UR[9], M[9];
        oi_mul(U, Rp, UR);
        oi_mul_t(UR, V, M);
        for (int k = 0; k < 9; ++k) R[9 * h + k] = s * M[k];
        const double f = neg ? d1 + d3 : d1 - d3;
        const double tp[3] = {x1[i] * f, 0.0, (neg ? x3[i] : -x3[i]) * f};
        oi_mv(U, tp, t + 3 * h);
        oi_unit(t + 3 * h);
        if (n) {
            const double np[3] = {x1[i], 0.0, x3[i]};
            oi_mv(V, np, n + 3 * h);
            if (n[3 * h + 2] < 0.0) for (int r = 0; r < 3; ++r) n[3 * h + r] = -n[3 * h + r];
        }
    }
    return 1;
}

void oi_decompose_essential(const double* E, double* R, double* t) {
    double U[9], d[3], V[9];
    oi_svd3(E, 1, U, d, V);
    double u3[3] = {U[2], U[5], U[8]};
    oi_unit(u3);
    const double W[2][9] = {{0, -1, 0, 1, 0, 0, 0, 0, 1}, {0, 1, 0, -1, 0, 0, 0, 0, 1}};
    for (int w = 0; w < 2; ++w) {
        double UW[9], M[9];
        oi_mul(U, W[w], UW);
        oi_mul_t(UW, V, M);
        if (oi_det(M) < 0.0) for (int k = 0; k < 9; ++k) M[k] = -M[k];
        for (int s = 0; s < 2; ++s) {
            memcpy(R + 9 * (2 * w + s), M, sizeof(M));
            for (int r = 0; r < 3; ++r) t[3 * (2 * w + s) + r] = s ? -u3[r] : u3[r];
        }
    }
}

void oi_decompose_fundamental(const double* F, const ob_camera* cam_1, const ob_camera* cam_2, double* R, double* t) {
    double K2[9], K2t[9], K1[9], T[9], E[9];
    oi_K(cam_2, K2);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) K2t[3 * r + c] = K2[3 * c + r];
    oi_K(cam_1, K1);
    oi_mul(K2t, F, T);
    oi_mul(T, K1, E);
    oi_decompose_essential(E, R, t);
}

/* solve::triangulator::triangulate(b_ref, b_cur, [I | 0], [R | t]): the eigenvector of A^T A's smallest eigenvalue */
static void oi_triangulate(const double* b1, const double* b2, const double* Rt, double* pos) {
    static const double P1[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    double A[4][4], M[16], ev[4], V[16], v[4];
    for (int c = 0; c < 4; ++c) {
        const double p1[3] = {c < 3 ? P1[c] : P1[9], c < 3 ? P1[3 + c] : P1[10], c < 3 ? P1[6 + c] : P1[11]};
        const double p2[3] = {c < 3 ? Rt[c] : Rt[9], c < 3 ? Rt[3 + c] : Rt[10], c < 3 ? Rt[6 + c] : Rt[11]};
        A[0][c] = b1[0] * p1[2] - b1[2] * p1[0];
        A[1][c] = b1[1] * p1[2] - b1[2] * p1[1];
        A[2][c] = b2[0] * p2[2] - b2[2] * p2[0];
        A[3][c] = b2[1] * p2[2] - b2[2] * p2[1];
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) M[4 * i + j] = A[0][i] * A[0][j] + A[1][i] * A[1][j] + A[2][i] * A[2][j] + A[3][i] * A[3][j];
    op_jacobi(4, M, ev, V);
    oi_eigvec(4, ev, V, 0, 0, v);
    for (int r = 0; r < 3; ++r) pos[r] = v[r] / v[3];
}

int oi_check_match(const double* Rt, const ob_camera* cam_ref, const ob_camera* cam_cur, const double* b_ref, const double* b_cur,
                   const float* kp_ref, const float* kp_cur, double reproj_err_thr_sq, int depth_is_positive, double* p, float* cos_par) {
    static const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
    oi_triangulate(b_ref, b_cur, Rt, p);
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) return 2;
    /* the current camera's centre -R^T t */
    double c[3];
    for (int i = 0; i < 3; ++i) c[i] = -(Rt[i] * Rt[9] + Rt[3 + i] * Rt[10] + Rt[6 + i] * Rt[11]);
    const double q[3] = {p[0] - c[0], p[1] - c[1], p[2] - c[2]};
    const double np = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]), nq = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    const float cp = (float)((p[0] * q[0] + p[1] * q[1] + p[2] * q[2]) / (np * nq));
    *cos_par = cp;
    if (isnan(cp)) return 2;
    const int small = OI_SMALL_PARALLAX_COS < cp;
    if (depth_is_positive && !small) {
        if (p[2] <= 0.0) return 3;
        double pc[3];
        oi_mv(Rt, p, pc);
        if (pc[2] + Rt[11] <= 0.0) return 4;
    }
    double uv[2], ex, ey;
    if (!os_reproject(cam_ref, I, zero, p, uv)) return 5;
    ex = uv[0] - kp_ref[0]; ey = uv[1] - kp_ref[1];
    if (reproj_err_thr_sq < ex * ex + ey * ey) return 5;
    if (!os_reproject(cam_cur, Rt, Rt + 9, p, uv)) return 6;
    ex = uv[0] - kp_cur[0]; ey = uv[1] - kp_cur[1];
    if (reproj_err_thr_sq < ex * ex + ey * ey) return 6;
    return small ? 1 : 0;
}

int oi_choose(int nh, const int* count, const float* cos_par, int min_num_triangulated, double cos_thr, int* best) {
    int b = 0;
    for (int h = 1; h < nh; ++h) if (count[h] > count[b]) b = h;
    *best = b;
    if (count[b] < min_num_triangulated) return 3;
    int similar = 0;
    for (int h = 0; h < nh; ++h) if (OI_AMBIGUITY * count[b] < count[h]) ++similar;
    if (1 < similar) return 4;
    if (cos_thr < cos_par[b]) return 5;
    return 0;
}

static int oi_cmp_float(const void* a, const void* b) {
    const float x = *(const float*)a, y = *(const float*)b;
    return (x > y) - (x < y);
}

void oi_initialize(int perspective, const ob_camera* cam_ref, const ob_camera* cam_cur, int n_ref, const float* kp_ref,
                   const double* bear_ref, int n_cur, const float* kp_cur, const double* bear_cur, const int* ref_matches_with_cur,
                   int num_ransac_iters, int min_num_triangulated, float parallax_deg_thr, float reproj_err_thr_sq, uint64_t seed,
                   oi_result* res, double* hyp_R, double* hyp_t, int* reason, uint8_t* is_triangulated, double* pts) {
    memset(res, 0, sizeof(*res));
    int m = 0;
    for (int r = 0; r < n_ref; ++r) m += 0 <= ref_matches_with_cur[r];
    int* pairs = malloc(sizeof(int) * 2 * (m + 1));
    double* b1 = malloc(sizeof(double) * 3 * (m + 1));
    double* b2 = malloc(sizeof(double) * 3 * (m + 1));
    uint8_t* flags[2] = {calloc(m + 1, 1), calloc(m + 1, 1)};
    float* cps = malloc(sizeof(float) * (m + 1));
    for (int r = 0, i = 0; r < n_ref; ++r) {
        const int c = ref_matches_with_cur[r];
        if (c < 0) continue;
        pairs[2 * i] = r; pairs[2 * i + 1] = c;
        memcpy(b1 + 3 * i, bear_ref + 3 * r, 24); memcpy(b2 + 3 * i, bear_cur + 3 * c, 24);
        ++i;
    }
    int valid[2] = {0, 0};
    for (int s = 0; s < (perspective ? 2 : 1); ++s) {
        int v, num, best;
        if (perspective)
            ot_solve_ransac(s ? OT_MODEL_F : OT_MODEL_H, n_ref, kp_ref, n_cur, kp_cur, m, pairs, 1.0f, num_ransac_iters, 1, seed,
                            res->solver_M[s], &v, &num, &best, &res->solver_score[s], flags[s], NULL, NULL, NULL, NULL);
        else
            oe_essential_solve_ransac(m, b1, b2, num_ransac_iters, 1, seed, res->solver_M[s], &v, &num, &best, &res->solver_score[s],
                                      flags[s], NULL, NULL, NULL, NULL);
        valid[s] = v; res->solver_valid[s] = (uint8_t)v; res->solver_num_inliers[s] = num;
    }
    int model = 0;   /* none */
    if (perspective) {
        const double rel = res->solver_score[0] / (res->solver_score[0] + res->solver_score[1]);
        if (OI_REL_SCORE_H < rel && valid[0]) model = 1;
        else if (valid[1]) model = 2;
    } else if (valid[0]) {
        model = 3;
    }
    double R[72], t[24];
    int nh = 0;
    res->status = 1;
    if (model == 1) {
        if (oi_decompose_homography(res->solver_M[0], cam_ref, cam_cur, R, t, NULL)) nh = 8;
        else res->status = 2;
    } else if (model == 2) {
        oi_decompose_fundamental(res->solver_M[1], cam_ref, cam_cur, R, t);
        nh = 4;
    } else if (model == 3) {
        oi_decompose_essential(res->solver_M[0], R, t);
        nh = 4;
    }
    res->model = model; res->num_hypotheses = nh; res->chosen = -1;
    const uint8_t* inl = flags[model == 2 ? 1 : 0];
    const int dpos = perspective;
    for (int h = 0; h < 8; ++h) {
        int n = 0;
        for (int i = 0; i < m; ++i) {
            int code = -1;
            if (h < nh) {
                code = 7;
                if (inl[i]) {
                    double Rt[12], p[3];
                    float cp;
                    memcpy(Rt, R + 9 * h, 72); memcpy(Rt + 9, t + 3 * h, 24);
                    code = oi_check_match(Rt, cam_ref, cam_cur, b1 + 3 * i, b2 + 3 * i, kp_ref + 2 * pairs[2 * i], kp_cur + 2 * pairs[2 * i + 1],
                                          (double)reproj_err_thr_sq, dpos, p, &cp);
                    if (code <= 1) cps[n++] = cp;
                }
            }
            if (reason) reason[(size_t)h * m + i] = code;
        }
        res->num_valid[h] = n;
        res->cos_parallax[h] = 1.0f;
        if (n) {
            qsort(cps, n, sizeof(float), oi_cmp_float);
            res->cos_parallax[h] = cps[n - 1 < OI_PARALLAX_RANK ? n - 1 : OI_PARALLAX_RANK];
        }
    }
    if (nh) res->status = oi_choose(nh, res->num_valid, res->cos_parallax, min_num_triangulated,
                                    cos((double)parallax_deg_thr / 180.0 * M_PI), &res->chosen);
    if (hyp_R) { memset(hyp_R, 0, 72 * 8); if (nh) memcpy(hyp_R, R, 72 * nh); }
    if (hyp_t) { memset(hyp_t, 0, 24 * 8); if (nh) memcpy(hyp_t, t, 24 * nh); }
    double Rt[12];
    if (res->status == 0) {
        memcpy(Rt, R + 9 * res->chosen, 72); memcpy(Rt + 9, t + 3 * res->chosen, 24);
        memcpy(res->rot_ref_to_cur, Rt, 72); memcpy(res->trans_ref_to_cur, Rt + 9, 24);
    }
    memset(is_triangulated, 0, n_ref);
    memset(pts, 0, 24 * (size_t)n_ref);
    for (int r = 0, i = 0; r < n_ref; ++r) {
        if (ref_matches_with_cur[r] < 0) continue;
        if (res->status == 0 && inl[i]) {
            double p[3];
            float cp;
            if (oi_check_match(Rt, cam_ref, cam_cur, b1 + 3 * i, b2 + 3 * i, kp_ref + 2 * r, kp_cur + 2 * ref_matches_with_cur[r],
                               (double)reproj_err_thr_sq, dpos, p, &cp) == 0) {
                is_triangulated[r] = 1;
                memcpy(pts + 3 * r, p, 24);
            }
        }
        ++i;
    }
    free(pairs); free(b1); free(b2); free(flags[0]); free(flags[1]); free(cps);
}
