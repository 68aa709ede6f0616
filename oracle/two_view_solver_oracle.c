/*
 * oracle/two_view_solver_oracle.c -- CPU restatement (float normalisation, FP64 solves) of OpenVSLAM's solve::homography_solver and
 * solve::fundamental_solver (the homography H_21 and the fundamental matrix F_21 of two views from keypoint matches, by RANSAC over
 * the 8-point DLT and the eight-point algorithm: perspective map initialisation), constructor and find_via_ransac(max_num_iter,
 * recompute), restated from memory.
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes (the kernels' csrc/two_view_math.cuh follows them operation for operation):
 *  - normalize per view over ALL its keypoints, in float: mean = running sum / (float)n, dev = running sum of |x - mean| / (float)n,
 *    inv = (float)(1.0 / (double)dev), normalised = (x - mean) * inv; T = [[inv_x, 0, -mean_x * inv_x (float)], [0, inv_y, ..],
 *    [0, 0, 1]];
 *  - the sampler is the counter-based one of the other solvers (op_ransac_sample, m = 8), seeded per problem;
 *  - H: per match the DLT rows r0 = [0, 0, 0, -x1, -y1, -1, y2 x1, y2 y1, y2], r1 = [x1, y1, 1, 0, 0, 0, -x2 x1, -x2 y1, -x2]
 *    (doubles from the float normalised points), one summation item r0_a r0_b + r1_a r1_b per upper entry of A^T A;
 *    F: the row [x2 x1, x2 y1, x2, y2 x1, y2 y1, y2, x1, y1, 1];
 *  - A^T A over more than 256 items takes 256 strided partials from 0, then their running sum (for n <= 256 the plain running
 *    sum), as the device's CTA-wide reduction does; the model is the eigenvector of the smallest eigenvalue (op_jacobi, lowest
 *    index on ties), read row-major;
 *  - F rank 2: F0 - (F0 v3) v3^T with v3 the smallest eigenvector of F0^T F0 (op_jacobi on 3 x 3, lowest index on ties);
 *  - denormalisation: H_21 = T2inv H T1 with T2inv = [[1 / inv_x, 0, mean_x], [0, 1 / inv_y, mean_y], [0, 0, 1]], F_21 = T2^T F T1,
 *    3 x 3 products left to right; then the entry of largest magnitude (first on ties) made positive;
 *  - check_inliers in double (the reference uses float): H by symmetric transfer (H_12 = adjugate / det) against 5.991f, F by the
 *    squared distance to both epipolar lines against 3.841f; each passing direction adds 5.991f - chi^2 (the first stays when the
 *    second fails); the tests are thr < chi, so a NaN passes and the score is NaN; the score is summed as 32 partials over the
 *    matches l, l + 32, .. then in order; inv_sigma_sq = (float)(1.0 / (double)(sigma * sigma));
 *  - the best hypothesis is the first whose score is strictly greater than the best so far (from 0); valid = best score > 0
 *    and at least 8 inliers; recompute (when valid) refits on all inliers in index order and re-checks.
 * Checks: tests/test_two_view_solvers_oracle.py (numpy restatements with SVDs, the truth, cv2, the kernel header compiled for the
 * host).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "pnp_solver_oracle.h"
#include "two_view_solver_oracle.h"

#define OT_MIN_SET 8
#define OT_SLOTS 256
#define OT_LANES 32

void ot_normalize(int n, const float* xy, float* norm, float* T4) {
    float mx = 0.f, my = 0.f, dx = 0.f, dy = 0.f;
    for (int i = 0; i < n; ++i) {
        mx += xy[2 * i];
        my += xy[2 * i + 1];
    }
    mx = mx / (float)n;
    my = my / (float)n;
    for (int i = 0; i < n; ++i) {
        dx += fabsf(xy[2 * i] - mx);
        dy += fabsf(xy[2 * i + 1] - my);
    }
    dx = dx / (float)n;
    dy = dy / (float)n;
    const float ix = (float)(1.0 / (double)dx), iy = (float)(1.0 / (double)dy);
    for (int i = 0; i < n; ++i) {
        norm[2 * i] = (xy[2 * i] - mx) * ix;
        norm[2 * i + 1] = (xy[2 * i + 1] - my) * iy;
    }
    T4[0] = mx; T4[1] = my; T4[2] = ix; T4[3] = iy;
}

static void ot_item(int model, const float* q1, const float* q2, double* v) {
    const double x1 = q1[0], y1 = q1[1], x2 = q2[0], y2 = q2[1];
    int q = 0;
    if (model == OT_MODEL_H) {
        const double r0[9] = {0.0, 0.0, 0.0, -x1, -y1, -1.0, y2 * x1, y2 * y1, y2};
        const double r1[9] = {x1, y1, 1.0, 0.0, 0.0, 0.0, -x2 * x1, -x2 * y1, -x2};
        for (int r = 0; r < 9; ++r)
            for (int c = r; c < 9; ++c) v[q++] = r0[r] * r0[c] + r1[r] * r1[c];
    } else {
        const double a[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
        for (int r = 0; r < 9; ++r)
            for (int c = r; c < 9; ++c) v[q++] = a[r] * a[c];
    }
}

static void ot_mul3(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

static void ot_T(const float* T4, double* T) {
    T[0] = T4[2]; T[1] = 0.0; T[2] = (double)(-T4[0] * T4[2]);
    T[3] = 0.0; T[4] = T4[3]; T[5] = (double)(-T4[1] * T4[3]);
    T[6] = 0.0; T[7] = 0.0; T[8] = 1.0;
}

void ot_compute(int model, int n, const float* norm_1, const float* norm_2, const int* pairs, const int* idx, const float* T4_1,
                const float* T4_2, double* M) {
    double up[45], v[45], s[45];
    for (int c = 0; c < 45; ++c) up[c] = 0.0;
#define OT_ITEM(i)                                                                                   \
    do {                                                                                             \
        const int m_ = idx ? idx[i] : (i);                                                           \
        ot_item(model, norm_1 + 2 * pairs[2 * m_], norm_2 + 2 * pairs[2 * m_ + 1], v);               \
    } while (0)
    if (n <= OT_SLOTS) {
        for (int i = 0; i < n; ++i) {
            OT_ITEM(i);
            for (int c = 0; c < 45; ++c) up[c] += v[c];
        }
    } else {
        for (int t = 0; t < OT_SLOTS; ++t) {
            for (int c = 0; c < 45; ++c) s[c] = 0.0;
            for (int i = t; i < n; i += OT_SLOTS) {
                OT_ITEM(i);
                for (int c = 0; c < 45; ++c) s[c] += v[c];
            }
            for (int c = 0; c < 45; ++c) up[c] += s[c];
        }
    }
#undef OT_ITEM
    double A[81], ev[9], V[81];
    int q = 0;
    for (int r = 0; r < 9; ++r)
        for (int c = r; c < 9; ++c) { A[9 * r + c] = up[q]; A[9 * c + r] = up[q]; ++q; }
    op_jacobi(9, A, ev, V);
    int mi = 0;
    for (int k = 1; k < 9; ++k)
        if (ev[k] < ev[mi]) mi = k;
    double X[9], L[9], T1[9], Y[9];
    for (int k = 0; k < 9; ++k) X[k] = V[9 * k + mi];
    ot_T(T4_1, T1);
    if (model == OT_MODEL_H) {
        L[0] = 1.0 / (double)T4_2[2]; L[1] = 0.0; L[2] = T4_2[0];
        L[3] = 0.0; L[4] = 1.0 / (double)T4_2[3]; L[5] = T4_2[1];
        L[6] = 0.0; L[7] = 0.0; L[8] = 1.0;
    } else {
        double G[9], gev[3], W[9], v3[3], u[3], T2[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) G[3 * i + j] = X[i] * X[j] + X[3 + i] * X[3 + j] + X[6 + i] * X[6 + j];
        op_jacobi(3, G, gev, W);
        int s3 = 0;
        for (int k = 1; k < 3; ++k)
            if (gev[k] < gev[s3]) s3 = k;
        for (int r = 0; r < 3; ++r) v3[r] = W[3 * r + s3];
        for (int r = 0; r < 3; ++r) u[r] = X[3 * r] * v3[0] + X[3 * r + 1] * v3[1] + X[3 * r + 2] * v3[2];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) X[3 * r + c] = X[3 * r + c] - u[r] * v3[c];
        ot_T(T4_2, T2);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) L[3 * r + c] = T2[3 * c + r];
    }
    ot_mul3(L, X, Y);
    ot_mul3(Y, T1, M);
    int a = 0;
    for (int k = 1; k < 9; ++k)
        if (fabs(M[k]) > fabs(M[a])) a = k;
    if (M[a] < 0.0)
        for (int k = 0; k < 9; ++k) M[k] = -M[k];
}

static const double ot_score_thr = (double)5.991f;
static const double ot_chi_f = (double)3.841f;

/* chi^2 of the transfer of src by G against dst */
static double ot_transfer(const double* G, const float* src, const float* dst, double iss) {
    const double p[3] = {src[0], src[1], 1.0};
    double q[3];
    for (int r = 0; r < 3; ++r) q[r] = G[3 * r] * p[0] + G[3 * r + 1] * p[1] + G[3 * r + 2] * p[2];
    const double w = q[2];
    for (int r = 0; r < 3; ++r) q[r] = q[r] / w;
    const double dx = (double)dst[0] - q[0], dy = (double)dst[1] - q[1], dz = 1.0 - q[2];
    return (dx * dx + dy * dy + dz * dz) * iss;
}

/* chi^2 of the point k against the line l */
static double ot_line(const double* l, const float* k, double iss) {
    const double d = l[0] * (double)k[0] + l[1] * (double)k[1] + l[2] * 1.0;
    return d * d / (l[0] * l[0] + l[1] * l[1]) * iss;
}

static void ot_inverse(const double* H, double* o) {
    const double a = H[0], b = H[1], c = H[2], d = H[3], e = H[4], f = H[5], g = H[6], h = H[7], i = H[8];
    const double c0 = e * i - f * h, c1 = f * g - d * i, c2 = d * h - e * g;
    const double det = a * c0 + b * c1 + c * c2;
    o[0] = c0 / det; o[1] = (c * h - b * i) / det; o[2] = (b * f - c * e) / det;
    o[3] = c1 / det; o[4] = (a * i - c * g) / det; o[5] = (c * d - a * f) / det;
    o[6] = c2 / det; o[7] = (b * g - a * h) / det; o[8] = (a * e - b * d) / det;
}

/* one match: whether it is an inlier; the passing directions' terms are added to *score in order */
static int ot_check_one(int model, const double* M, const double* Minv, const float* k1, const float* k2, double iss, double* score) {
    double chi1, chi2, thr;
    if (model == OT_MODEL_H) {
        thr = ot_score_thr;
        chi1 = ot_transfer(M, k1, k2, iss);
        if (thr < chi1) return 0;
        *score += ot_score_thr - chi1;
        chi2 = ot_transfer(Minv, k2, k1, iss);
    } else {
        const double p1[3] = {k1[0], k1[1], 1.0}, p2[3] = {k2[0], k2[1], 1.0};
        double l2[3], l1[3];
        thr = ot_chi_f;
        for (int r = 0; r < 3; ++r) l2[r] = M[3 * r] * p1[0] + M[3 * r + 1] * p1[1] + M[3 * r + 2] * p1[2];
        chi1 = ot_line(l2, k2, iss);
        if (thr < chi1) return 0;
        *score += ot_score_thr - chi1;
        for (int c = 0; c < 3; ++c) l1[c] = M[c] * p2[0] + M[3 + c] * p2[1] + M[6 + c] * p2[2];
        chi2 = ot_line(l1, k1, iss);
    }
    if (thr < chi2) return 0;
    *score += ot_score_thr - chi2;
    return 1;
}

int ot_check_inliers(int model, const double* M, int n, const float* xy_1, const float* xy_2, const int* pairs, float sigma,
                     uint8_t* flags, double* score) {
    const double iss = (double)(float)(1.0 / (double)(sigma * sigma));
    double Minv[9];
    if (model == OT_MODEL_H) ot_inverse(M, Minv);
    int count = 0;
    double total = 0.0;
    for (int l = 0; l < OT_LANES; ++l) {
        double part = 0.0;
        for (int i = l; i < n; i += OT_LANES) {
            const int in = ot_check_one(model, M, Minv, xy_1 + 2 * pairs[2 * i], xy_2 + 2 * pairs[2 * i + 1], iss, &part);
            if (flags) flags[i] = (uint8_t)in;
            count += in;
        }
        total += part;
    }
    *score = total;
    return count;
}

void ot_solve_ransac(int model, int n1, const float* xy_1, int n2, const float* xy_2, int n, const int* pairs, float sigma,
                     int max_num_iter, int recompute, uint64_t seed, double* M, int* valid, int* num_inliers, int* best_iter,
                     double* best_score, uint8_t* inlier_out, int* hyp_idx, double* hyp_M, double* hyp_score, int* hyp_count) {
    for (int k = 0; k < 9; ++k) M[k] = 0.0;
    *valid = 0; *num_inliers = 0; *best_iter = -1; *best_score = 0.0;
    for (int i = 0; i < n; ++i) inlier_out[i] = 0;
    if (hyp_idx) for (int k = 0; k < OT_MIN_SET * max_num_iter; ++k) hyp_idx[k] = -1;
    if (hyp_M) for (int k = 0; k < 9 * max_num_iter; ++k) hyp_M[k] = 0.0;
    if (hyp_score) for (int k = 0; k < max_num_iter; ++k) hyp_score[k] = 0.0;
    if (hyp_count) for (int k = 0; k < max_num_iter; ++k) hyp_count[k] = 0;
    if (n < OT_MIN_SET) return;
    float* nm1 = (float*)malloc(sizeof(float) * 2 * (size_t)(n1 > 0 ? n1 : 1));
    float* nm2 = (float*)malloc(sizeof(float) * 2 * (size_t)(n2 > 0 ? n2 : 1));
    float T1[4], T2[4];
    ot_normalize(n1, xy_1, nm1, T1);
    ot_normalize(n2, xy_2, nm2, T2);
    uint8_t* flags = (uint8_t*)malloc((size_t)n);
    double best = 0.0;
    int best_k = -1, best_cnt = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        int idx[OT_MIN_SET];
        op_ransac_sample(seed, k, n, OT_MIN_SET, idx);
        double Mk[9], sc;
        ot_compute(model, OT_MIN_SET, nm1, nm2, pairs, idx, T1, T2, Mk);
        const int cnt = ot_check_inliers(model, Mk, n, xy_1, xy_2, pairs, sigma, flags, &sc);
        if (hyp_idx) memcpy(hyp_idx + OT_MIN_SET * k, idx, sizeof(idx));
        if (hyp_M) memcpy(hyp_M + 9 * k, Mk, sizeof(Mk));
        if (hyp_score) hyp_score[k] = sc;
        if (hyp_count) hyp_count[k] = cnt;
        if (best < sc) {
            best = sc; best_k = k; best_cnt = cnt;
            memcpy(M, Mk, sizeof(Mk));
            memcpy(inlier_out, flags, (size_t)n);
        }
    }
    free(flags);
    *best_iter = best_k;
    *best_score = best;
    *num_inliers = best_cnt;
    *valid = (best > 0.0 && best_cnt >= OT_MIN_SET) ? 1 : 0;
    if (*valid && recompute) {
        int* inl = (int*)malloc(sizeof(int) * (size_t)n);
        int m = 0;
        for (int i = 0; i < n; ++i)
            if (inlier_out[i]) inl[m++] = i;
        ot_compute(model, m, nm1, nm2, pairs, inl, T1, T2, M);
        free(inl);
        *num_inliers = ot_check_inliers(model, M, n, xy_1, xy_2, pairs, sigma, inlier_out, best_score);
    }
    free(nm1);
    free(nm2);
}
