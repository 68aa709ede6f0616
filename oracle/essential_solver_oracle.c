/*
 * oracle/essential_solver_oracle.c -- CPU restatement (FP64) of OpenVSLAM's solve::essential_solver (the essential matrix E_21 of
 * two views from bearing matches, by RANSAC over the eight-point algorithm: the tracker's robust match and equirectangular map
 * initialisation), constructor and find_via_ransac(max_num_iter, recompute), restated from memory.
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes (the kernel's csrc/essential_math.cuh follows them operation for operation):
 *  - the sampler is the counter-based one of the other solvers (op_ransac_sample, m = 8), seeded per problem;
 *  - the eight-point E: rows a = b2 (x) b1, M = A^T A (45 upper entries), e = the eigenvector of M's smallest eigenvalue by the
 *    cyclic Jacobi (op_jacobi; lowest index on ties); rank 2 by U diag(s, s, 0) V^T formed from the eigenpairs of E^T E
 *    (s = the mean of the two largest singular values; E' = 0 unless the second is positive); the entry of largest magnitude
 *    (first on ties) made positive;
 *  - A^T A over more than 256 matches takes 256 strided partials from 0, then their running sum (for n <= 256 the plain running
 *    sum), as the device's CTA-wide reduction does;
 *  - check_inliers: r2 = |(E b1) . b2| / |E b1| against sin(1 deg) first, then r1 = |(E^T b2) . b1| / |E^T b2|; each passing
 *    residual joins the score (r2 stays when r1 fails); the tests are !(thr < r), so a zero norm passes and the score is NaN;
 *    the score is a double summed as 32 partials over the matches l, l + 32, .. then in order (the reference sums in float);
 *  - the best hypothesis is the first whose score is strictly greater than the best so far (from 0); valid = best score > 0
 *    and at least 8 inliers; recompute (when valid) refits on all inliers in index order and re-checks.
 * Checks: tests/test_essential_solver_oracle.py (a numpy restatement with SVDs, the truth, cv2.decomposeEssentialMat, the
 * kernel header compiled for the host).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "essential_solver_oracle.h"
#include "pnp_solver_oracle.h"

#define OE_MIN_SET 8
#define OE_SLOTS 256
#define OE_LANES 32
static const double oe_thr = 0.01745240643;

static void oe_row(const double* b1, const double* b2, double* v) {
    double a[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) a[3 * r + c] = b2[r] * b1[c];
    int q = 0;
    for (int r = 0; r < 9; ++r)
        for (int c = r; c < 9; ++c) v[q++] = a[r] * a[c];
}

void oe_compute_E(int n, const double* b1, const double* b2, const int* idx, double* E) {
    double up[45], v[45], s[45];
    for (int c = 0; c < 45; ++c) up[c] = 0.0;
    if (n <= OE_SLOTS) {
        for (int i = 0; i < n; ++i) {
            const int m = idx ? idx[i] : i;
            oe_row(b1 + 3 * m, b2 + 3 * m, v);
            for (int c = 0; c < 45; ++c) up[c] += v[c];
        }
    } else {
        for (int t = 0; t < OE_SLOTS; ++t) {
            for (int c = 0; c < 45; ++c) s[c] = 0.0;
            for (int i = t; i < n; i += OE_SLOTS) {
                const int m = idx ? idx[i] : i;
                oe_row(b1 + 3 * m, b2 + 3 * m, v);
                for (int c = 0; c < 45; ++c) s[c] += v[c];
            }
            for (int c = 0; c < 45; ++c) up[c] += s[c];
        }
    }
    double M[81], ev[9], V[81];
    int q = 0;
    for (int r = 0; r < 9; ++r)
        for (int c = r; c < 9; ++c) { M[9 * r + c] = up[q]; M[9 * c + r] = up[q]; ++q; }
    op_jacobi(9, M, ev, V);
    int mi = 0;
    for (int k = 1; k < 9; ++k)
        if (ev[k] < ev[mi]) mi = k;
    double E0[9];
    for (int k = 0; k < 9; ++k) E0[k] = V[9 * k + mi];
    double G[9], gev[3], W[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) G[3 * i + j] = E0[i] * E0[j] + E0[3 + i] * E0[3 + j] + E0[6 + i] * E0[6 + j];
    op_jacobi(3, G, gev, W);
    /* descending, lowest index on ties */
    int o1 = 0;
    for (int k = 1; k < 3; ++k)
        if (gev[k] > gev[o1]) o1 = k;
    int o2 = -1;
    for (int k = 0; k < 3; ++k) {
        if (k == o1) continue;
        if (o2 < 0 || gev[k] > gev[o2]) o2 = k;
    }
    const double l1 = gev[o1], l2 = gev[o2];
    const double s1 = sqrt(l1 > 0.0 ? l1 : 0.0), s2 = sqrt(l2 > 0.0 ? l2 : 0.0);
    if (!(s2 > 0.0)) {
        for (int k = 0; k < 9; ++k) E[k] = 0.0;
        return;
    }
    const double sm = (s1 + s2) / 2.0;
    double v1[3], v2[3], u1[3], u2[3];
    for (int r = 0; r < 3; ++r) { v1[r] = W[3 * r + o1]; v2[r] = W[3 * r + o2]; }
    for (int r = 0; r < 3; ++r) {
        u1[r] = E0[3 * r] * v1[0] + E0[3 * r + 1] * v1[1] + E0[3 * r + 2] * v1[2];
        u2[r] = E0[3 * r] * v2[0] + E0[3 * r + 1] * v2[1] + E0[3 * r + 2] * v2[2];
    }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) E[3 * r + c] = sm * (u1[r] * v1[c] / s1 + u2[r] * v2[c] / s2);
    int a = 0;
    for (int k = 1; k < 9; ++k)
        if (fabs(E[k]) > fabs(E[a])) a = k;
    if (E[a] < 0.0)
        for (int k = 0; k < 9; ++k) E[k] = -E[k];
}

/* one match: returns whether it is an inlier; the passing residuals are added to *score in order (r2, then r1) */
static int oe_check_one(const double* E, const double* b1, const double* b2, double* score) {
    double e1[3], e2[3];
    for (int r = 0; r < 3; ++r) e1[r] = E[3 * r] * b1[0] + E[3 * r + 1] * b1[1] + E[3 * r + 2] * b1[2];
    const double r2 = fabs(e1[0] * b2[0] + e1[1] * b2[1] + e1[2] * b2[2]) / sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
    if (oe_thr < r2) return 0;
    *score += r2;
    for (int c = 0; c < 3; ++c) e2[c] = E[c] * b2[0] + E[3 + c] * b2[1] + E[6 + c] * b2[2];
    const double r1 = fabs(e2[0] * b1[0] + e2[1] * b1[1] + e2[2] * b1[2]) / sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    if (oe_thr < r1) return 0;
    *score += r1;
    return 1;
}

int oe_check_inliers(const double* E, int n, const double* b1, const double* b2, uint8_t* flags, double* score) {
    int count = 0;
    double total = 0.0;
    for (int l = 0; l < OE_LANES; ++l) {
        double part = 0.0;
        for (int i = l; i < n; i += OE_LANES) {
            const int in = oe_check_one(E, b1 + 3 * i, b2 + 3 * i, &part);
            if (flags) flags[i] = (uint8_t)in;
            count += in;
        }
        total += part;
    }
    *score = total;
    return count;
}

void oe_essential_solve_ransac(int n, const double* b1, const double* b2, int max_num_iter, int recompute, uint64_t seed, double* E,
                               int* valid, int* num_inliers, int* best_iter, double* best_score, uint8_t* inlier_out, int* hyp_idx,
                               double* hyp_E, double* hyp_score, int* hyp_count) {
    for (int k = 0; k < 9; ++k) E[k] = 0.0;
    *valid = 0; *num_inliers = 0; *best_iter = -1; *best_score = 0.0;
    for (int i = 0; i < n; ++i) inlier_out[i] = 0;
    if (hyp_idx) for (int k = 0; k < OE_MIN_SET * max_num_iter; ++k) hyp_idx[k] = -1;
    if (hyp_E) for (int k = 0; k < 9 * max_num_iter; ++k) hyp_E[k] = 0.0;
    if (hyp_score) for (int k = 0; k < max_num_iter; ++k) hyp_score[k] = 0.0;
    if (hyp_count) for (int k = 0; k < max_num_iter; ++k) hyp_count[k] = 0;
    if (n < OE_MIN_SET) return;
    uint8_t* flags = (uint8_t*)malloc((size_t)n);
    double best = 0.0;
    int best_k = -1, best_cnt = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        int idx[OE_MIN_SET];
        op_ransac_sample(seed, k, n, OE_MIN_SET, idx);
        double Ek[9], sc;
        oe_compute_E(OE_MIN_SET, b1, b2, idx, Ek);
        const int cnt = oe_check_inliers(Ek, n, b1, b2, flags, &sc);
        if (hyp_idx) memcpy(hyp_idx + OE_MIN_SET * k, idx, sizeof(idx));
        if (hyp_E) memcpy(hyp_E + 9 * k, Ek, sizeof(Ek));
        if (hyp_score) hyp_score[k] = sc;
        if (hyp_count) hyp_count[k] = cnt;
        if (best < sc) {
            best = sc; best_k = k; best_cnt = cnt;
            memcpy(E, Ek, sizeof(Ek));
            memcpy(inlier_out, flags, (size_t)n);
        }
    }
    free(flags);
    *best_iter = best_k;
    *best_score = best;
    *num_inliers = best_cnt;
    *valid = (best > 0.0 && best_cnt >= OE_MIN_SET) ? 1 : 0;
    if (!*valid || !recompute) return;
    int* inl = (int*)malloc(sizeof(int) * (size_t)n);
    int m = 0;
    for (int i = 0; i < n; ++i)
        if (inlier_out[i]) inl[m++] = i;
    oe_compute_E(m, b1, b2, inl, E);
    free(inl);
    *num_inliers = oe_check_inliers(E, n, b1, b2, inlier_out, best_score);
}
