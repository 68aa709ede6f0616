// essential_math.cuh -- FP64 arithmetic of the essential-matrix RANSAC solver (solve::essential_solver, the tracker's robust
// match and equirectangular map initialisation): the eight-point E_21 on bearing pairs, its rank-2 projection, and the
// per-match angular inlier test and score.
// __host__ __device__ so tests/essentialsolvercheck can compare the same code with the oracle (oracle/essential_solver_oracle.c)
// on the CPU.  Only + - * / sqrt are used, so with contraction off the host and the device give the same bits.
//
// A match is a pair of unit bearings (b1 of keypoint idx_1 in camera 1, b2 of keypoint idx_2 in camera 2); E_21 (row-major)
// satisfies b2^T E_21 b1 = 0.  Every sum follows a fixed order:
//  - A^T A over the pairs of one solve: pnp_sum (pnp_math.cuh), i.e. the running sum in index order up to 256 pairs, else 256
//    strided partials summed in order -- the same bits from one thread (PnpSeqSum) and from one CTA (PnpBlockSum);
//  - a hypothesis's score over the matches: 32 partials p_l over the matches l, l + 32, .. (each match adds r2, then r1), then
//    ((0 + p_0) + p_1) + .. + p_31 -- the same bits from a host loop (essential_score_seq) and from one warp.
#pragma once
#include "pnp_math.cuh"

namespace ovs {

constexpr int kEssMinSet = 8;                        // the eight-point algorithm's minimal set
constexpr double kEssResidualCosThr = 0.01745240643; // sin(1 degree): the largest accepted |b . n| of a bearing and its epipolar plane
constexpr int kEssScoreLanes = 32;

// The matches of one solve.  Match m is (bear_1 entry j1, bear_2 entry j2) with (j1, j2) = (pairs[2 m], pairs[2 m + 1]), or
// (m, m) when pairs is null (bearings already gathered per match).
struct EssPairs {
    const double* bear_1;
    const double* bear_2;
    const int* pairs;
    OVS_PNP_HDM const double* b1(int m) const { return bear_1 + 3 * (size_t)(pairs ? pairs[2 * m] : m); }
    OVS_PNP_HDM const double* b2(int m) const { return bear_2 + 3 * (size_t)(pairs ? pairs[2 * m + 1] : m); }
};

// compute_E_21 on the n matches idx[0 .. n) (idx null: 0 .. n):
//  1. a = b2 (x) b1 (a[3 r + c] = b2[r] b1[c]) per match; the 45 upper entries of M = A^T A by the summation policy S;
//  2. e = the eigenvector of M's smallest eigenvalue (jacobi_sym<9>, lowest index on ties), read as E row-major;
//  3. rank 2 without a 3 x 3 SVD: jacobi_sym<3> on E^T E, eigenvalues descending (eig_order, lowest index on ties),
//     sigma_i = sqrt(max(lambda_i, 0)), s = (sigma_1 + sigma_2) / 2, E' = s (E v_1 v_1^T / sigma_1 + E v_2 v_2^T / sigma_2)
//     = U diag(s, s, 0) V^T, independent of the eigenvector signs; E' = 0 unless sigma_2 > 0;
//  4. the entry of largest magnitude (first on ties) is made positive.
template <class Sum>
OVS_BA_HD void essential_from_pairs(const EssPairs& P, const int* idx, const Sum& S, double* E) {
    double up[45];
    S.template run<45>([&](int i, double* v) {
        const int m = idx ? idx[i] : i;
        const double* b1 = P.b1(m);
        const double* b2 = P.b2(m);
        double a[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) a[3 * r + c] = b2[r] * b1[c];
        int q = 0;
        for (int r = 0; r < 9; ++r)
            for (int c = r; c < 9; ++c) v[q++] = a[r] * a[c];
    }, up);
    double M[81], V[81];
    {
        int q = 0;
        for (int r = 0; r < 9; ++r)
            for (int c = r; c < 9; ++c) { M[9 * r + c] = up[q]; M[9 * c + r] = up[q]; ++q; }
    }
    jacobi_sym<9>(M, V);
    int m = 0;
    for (int k = 1; k < 9; ++k)
        if (M[10 * k] < M[10 * m]) m = k;
    double E0[9];
    for (int k = 0; k < 9; ++k) E0[k] = V[9 * k + m];
    // E0^T E0, each entry summed over the rows in order
    double G[9], W[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) G[3 * i + j] = E0[i] * E0[j] + E0[3 + i] * E0[3 + j] + E0[6 + i] * E0[6 + j];
    jacobi_sym<3>(G, W);
    int order[3];
    eig_order<3>(G, true, order);
    const double l1 = G[4 * order[0]], l2 = G[4 * order[1]];
    const double s1 = sqrt(l1 > 0.0 ? l1 : 0.0), s2 = sqrt(l2 > 0.0 ? l2 : 0.0);
    if (!(s2 > 0.0)) {
        for (int k = 0; k < 9; ++k) E[k] = 0.0;
        return;
    }
    const double s = (s1 + s2) / 2.0;
    double v1[3], v2[3], u1[3], u2[3];
    for (int r = 0; r < 3; ++r) { v1[r] = W[3 * r + order[0]]; v2[r] = W[3 * r + order[1]]; }
    mat3_vec(E0, v1, u1);
    mat3_vec(E0, v2, u2);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) E[3 * r + c] = s * (u1[r] * v1[c] / s1 + u2[r] * v2[c] / s2);
    int a = 0;
    for (int k = 1; k < 9; ++k)
        if (fabs(E[k]) > fabs(E[a])) a = k;
    if (E[a] < 0.0)
        for (int k = 0; k < 9; ++k) E[k] = -E[k];
}

// check_inliers for one match: r2 = |(E b1) . b2| / |E b1| first; r2 > thr is an outlier; otherwise r2 joins the score and
// r1 = |(E^T b2) . b1| / |E^T b2| is tested the same way (r1 joins the score when it passes; r2 stays in it when r1 fails).
// The tests are !(thr < r): a zero norm (NaN) passes and makes the score NaN, so that hypothesis is never best.
OVS_BA_HD bool essential_check(const double* E, const double* b1, const double* b2, double& score) {
    double e1[3];
    mat3_vec(E, b1, e1);
    const double r2 = fabs(e1[0] * b2[0] + e1[1] * b2[1] + e1[2] * b2[2]) / sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
    if (kEssResidualCosThr < r2) return false;
    score += r2;
    double e2[3];
    for (int c = 0; c < 3; ++c) e2[c] = E[c] * b2[0] + E[3 + c] * b2[1] + E[6 + c] * b2[2];
    const double r1 = fabs(e2[0] * b1[0] + e2[1] * b1[1] + e2[2] * b1[2]) / sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    if (kEssResidualCosThr < r1) return false;
    score += r1;
    return true;
}

// check_inliers over n matches in the warp's order (header comment), from one thread: the inlier count, the flags (may be null)
// and the score.
OVS_BA_HD int essential_score_seq(const double* E, const EssPairs& P, int n, unsigned char* flags, double* score) {
    int count = 0;
    double total = 0.0;
    for (int l = 0; l < kEssScoreLanes; ++l) {
        double part = 0.0;
        for (int i = l; i < n; i += kEssScoreLanes) {
            const bool in = essential_check(E, P.b1(i), P.b2(i), part);
            if (flags) flags[i] = in ? 1 : 0;
            count += in ? 1 : 0;
        }
        total += part;
    }
    *score = total;
    return count;
}

}  // namespace ovs
