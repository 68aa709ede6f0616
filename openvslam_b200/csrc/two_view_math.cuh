// two_view_math.cuh -- arithmetic of the two RANSAC solvers of perspective map initialisation (initialize::perspective):
// solve::homography_solver (H_21, p2 ~ H_21 p1) and solve::fundamental_solver (F_21, p2^T F_21 p1 = 0) on keypoint matches.
// __host__ __device__ so tests/twoviewsolvercheck can compare the same code with the oracle (oracle/two_view_solver_oracle.c)
// on the CPU.  Only + - * / sqrt (and fabs) are used, so with contraction off the host and the device give the same bits.
//
// A problem is the undistorted keypoints of both views (x, y as floats, 2 per keypoint) and matches (idx_1, idx_2) into them.
//  - Normalisation (solve::common's normalize, once per view over ALL its keypoints): in float, mean = (running sum in index
//    order) / (float)n, dev = (running sum of |x - mean|) / (float)n, inv = (float)(1.0 / (double)dev), normalised point =
//    (x - mean) * inv; T = [[inv_x, 0, (double)(-mean_x * inv_x)], [0, inv_y, (double)(-mean_y * inv_y)], [0, 0, 1]] (each product
//    formed in float, then widened).  A zero deviation is not special-cased (inf / NaN: no inliers, invalid).
//  - The minimal solves take the normalised points as doubles.  H (DLT): per match the rows [0, 0, 0, -x1, -y1, -1, y2 x1, y2 y1, y2]
//    and [x1, y1, 1, 0, 0, 0, -x2 x1, -x2 y1, -x2]; F (eight-point): the row [x2 x1, x2 y1, x2, y2 x1, y2 y1, y2, x1, y1, 1].  One
//    match is one summation item of the 45 upper entries of A^T A (for H: v = r0_a r0_b + r1_a r1_b, row 2i first).  Items are summed
//    by pnp_sum (pnp_math.cuh): the running sum in index order up to 256 items, else 256 strided partials summed in order -- the
//    same bits from one thread (PnpSeqSum) and from one CTA (PnpBlockSum).  The model is the eigenvector of the smallest eigenvalue
//    of A^T A (jacobi_sym<9>, lowest index on ties), read row-major.
//  - F rank 2 without a 3 x 3 SVD: jacobi_sym<3> on F0^T F0, v3 = the eigenvector of its smallest eigenvalue (lowest index on
//    ties), F = F0 - (F0 v3) v3^T = U diag(s1, s2, 0) V^T (s1, s2 kept).
//  - Denormalisation, 3 x 3 products by mat3_mat3 left to right: H_21 = T2inv H T1 with the closed form
//    T2inv = [[1.0 / inv_x, 0, mean_x], [0, 1.0 / inv_y, mean_y], [0, 0, 1]] (in double from the widened floats);
//    F_21 = T2^T F T1.  Then the entry of largest magnitude (first on ties) is made positive.
//  - check_inliers per match, p = (x, y, 1) from the undistorted keypoints (doubles), in double (the reference uses float):
//    H: q = H_21 p1 / (H_21 p1)_z, chi = ((d_x^2 + d_y^2) + d_z^2) inv_sigma_sq with d = p2 - q; then the same with H_12 = H_21^-1
//       on p2 against p1; each direction is an outlier when 5.991f < chi, else adds 5.991f - chi to the score;
//    F: l2 = F_21 p1, chi = (l2 . p2)^2 / (l2_x^2 + l2_y^2) inv_sigma_sq; then l1 = F_21^T p2 against p1; an outlier when
//       3.841f < chi, else adds 5.991f - chi.
//    The first direction's term stays in the score when the second fails.  A NaN chi passes and makes the score NaN, so that
//    hypothesis never wins.  inv_sigma_sq = (float)(1.0 / (double)(sigma * sigma)) (sigma * sigma in float).
//  - A hypothesis's score over the matches: 32 partials p_l over the matches l, l + 32, .. then ((0 + p_0) + p_1) + .. + p_31 --
//    the same bits from a host loop (two_view_score_seq) and from one warp.
#pragma once
#include "pnp_math.cuh"

namespace ovs {

constexpr int kTwoViewH = 0;                         // homography_solver
constexpr int kTwoViewF = 1;                         // fundamental_solver
constexpr int kTwoViewMinSet = 8;
constexpr int kTwoViewScoreLanes = 32;
constexpr double kTwoViewScoreThr = (double)5.991f;  // the score's offset, and H's chi^2 threshold
constexpr double kTwoViewChiSqThrF = (double)3.841f; // F's chi^2 threshold

// solve::common's normalize for one view: mean and inverse mean L1 deviation per axis.
struct TwoViewNorm {
    float mean_x, mean_y, inv_x, inv_y;
};

OVS_BA_HD float two_view_inv_sigma_sq(float sigma) { return (float)(1.0 / (double)(sigma * sigma)); }

// n keypoints xy (2 floats each) -> their normalised points norm (2 floats each) and the view's TwoViewNorm.
OVS_BA_HD TwoViewNorm two_view_normalize(const float* xy, int n, float* norm) {
    float mx = 0.f, my = 0.f;
    for (int i = 0; i < n; ++i) { mx += xy[2 * i]; my += xy[2 * i + 1]; }
    const float fn = (float)n;
    mx = mx / fn; my = my / fn;
    float dx = 0.f, dy = 0.f;
    for (int i = 0; i < n; ++i) { dx += fabsf(xy[2 * i] - mx); dy += fabsf(xy[2 * i + 1] - my); }
    dx = dx / fn; dy = dy / fn;
    const float ix = (float)(1.0 / (double)dx), iy = (float)(1.0 / (double)dy);
    for (int i = 0; i < n; ++i) { norm[2 * i] = (xy[2 * i] - mx) * ix; norm[2 * i + 1] = (xy[2 * i + 1] - my) * iy; }
    return TwoViewNorm{mx, my, ix, iy};
}

// T (row-major) of a view
OVS_BA_HD void two_view_T(const TwoViewNorm& N, double* T) {
    T[0] = N.inv_x; T[1] = 0.0; T[2] = (double)(-N.mean_x * N.inv_x);
    T[3] = 0.0; T[4] = N.inv_y; T[5] = (double)(-N.mean_y * N.inv_y);
    T[6] = 0.0; T[7] = 0.0; T[8] = 1.0;
}

// The matches of one problem: match m is (keypoint pairs[2 m] of view 1, keypoint pairs[2 m + 1] of view 2).
struct TwoViewPairs {
    const float* kp_1; const float* kp_2;            // undistorted x, y per keypoint
    const float* np_1; const float* np_2;            // normalised x, y per keypoint
    const int* pairs;
    OVS_PNP_HDM const float* k1(int m) const { return kp_1 + 2 * (size_t)pairs[2 * m]; }
    OVS_PNP_HDM const float* k2(int m) const { return kp_2 + 2 * (size_t)pairs[2 * m + 1]; }
    OVS_PNP_HDM const float* n1(int m) const { return np_1 + 2 * (size_t)pairs[2 * m]; }
    OVS_PNP_HDM const float* n2(int m) const { return np_2 + 2 * (size_t)pairs[2 * m + 1]; }
};

// one match's 45 upper entries of A^T A
template <int Model>
OVS_BA_HD void two_view_item(const float* q1, const float* q2, double* v) {
    const double x1 = q1[0], y1 = q1[1], x2 = q2[0], y2 = q2[1];
    int q = 0;
    if (Model == kTwoViewH) {
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

// The model (H_21 or F_21, row-major) on the n matches idx[0 .. n) (idx null: 0 .. n) of P, sums by the policy S.
template <int Model, class Sum>
OVS_BA_HD void two_view_solve(const TwoViewPairs& P, const int* idx, const Sum& S, const TwoViewNorm& N1, const TwoViewNorm& N2,
                              double* out) {
    double up[45];
    S.template run<45>([&](int i, double* v) {
        const int m = idx ? idx[i] : i;
        two_view_item<Model>(P.n1(m), P.n2(m), v);
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
    double X[9];
    for (int k = 0; k < 9; ++k) X[k] = V[9 * k + m];
    double T1[9], L[9];
    two_view_T(N1, T1);
    if (Model == kTwoViewH) {
        L[0] = 1.0 / (double)N2.inv_x; L[1] = 0.0; L[2] = N2.mean_x;
        L[3] = 0.0; L[4] = 1.0 / (double)N2.inv_y; L[5] = N2.mean_y;
        L[6] = 0.0; L[7] = 0.0; L[8] = 1.0;
    } else {
        double G[9], W[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) G[3 * i + j] = X[i] * X[j] + X[3 + i] * X[3 + j] + X[6 + i] * X[6 + j];
        jacobi_sym<3>(G, W);
        int s = 0;
        for (int k = 1; k < 3; ++k)
            if (G[4 * k] < G[4 * s]) s = k;
        double v3[3], u[3];
        for (int r = 0; r < 3; ++r) v3[r] = W[3 * r + s];
        mat3_vec(X, v3, u);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) X[3 * r + c] = X[3 * r + c] - u[r] * v3[c];
        double T2[9];
        two_view_T(N2, T2);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) L[3 * r + c] = T2[3 * c + r];
    }
    double Y[9];
    mat3_mat3(L, X, Y);
    mat3_mat3(Y, T1, out);
    int a = 0;
    for (int k = 1; k < 9; ++k)
        if (fabs(out[k]) > fabs(out[a])) a = k;
    if (out[a] < 0.0)
        for (int k = 0; k < 9; ++k) out[k] = -out[k];
}

// H_12 = H_21^-1 as the adjugate over the determinant: with H = [[a, b, c], [d, e, f], [g, h, i]],
// c0 = e i - f h, c1 = f g - d i, c2 = d h - e g, det = (a c0 + b c1) + c c2, and
// H_12 = [[c0, c h - b i, b f - c e], [c1, a i - c g, c d - a f], [c2, b g - a h, a e - b d]] / det, entry by entry.
OVS_BA_HD void two_view_inverse(const double* H, double* o) {
    const double a = H[0], b = H[1], c = H[2], d = H[3], e = H[4], f = H[5], g = H[6], h = H[7], i = H[8];
    const double c0 = e * i - f * h, c1 = f * g - d * i, c2 = d * h - e * g;
    const double det = a * c0 + b * c1 + c * c2;
    o[0] = c0 / det; o[1] = (c * h - b * i) / det; o[2] = (b * f - c * e) / det;
    o[3] = c1 / det; o[4] = (a * i - c * g) / det; o[5] = (c * d - a * f) / det;
    o[6] = c2 / det; o[7] = (b * g - a * h) / det; o[8] = (a * e - b * d) / det;
}

// check_inliers of one match for a model, as the header comment states.  TwoViewCheck<Model>{model} holds what the test needs.
template <int Model> struct TwoViewCheck;

template <> struct TwoViewCheck<kTwoViewH> {
    double h21[9], h12[9];
    OVS_PNP_HDM explicit TwoViewCheck(const double* H) {
        for (int k = 0; k < 9; ++k) h21[k] = H[k];
        two_view_inverse(H, h12);
    }
    OVS_PNP_HDM static double transfer_chi(const double* G, const float* src, const float* dst, double inv_sigma_sq) {
        const double p[3] = {(double)src[0], (double)src[1], 1.0};
        double q[3];
        mat3_vec(G, p, q);
        const double w = q[2];
        q[0] = q[0] / w; q[1] = q[1] / w; q[2] = q[2] / w;
        const double dx = (double)dst[0] - q[0], dy = (double)dst[1] - q[1], dz = 1.0 - q[2];
        return (dx * dx + dy * dy + dz * dz) * inv_sigma_sq;
    }
    OVS_PNP_HDM bool operator()(const float* k1, const float* k2, double inv_sigma_sq, double& score) const {
        const double chi1 = transfer_chi(h21, k1, k2, inv_sigma_sq);
        if (kTwoViewScoreThr < chi1) return false;
        score += kTwoViewScoreThr - chi1;
        const double chi2 = transfer_chi(h12, k2, k1, inv_sigma_sq);
        if (kTwoViewScoreThr < chi2) return false;
        score += kTwoViewScoreThr - chi2;
        return true;
    }
};

template <> struct TwoViewCheck<kTwoViewF> {
    double f[9];
    OVS_PNP_HDM explicit TwoViewCheck(const double* F) {
        for (int k = 0; k < 9; ++k) f[k] = F[k];
    }
    OVS_PNP_HDM static double line_chi(const double* l, const float* k, double inv_sigma_sq) {
        const double d = l[0] * (double)k[0] + l[1] * (double)k[1] + l[2] * 1.0;
        return d * d / (l[0] * l[0] + l[1] * l[1]) * inv_sigma_sq;
    }
    OVS_PNP_HDM bool operator()(const float* k1, const float* k2, double inv_sigma_sq, double& score) const {
        const double p1[3] = {(double)k1[0], (double)k1[1], 1.0}, p2[3] = {(double)k2[0], (double)k2[1], 1.0};
        double l2[3], l1[3];
        mat3_vec(f, p1, l2);
        const double chi1 = line_chi(l2, k2, inv_sigma_sq);
        if (kTwoViewChiSqThrF < chi1) return false;
        score += kTwoViewScoreThr - chi1;
        for (int c = 0; c < 3; ++c) l1[c] = f[c] * p2[0] + f[3 + c] * p2[1] + f[6 + c] * p2[2];
        const double chi2 = line_chi(l1, k1, inv_sigma_sq);
        if (kTwoViewChiSqThrF < chi2) return false;
        score += kTwoViewScoreThr - chi2;
        return true;
    }
};

// check_inliers over n matches in the warp's order (header comment), from one thread: the inlier count, the flags (may be null)
// and the score.
template <int Model>
OVS_BA_HD int two_view_score_seq(const double* M, const TwoViewPairs& P, int n, double inv_sigma_sq, unsigned char* flags, double* score) {
    const TwoViewCheck<Model> chk(M);
    int count = 0;
    double total = 0.0;
    for (int l = 0; l < kTwoViewScoreLanes; ++l) {
        double part = 0.0;
        for (int i = l; i < n; i += kTwoViewScoreLanes) {
            const bool in = chk(P.k1(i), P.k2(i), inv_sigma_sq, part);
            if (flags) flags[i] = in ? 1 : 0;
            count += in ? 1 : 0;
        }
        total += part;
    }
    *score = total;
    return count;
}

}  // namespace ovs
