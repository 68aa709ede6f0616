// initializer_math.cuh -- FP64 arithmetic of monocular map initialisation (initialize::perspective, initialize::bearing_vector and
// their base's check_pose / find_most_plausible_pose; homography_solver::decompose, fundamental_solver::decompose and
// essential_solver::decompose; names as recalled, DESIGN.md section 5).
// __host__ __device__ so tests/initializercheck can compare the same code with the oracle (oracle/initializer_oracle.c) on the
// CPU.  Only + - * / sqrt and fabs are used, except the equirectangular reprojection's atan2 / asin (ransac_reproject), so with
// contraction off the host and the device give the same bits.
//
// A hypothesis is {R row-major (9), t (3)} of the current camera relative to the reference one: p_cur = R p_ref + t.
#pragma once
#include <string.h>

#include "triangulation_math.cuh"

namespace ovs {

// The recalled constants, each named once.
constexpr double kInitRankRatio = 1.00001;           // decompose (H): refused when d1 / d2 or d2 / d3 is below it
constexpr double kInitSmallParallaxCos = 0.99998;    // check_pose: cos_parallax above it is a small parallax
constexpr int kInitParallaxRank = 50;                // check_pose: the min(50, n - 1)-th smallest cos_parallax
constexpr double kInitAmbiguity = 0.8;               // find_most_plausible_pose: a count above 0.8 x the best is similar
constexpr double kInitRelScoreH = 0.40;              // perspective::initialize: H when S_H / (S_H + S_F) is above it
constexpr int kInitMaxHyp = 8;

// The outcome of one match under one hypothesis, in the order check_pose tests it.
enum : int {
    kInitValid = 0,          // valid, parallax not small: triangulated
    kInitValidSmall = 1,     // valid, small parallax: counted, not triangulated
    kInitNonFinite = 2,
    kInitDepthRef = 3, kInitDepthCur = 4,
    kInitReprojRef = 5, kInitReprojCur = 6,
};

// The decision of find_most_plausible_pose (kInitChoice* match OVS_INIT_* of ovs_b200.h).
enum : int { kInitChoiceOk = 0, kInitChoiceTooFew = 3, kInitChoiceAmbiguous = 4, kInitChoiceSmallParallax = 5 };

OVS_BA_HD double det3(const double* M) {
    return (M[0] * (M[4] * M[8] - M[5] * M[7]) + M[1] * (M[5] * M[6] - M[3] * M[8])) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// C = A B^T
OVS_BA_HD void mat3_mat3t(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}

// K^-1 of a perspective camera: [[1 / fx, 0, -cx / fx], [0, 1 / fy, -cy / fy], [0, 0, 1]]
OVS_BA_HD void init_k_inv(const CameraD& c, double* Ki) {
    Ki[0] = 1.0 / c.fx; Ki[1] = 0.0; Ki[2] = -c.cx / c.fx;
    Ki[3] = 0.0; Ki[4] = 1.0 / c.fy; Ki[5] = -c.cy / c.fy;
    Ki[6] = 0.0; Ki[7] = 0.0; Ki[8] = 1.0;
}

OVS_BA_HD void init_k(const CameraD& c, double* K) {
    K[0] = c.fx; K[1] = 0.0; K[2] = c.cx;
    K[3] = 0.0; K[4] = c.fy; K[5] = c.cy;
    K[6] = 0.0; K[7] = 0.0; K[8] = 1.0;
}

// A = U diag(d) V^T without a 3 x 3 SVD: V and d_i^2 from jacobi_sym<3> on A^T A (summed over rows 0, 1, 2 in order), ordered
// descending (eig_order, lowest index on ties), each column of V signed by eig_column (its largest-magnitude entry positive);
// d_i = sqrt(max(d_i^2, 0)); u_i = A v_i / d_i for i = 1, 2; u_3 = A v_3 / d_3, or u_1 x u_2 with third_by_cross (E, whose
// d_3 is about 0).  U and V row-major.  Forming A^T A squares A's condition number (DESIGN.md section 5).
OVS_BA_HD void svd3(const double* A, bool third_by_cross, double* U, double* d, double* V) {
    double G[9], W[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) G[3 * i + j] = (A[i] * A[j] + A[3 + i] * A[3 + j]) + A[6 + i] * A[6 + j];
    jacobi_sym<3>(G, W);
    int order[3];
    eig_order<3>(G, true, order);
    for (int k = 0; k < 3; ++k) {
        double v[3];
        eig_column<3>(W, order[k], v);
        for (int r = 0; r < 3; ++r) V[3 * r + k] = v[r];
        const double l = G[4 * order[k]];
        d[k] = l > 0.0 ? sqrt(l) : 0.0;
    }
    for (int k = 0; k < 3; ++k) {
        if (k == 2 && third_by_cross) {
            U[2] = U[3] * U[7] - U[6] * U[4];
            U[5] = U[6] * U[1] - U[0] * U[7];
            U[8] = U[0] * U[4] - U[3] * U[1];
            break;
        }
        const double v[3] = {V[k], V[3 + k], V[6 + k]};
        double a[3];
        mat3_vec(A, v, a);
        for (int r = 0; r < 3; ++r) U[3 * r + k] = a[r] / d[k];
    }
}

// t / |t|, component by component
OVS_BA_HD void init_normalize3(double* t) {
    const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    for (int r = 0; r < 3; ++r) t[r] = t[r] / n;
}

// homography_solver::decompose(H_21, K_1, K_2) by Faugeras' method on A = (K_2^-1 H_21) K_1 = U diag(d1, d2, d3) V^T (svd3),
// s = det U det V.  Refused (false) when d1 / d2 < 1.00001 or d2 / d3 < 1.00001 (or either ratio is NaN).  Otherwise hypothesis
// i (0..3, d' = d2) and 4 + i (d' = -d2): R = s ((U R') V^T), t = U t' normalised, n = V (x1, 0, x3) with n_z >= 0, where
//   x1 = {a1, a1, -a1, -a1}, x3 = {a3, -a3, a3, -a3}, a1 = sqrt((d1^2 - d2^2) / (d1^2 - d3^2)), a3 = sqrt((d2^2 - d3^2) / (d1^2 - d3^2));
//   d' = d2: R' = [[c, 0, -s_i], [0, 1, 0], [s_i, 0, c]], s_i = {st, -st, -st, st}, t' = (d1 - d3) (x1, 0, -x3),
//            st = sqrt((d1^2 - d2^2)(d2^2 - d3^2)) / ((d1 + d3) d2), c = (d2^2 + d1 d3) / ((d1 + d3) d2);
//   d' = -d2: R' = [[c, 0, s_i], [0, -1, 0], [s_i, 0, -c]], s_i = {sp, -sp, -sp, sp}, t' = (d1 + d3) (x1, 0, x3),
//            sp = sqrt((d1^2 - d2^2)(d2^2 - d3^2)) / ((d1 - d3) d2), c = (d1 d3 - d2^2) / ((d1 - d3) d2).
// R[i] (9 each), t[i] (3 each), n[i] (3 each; may be null).
OVS_BA_HD bool decompose_homography(const double* H, const CameraD& cam_1, const CameraD& cam_2, double* R, double* t, double* n) {
    double K2i[9], K1[9], T[9], A[9];
    init_k_inv(cam_2, K2i);
    init_k(cam_1, K1);
    mat3_mat3(K2i, H, T);
    mat3_mat3(T, K1, A);
    double U[9], d[3], V[9];
    svd3(A, false, U, d, V);
    const double d1 = d[0], d2 = d[1], d3 = d[2];
    if (!(d1 / d2 >= kInitRankRatio && d2 / d3 >= kInitRankRatio)) return false;
    const double s = det3(U) * det3(V);
    const double d1s = d1 * d1, d2s = d2 * d2, d3s = d3 * d3;
    const double a1 = sqrt((d1s - d2s) / (d1s - d3s)), a3 = sqrt((d2s - d3s) / (d1s - d3s));
    const double x1[4] = {a1, a1, -a1, -a1}, x3[4] = {a3, -a3, a3, -a3};
    const double root = sqrt((d1s - d2s) * (d2s - d3s));
    for (int neg = 0; neg < 2; ++neg) {
        const double den = neg ? (d1 - d3) * d2 : (d1 + d3) * d2;
        const double sn = root / den, c = neg ? (d1 * d3 - d2s) / den : (d2s + d1 * d3) / den;
        const double sg[4] = {sn, -sn, -sn, sn};
        for (int i = 0; i < 4; ++i) {
            const int h = 4 * neg + i;
            double Rp[9] = {c, 0.0, neg ? sg[i] : -sg[i], 0.0, neg ? -1.0 : 1.0, 0.0, sg[i], 0.0, neg ? -c : c};
            double UR[9], Rh[9];
            mat3_mat3(U, Rp, UR);
            mat3_mat3t(UR, V, Rh);
            for (int k = 0; k < 9; ++k) R[9 * h + k] = s * Rh[k];
            const double f = neg ? d1 + d3 : d1 - d3;
            const double tp[3] = {x1[i] * f, 0.0, (neg ? x3[i] : -x3[i]) * f};
            mat3_vec(U, tp, t + 3 * h);
            init_normalize3(t + 3 * h);
            if (n) {
                const double np[3] = {x1[i], 0.0, x3[i]};
                mat3_vec(V, np, n + 3 * h);
                if (n[3 * h + 2] < 0.0)
                    for (int r = 0; r < 3; ++r) n[3 * h + r] = -n[3 * h + r];
            }
        }
    }
    return true;
}

// essential_solver::decompose(E_21): E = U diag(d) V^T (svd3 with u_3 = u_1 x u_2), t = u_3 normalised,
// W = [[0, -1, 0], [1, 0, 0], [0, 0, 1]], R1 = (U W) V^T, R2 = (U W^T) V^T, each negated when its determinant is negative.
// Hypotheses {(R1, t), (R1, -t), (R2, t), (R2, -t)}.
OVS_BA_HD void decompose_essential(const double* E, double* R, double* t) {
    double U[9], d[3], V[9];
    svd3(E, true, U, d, V);
    double u3[3] = {U[2], U[5], U[8]};
    init_normalize3(u3);
    for (int w = 0; w < 2; ++w) {
        const double W[9] = {0.0, w ? 1.0 : -1.0, 0.0, w ? -1.0 : 1.0, 0.0, 0.0, 0.0, 0.0, 1.0};
        double UW[9], Rw[9];
        mat3_mat3(U, W, UW);
        mat3_mat3t(UW, V, Rw);
        if (det3(Rw) < 0.0)
            for (int k = 0; k < 9; ++k) Rw[k] = -Rw[k];
        for (int s = 0; s < 2; ++s) {
            const int h = 2 * w + s;
            for (int k = 0; k < 9; ++k) R[9 * h + k] = Rw[k];
            for (int r = 0; r < 3; ++r) t[3 * h + r] = s ? -u3[r] : u3[r];
        }
    }
}

// fundamental_solver::decompose(F_21, K_1, K_2): E_21 = (K_2^T F_21) K_1, then decompose_essential.
OVS_BA_HD void decompose_fundamental(const double* F, const CameraD& cam_1, const CameraD& cam_2, double* R, double* t) {
    double K2[9], K2t[9], K1[9], T[9], E[9];
    init_k(cam_2, K2);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) K2t[3 * r + c] = K2[3 * c + r];
    init_k(cam_1, K1);
    mat3_mat3(K2t, F, T);
    mat3_mat3(T, K1, E);
    decompose_essential(E, R, t);
}

// check_pose for one inlier match under one hypothesis {R, t}: p = tri_two_cameras(b_ref, b_cur, [I | 0], [R | t]) (a match with
// a non-finite p is skipped); cos_parallax = p . (p - c) / (|p| |p - c|) in double, c = -R^T t, kept as a float (*cos_par);
// small = 0.99998 < cos_parallax; with depth_is_positive and a parallax that is not small, p_z <= 0 rejects (reference camera),
// then (R p + t)_z <= 0 (current camera); then each view's ransac_reproject (invalid: rejected) and its squared pixel error
// against reproj_err_thr_sq (rejected above it).  Returns kInitValid, kInitValidSmall or the first failed test; p is written
// whenever it was formed.  A NaN cos_parallax (p at a camera centre) counts as non-finite.
OVS_BA_HD int init_check_match(const double* Rt, const CameraD& cam_ref, const CameraD& cam_cur, const double* b_ref, const double* b_cur,
                               const float* kp_ref, const float* kp_cur, double reproj_err_thr_sq, bool depth_is_positive, double* p,
                               float* cos_par) {
    const double P1[12] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};
    tri_two_cameras(b_ref, b_cur, P1, Rt, p);
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) return kInitNonFinite;
    double c[3];
    tri_cam_center(Rt, c);
    const double q[3] = {p[0] - c[0], p[1] - c[1], p[2] - c[2]};
    const double np = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]), nq = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    const float cp = (float)((p[0] * q[0] + p[1] * q[1] + p[2] * q[2]) / (np * nq));
    *cos_par = cp;
    if (cp != cp) return kInitNonFinite;             // p at a camera centre
    const bool small = kInitSmallParallaxCos < (double)cp;
    if (depth_is_positive && !small) {
        if (p[2] <= 0.0) return kInitDepthRef;
        double pc[3];
        mat3_vec(Rt, p, pc);
        if (pc[2] + Rt[11] <= 0.0) return kInitDepthCur;
    }
    const double zero[3] = {0.0, 0.0, 0.0};
    double uv[2];
    if (!ransac_reproject(cam_ref, P1, zero, p, uv)) return kInitReprojRef;
    double ex = uv[0] - (double)kp_ref[0], ey = uv[1] - (double)kp_ref[1];
    if (reproj_err_thr_sq < ex * ex + ey * ey) return kInitReprojRef;
    if (!ransac_reproject(cam_cur, Rt, Rt + 9, p, uv)) return kInitReprojCur;
    ex = uv[0] - (double)kp_cur[0]; ey = uv[1] - (double)kp_cur[1];
    if (reproj_err_thr_sq < ex * ex + ey * ey) return kInitReprojCur;
    return small ? kInitValidSmall : kInitValid;
}

// The order-preserving key of a float: a < b (neither NaN) exactly when key(a) < key(b) as unsigned.  0xffffffff marks a match
// that is not valid (no float maps to it but the all-ones NaN, which cos_parallax never is).
constexpr unsigned kInitNoKey = 0xffffffffu;
OVS_BA_HD unsigned init_key(float f) {
    unsigned u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
OVS_BA_HD float init_key_value(unsigned k) {
    const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// The rank check_pose takes among n valid points: min(50, n - 1).
OVS_BA_HD int init_parallax_rank(int n) { return n - 1 < kInitParallaxRank ? n - 1 : kInitParallaxRank; }

// find_most_plausible_pose over nh hypotheses: best = the most valid points (first on ties); too few when below
// min_num_triangulated; ambiguous when more than one count exceeds 0.8 x the best; small parallax when the best's selected
// cos_parallax is greater than cos_thr = cos(parallax_deg_thr pi / 180).  *best is written in every case.
OVS_BA_HD int init_choose(int nh, const int* count, const float* cos_par, int min_num_triangulated, double cos_thr, int* best) {
    int b = 0;
    for (int h = 1; h < nh; ++h)
        if (count[h] > count[b]) b = h;
    *best = b;
    if (count[b] < min_num_triangulated) return kInitChoiceTooFew;
    int similar = 0;
    for (int h = 0; h < nh; ++h)
        if (kInitAmbiguity * (double)count[b] < (double)count[h]) ++similar;
    if (1 < similar) return kInitChoiceAmbiguous;
    if (cos_thr < (double)cos_par[b]) return kInitChoiceSmallParallax;
    return kInitChoiceOk;
}

}  // namespace ovs
