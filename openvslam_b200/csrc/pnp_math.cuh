// pnp_math.cuh -- FP64 arithmetic of the PnP RANSAC solver (solve::pnp_solver, relocalisation): EPnP (Lepetit, Moreno-Noguer
// and Fua) in the bearing form, the per-correspondence angular inlier test and its bound.
// __host__ __device__ so tests/pnpsolvercheck can compare the same code with the oracle (oracle/pnp_solver_oracle.c) on the CPU.
// Only + - * / sqrt are used (the bound's cos included), so with contraction off the host and the device give the same bits.
//
// Pose = {R row-major (9), t (3)} of cam_pose_cw: p_c = R p_w + t.  A correspondence is a unit bearing b of the frame keypoint
// and the landmark's world position p_w.
//
// Sums over the points of an EPnP solve (the centroid, the covariance, M^T M, the camera-frame centroid, the orientation matrix
// and the error) all follow ONE fixed order, pnp_sum: 256 partial sums s_t = ((0 + f(t)) + f(t + 256)) + ..., then
// total = ((0 + s_0) + s_1) + ... + s_255.  Adding +0.0 changes no value that arises here (a running sum from +0.0 is never
// -0.0), so for n <= 256 this is the plain running sum in index order.  The device's CTA-wide reduction (one partial per
// thread, then one thread per component over the 256 partials) gives the same bits.
#pragma once
#include "sim3_math.cuh"

// member functions: OVS_BA_HD is `static inline` on the host, which a member cannot be
#if defined(__CUDACC__)
#define OVS_PNP_HDM __host__ __device__ __forceinline__
#else
#define OVS_PNP_HDM inline
#endif

namespace ovs {

constexpr int kPnpMinSet = 6;                        // the minimal set: EPnP on 4 points is not exact in general
constexpr int kPnpSumSlots = 256;

// pnp_sum for K components at once: f(i, v) writes point i's K values.  Host and single-thread device use.
template <int K, class F>
OVS_BA_HD void pnp_sum_seq(int n, F f, double* out) {
    double v[K], s[K];
    for (int c = 0; c < K; ++c) out[c] = 0.0;
    if (n <= kPnpSumSlots) {
        for (int i = 0; i < n; ++i) {
            f(i, v);
            for (int c = 0; c < K; ++c) out[c] += v[c];
        }
        return;
    }
    for (int t = 0; t < kPnpSumSlots; ++t) {
        for (int c = 0; c < K; ++c) s[c] = 0.0;
        for (int i = t; i < n; i += kPnpSumSlots) {
            f(i, v);
            for (int c = 0; c < K; ++c) s[c] += v[c];
        }
        for (int c = 0; c < K; ++c) out[c] += s[c];
    }
}

struct PnpSeqSum {
    int n;
    template <int K, class F> OVS_PNP_HDM void run(F f, double* out) const { pnp_sum_seq<K>(n, f, out); }
};

// The correspondences of one EPnP solve: point i is entry idx[i] (or i when idx is null) of the arrays.
struct PnpPoints {
    const double* pw;                                // 3 per entry
    const double* bear;                              // 3 per entry, unit
    const int* idx;
    int n;
    OVS_PNP_HDM int at(int i) const { return idx ? idx[i] : i; }
};

// cos(x) for x in (0, pi / 2] with + - * / only: up to pi / 4 the Taylor series of cos to x^26; above it sin(d) with
// d = pi / 2 - x = d_hi + d_lo (pi / 2 split in two doubles, so d_hi = hi - x is exact), as d_hi + (d_lo - d_hi^3 / 6 p(d_hi^2))
// with the series of sin to d^25 in p.  Within one ulp of the correctly rounded cos over the range.
OVS_BA_HD double pnp_cos(double x) {
    const double kPio2Hi = 1.5707963267948966, kPio2Lo = 6.123233995736766e-17;
    if (x <= 0.7853981633974483) {
        const double x2 = x * x;
        double p = 1.0;
        for (int k = 13; k >= 1; --k) p = 1.0 - x2 / (double)((2 * k - 1) * (2 * k)) * p;
        return p;
    }
    const double dh = kPio2Hi - x, d2 = dh * dh;
    double p = 1.0;
    for (int k = 12; k >= 2; --k) p = 1.0 - d2 / (double)((2 * k) * (2 * k + 1)) * p;
    return dh + (kPio2Lo - dh * d2 / 6.0 * p);
}

// max_cos_error of a correspondence: cos(pi / 180 * scale_factor) in double, scale_factor in (0, 90].
OVS_BA_HD double pnp_max_cos(float scale_factor) { return pnp_cos(3.14159265358979323846 / 180.0 * (double)scale_factor); }

// check_inliers for one correspondence: (R p_w + t) . b / |R p_w + t| > max_cos, strictly; a NaN pose is never an inlier.
OVS_BA_HD bool pnp_is_inlier(const double* pose, const double* pw, const double* b, double max_cos) {
    double pc[3];
    mat3_vec(pose, pw, pc);
    for (int k = 0; k < 3; ++k) pc[k] += pose[9 + k];
    const double dot = pc[0] * b[0] + pc[1] * b[1] + pc[2] * b[2];
    return dot / sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]) > max_cos;
}

// Eigenvector order of a Jacobi result: rank r takes the largest (descending) or smallest (ascending) diagonal value not yet
// taken, the lowest index on ties.  Each column is signed so that its entry of largest magnitude (first on ties) is positive.
template <int N>
OVS_BA_HD void eig_order(const double* A, bool descending, int* order) {
    bool used[N];
    for (int k = 0; k < N; ++k) used[k] = false;
    for (int r = 0; r < N; ++r) {
        int m = -1;
        for (int k = 0; k < N; ++k) {
            if (used[k]) continue;
            if (m < 0 || (descending ? A[(N + 1) * k] > A[(N + 1) * m] : A[(N + 1) * k] < A[(N + 1) * m])) m = k;
        }
        used[m] = true;
        order[r] = m;
    }
}

template <int N>
OVS_BA_HD void eig_column(const double* V, int col, double* v) {
    int m = 0;
    for (int r = 1; r < N; ++r)
        if (fabs(V[N * r + col]) > fabs(V[N * m + col])) m = r;
    const double sg = V[N * m + col] < 0.0 ? -1.0 : 1.0;
    for (int r = 0; r < N; ++r) v[r] = sg * V[N * r + col];
}

// x = argmin |A x - b| for an m x n A (row-major, m <= 6, n <= 5) by Householder QR; A and b are overwritten.  Column k:
// nrm = |A[k.., k]|, alpha = -sign(a_kk) nrm (+nrm for a_kk <= 0), v = A[k.., k] - alpha e_1, each later column and b
// minus 2 (v . a) / (v . v) v; then back substitution on R (diagonal alpha).  A rank-deficient A is not special-cased.
OVS_BA_HD void lsq_householder(double* A, double* b, int m, int n, double* x) {
    for (int k = 0; k < n; ++k) {
        double nrm2 = 0.0;
        for (int i = k; i < m; ++i) nrm2 += A[n * i + k] * A[n * i + k];
        const double nrm = sqrt(nrm2);
        const double alpha = A[n * k + k] > 0.0 ? -nrm : nrm;
        const double v0 = A[n * k + k] - alpha;
        double vtv = v0 * v0;
        for (int i = k + 1; i < m; ++i) vtv += A[n * i + k] * A[n * i + k];
        if (vtv > 0.0) {
            for (int j = k + 1; j <= n; ++j) {           // j == n: the right-hand side
                double dot = v0 * (j < n ? A[n * k + j] : b[k]);
                for (int i = k + 1; i < m; ++i) dot += A[n * i + k] * (j < n ? A[n * i + j] : b[i]);
                const double f = 2.0 * dot / vtv;
                if (j < n) {
                    A[n * k + j] -= f * v0;
                    for (int i = k + 1; i < m; ++i) A[n * i + j] -= f * A[n * i + k];
                } else {
                    b[k] -= f * v0;
                    for (int i = k + 1; i < m; ++i) b[i] -= f * A[n * i + k];
                }
            }
        }
        A[n * k + k] = alpha;
    }
    for (int k = n - 1; k >= 0; --k) {
        double s = b[k];
        for (int j = k + 1; j < n; ++j) s -= A[n * k + j] * x[j];
        x[k] = s / A[n * k + k];
    }
}

// The control-point frame of an EPnP solve: cws[4][3] and the inverse of the 3 x 3 matrix of control-point differences.
struct EpnpFrame {
    double cws[12];
    double ccinv[9];
};

// alphas of a world point: a_j (j = 1..3) = row j - 1 of ccinv times (p - c_0), a_0 = ((1 - a_1) - a_2) - a_3
OVS_BA_HD void epnp_alphas(const EpnpFrame& F, const double* p, double* a) {
    const double d[3] = {p[0] - F.cws[0], p[1] - F.cws[1], p[2] - F.cws[2]};
    for (int j = 0; j < 3; ++j) a[1 + j] = F.ccinv[3 * j] * d[0] + F.ccinv[3 * j + 1] * d[1] + F.ccinv[3 * j + 2] * d[2];
    a[0] = 1.0 - a[1] - a[2] - a[3];
}

// EPnP of the n >= 4 points P (n >= 6 for an exact minimal solve) -> pose (cam_pose_cw).  Sum: the summation policy (run<K>),
// PnpSeqSum on the host and in one device thread, a CTA-wide reduction in the recompute kernel; the result is the same.
//  1. control points: c_0 = the centroid, c_j = c_0 + sqrt(max(lambda_j, 0) / n) u_j for the eigenpairs of the covariance
//     sum (p - c_0)(p - c_0)^T by jacobi_sym<3>, largest first (eig_order / eig_column);
//  2. alphas through the adjugate inverse of [c_1 - c_0, c_2 - c_0, c_3 - c_0] (columns);
//  3. M^T M (12 x 12) from the bearing rows [a_j w, 0, -a_j u] and [0, a_j w, -a_j v]; the eigenvectors v_0..v_3 of its four
//     smallest eigenvalues by jacobi_sym<12>;
//  4. L_6x10 and rho as in OpenCV's epnp.cpp; betas by approximations 1, 2 and 3 (lsq_householder), each followed by five
//     Gauss-Newton steps (lsq_householder on the 6 x 4 system);
//  5. per approximation: ccs = sum_i beta_i v_i, pcs = sum_j a_j ccs_j; the sign of ccs is flipped when b . pcs < 0 for point 0;
//     R = horn_rotation(sum (p_w - c_0)(p_c - p_c0)^T), t = p_c0 - R c_0; error = sum (1 - cos) / n;
//  6. the approximation with the smallest error, the first among equal ones (NaN errors never replace).
template <class Sum>
OVS_BA_HD void epnp_pose(const PnpPoints& P, const Sum& S, double* pose) {
    const int n = P.n;
    const double dn = (double)n;
    EpnpFrame F;
    // 1. control points
    S.template run<3>([&](int i, double* v) {
        const double* p = P.pw + 3 * P.at(i);
        v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
    }, F.cws);
    for (int k = 0; k < 3; ++k) F.cws[k] = F.cws[k] / dn;
    double cov6[6];
    S.template run<6>([&](int i, double* v) {
        const double* p = P.pw + 3 * P.at(i);
        const double d0 = p[0] - F.cws[0], d1 = p[1] - F.cws[1], d2 = p[2] - F.cws[2];
        v[0] = d0 * d0; v[1] = d0 * d1; v[2] = d0 * d2; v[3] = d1 * d1; v[4] = d1 * d2; v[5] = d2 * d2;
    }, cov6);
    {
        double C[9] = {cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]}, V[9];
        jacobi_sym<3>(C, V);
        int order[3];
        eig_order<3>(C, true, order);
        for (int j = 0; j < 3; ++j) {
            double u[3];
            eig_column<3>(V, order[j], u);
            const double lam = C[4 * order[j]];
            const double kj = sqrt((lam > 0.0 ? lam : 0.0) / dn);
            for (int c = 0; c < 3; ++c) F.cws[3 * (j + 1) + c] = F.cws[c] + kj * u[c];
        }
    }
    // 2. the inverse of CC (CC[3 * r + j] = c_{j+1}[r] - c_0[r])
    {
        double cc[9];
        for (int r = 0; r < 3; ++r)
            for (int j = 0; j < 3; ++j) cc[3 * r + j] = F.cws[3 * (j + 1) + r] - F.cws[r];
        const double c00 = cc[4] * cc[8] - cc[5] * cc[7], c01 = cc[5] * cc[6] - cc[3] * cc[8], c02 = cc[3] * cc[7] - cc[4] * cc[6];
        const double c10 = cc[2] * cc[7] - cc[1] * cc[8], c11 = cc[0] * cc[8] - cc[2] * cc[6], c12 = cc[1] * cc[6] - cc[0] * cc[7];
        const double c20 = cc[1] * cc[5] - cc[2] * cc[4], c21 = cc[2] * cc[3] - cc[0] * cc[5], c22 = cc[0] * cc[4] - cc[1] * cc[3];
        const double det = cc[0] * c00 + cc[1] * c01 + cc[2] * c02;
        const double inv[9] = {c00, c10, c20, c01, c11, c21, c02, c12, c22};
        for (int k = 0; k < 9; ++k) F.ccinv[k] = inv[k] / det;
    }
    // 3. M^T M and its null-space basis
    double MtM[144], vs[4][12];
    {
        double up[78];
        S.template run<78>([&](int i, double* v) {
            const int e = P.at(i);
            double a[4];
            epnp_alphas(F, P.pw + 3 * e, a);
            const double* b = P.bear + 3 * e;
            double r1[12], r2[12];
            for (int j = 0; j < 4; ++j) {
                r1[3 * j] = a[j] * b[2]; r1[3 * j + 1] = 0.0;         r1[3 * j + 2] = -a[j] * b[0];
                r2[3 * j] = 0.0;         r2[3 * j + 1] = a[j] * b[2]; r2[3 * j + 2] = -a[j] * b[1];
            }
            int q = 0;
            for (int r = 0; r < 12; ++r)
                for (int c = r; c < 12; ++c) v[q++] = r1[r] * r1[c] + r2[r] * r2[c];
        }, up);
        int q = 0;
        for (int r = 0; r < 12; ++r)
            for (int c = r; c < 12; ++c) { MtM[12 * r + c] = up[q]; MtM[12 * c + r] = up[q]; ++q; }
        double V[144];
        jacobi_sym<12>(MtM, V);
        int order[12];
        eig_order<12>(MtM, false, order);
        for (int i = 0; i < 4; ++i) eig_column<12>(V, order[i], vs[i]);
    }
    // 4. L_6x10, rho and the betas
    double L[60], rho[6];
    {
        double dv[4][6][3];
        for (int i = 0; i < 4; ++i) {
            int a = 0, b = 1;
            for (int j = 0; j < 6; ++j) {
                for (int c = 0; c < 3; ++c) dv[i][j][c] = vs[i][3 * a + c] - vs[i][3 * b + c];
                if (++b > 3) { ++a; b = a + 1; }
            }
        }
        for (int j = 0; j < 6; ++j) {
            double d[4][4];
            for (int x = 0; x < 4; ++x)
                for (int y = 0; y < 4; ++y) d[x][y] = dv[x][j][0] * dv[y][j][0] + dv[x][j][1] * dv[y][j][1] + dv[x][j][2] * dv[y][j][2];
            double* row = L + 10 * j;
            row[0] = d[0][0];       row[1] = 2.0 * d[0][1]; row[2] = d[1][1];       row[3] = 2.0 * d[0][2]; row[4] = 2.0 * d[1][2];
            row[5] = d[2][2];       row[6] = 2.0 * d[0][3]; row[7] = 2.0 * d[1][3]; row[8] = 2.0 * d[2][3]; row[9] = d[3][3];
        }
        int a = 0, b = 1;
        for (int j = 0; j < 6; ++j) {
            const double* ca = F.cws + 3 * a; const double* cb = F.cws + 3 * b;
            const double e0 = ca[0] - cb[0], e1 = ca[1] - cb[1], e2 = ca[2] - cb[2];
            rho[j] = e0 * e0 + e1 * e1 + e2 * e2;
            if (++b > 3) { ++a; b = a + 1; }
        }
    }
    double best_err = 0.0;
    for (int approx = 1; approx <= 3; ++approx) {
        double betas[4];
        {
            const int kCols[3][5] = {{0, 1, 3, 6, -1}, {0, 1, 2, -1, -1}, {0, 1, 2, 3, 4}};
            const int nc = approx == 1 ? 4 : (approx == 2 ? 3 : 5);
            double A[30], rhs[6], x[5];
            for (int j = 0; j < 6; ++j) {
                for (int c = 0; c < nc; ++c) A[nc * j + c] = L[10 * j + kCols[approx - 1][c]];
                rhs[j] = rho[j];
            }
            lsq_householder(A, rhs, 6, nc, x);
            if (approx == 1) {
                if (x[0] < 0.0) {
                    betas[0] = sqrt(-x[0]);
                    betas[1] = -x[1] / betas[0]; betas[2] = -x[2] / betas[0]; betas[3] = -x[3] / betas[0];
                } else {
                    betas[0] = sqrt(x[0]);
                    betas[1] = x[1] / betas[0]; betas[2] = x[2] / betas[0]; betas[3] = x[3] / betas[0];
                }
            } else {
                if (x[0] < 0.0) {
                    betas[0] = sqrt(-x[0]);
                    betas[1] = x[2] < 0.0 ? sqrt(-x[2]) : 0.0;
                } else {
                    betas[0] = sqrt(x[0]);
                    betas[1] = x[2] > 0.0 ? sqrt(x[2]) : 0.0;
                }
                if (x[1] < 0.0) betas[0] = -betas[0];
                betas[2] = approx == 3 ? x[3] / betas[0] : 0.0;
                betas[3] = 0.0;
            }
        }
        for (int it = 0; it < 5; ++it) {                 // Gauss-Newton on rho_j = L_j . (beta products)
            double A[24], rhs[6], x[4];
            for (int j = 0; j < 6; ++j) {
                const double* l = L + 10 * j;
                const double* bt = betas;
                A[4 * j]     = 2.0 * l[0] * bt[0] + l[1] * bt[1] + l[3] * bt[2] + l[6] * bt[3];
                A[4 * j + 1] = l[1] * bt[0] + 2.0 * l[2] * bt[1] + l[4] * bt[2] + l[7] * bt[3];
                A[4 * j + 2] = l[3] * bt[0] + l[4] * bt[1] + 2.0 * l[5] * bt[2] + l[8] * bt[3];
                A[4 * j + 3] = l[6] * bt[0] + l[7] * bt[1] + l[8] * bt[2] + 2.0 * l[9] * bt[3];
                rhs[j] = rho[j] - (l[0] * bt[0] * bt[0] + l[1] * bt[0] * bt[1] + l[2] * bt[1] * bt[1] + l[3] * bt[0] * bt[2] +
                                   l[4] * bt[1] * bt[2] + l[5] * bt[2] * bt[2] + l[6] * bt[0] * bt[3] + l[7] * bt[1] * bt[3] +
                                   l[8] * bt[2] * bt[3] + l[9] * bt[3] * bt[3]);
            }
            lsq_householder(A, rhs, 6, 4, x);
            for (int k = 0; k < 4; ++k) betas[k] += x[k];
        }
        // 5. camera-frame control points, the sign, R and t, the error
        double ccs[12];
        for (int k = 0; k < 12; ++k) ccs[k] = 0.0;
        for (int i = 0; i < 4; ++i)
            for (int k = 0; k < 12; ++k) ccs[k] += betas[i] * vs[i][k];
        auto pcs_of = [&](int e, double* pc) {
            double a[4];
            epnp_alphas(F, P.pw + 3 * e, a);
            for (int c = 0; c < 3; ++c) pc[c] = a[0] * ccs[c] + a[1] * ccs[3 + c] + a[2] * ccs[6 + c] + a[3] * ccs[9 + c];
        };
        {
            const int e0 = P.at(0);
            double pc[3];
            pcs_of(e0, pc);
            const double* b = P.bear + 3 * e0;
            if (pc[0] * b[0] + pc[1] * b[1] + pc[2] * b[2] < 0.0)
                for (int k = 0; k < 12; ++k) ccs[k] = -ccs[k];
        }
        double pc0[3];
        S.template run<3>([&](int i, double* v) { pcs_of(P.at(i), v); }, pc0);
        for (int c = 0; c < 3; ++c) pc0[c] = pc0[c] / dn;
        double Mo[9];
        S.template run<9>([&](int i, double* v) {
            const int e = P.at(i);
            double pc[3];
            pcs_of(e, pc);
            const double* p = P.pw + 3 * e;
            const double dw[3] = {p[0] - F.cws[0], p[1] - F.cws[1], p[2] - F.cws[2]};
            const double dc[3] = {pc[0] - pc0[0], pc[1] - pc0[1], pc[2] - pc0[2]};
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) v[3 * r + c] = dw[r] * dc[c];
        }, Mo);
        double cand[12];
        horn_rotation(Mo, cand);
        double rc[3];
        mat3_vec(cand, F.cws, rc);
        for (int c = 0; c < 3; ++c) cand[9 + c] = pc0[c] - rc[c];
        double err;
        S.template run<1>([&](int i, double* v) {
            const int e = P.at(i);
            const double* p = P.pw + 3 * e;
            const double* b = P.bear + 3 * e;
            double q[3];
            mat3_vec(cand, p, q);
            for (int c = 0; c < 3; ++c) q[c] += cand[9 + c];
            v[0] = 1.0 - (q[0] * b[0] + q[1] * b[1] + q[2] * b[2]) / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        }, &err);
        err = err / dn;
        if (approx == 1 || err < best_err) {
            best_err = err;
            for (int k = 0; k < 12; ++k) pose[k] = cand[k];
        }
    }
}

// The identity pose, returned when no hypothesis has an inlier.
OVS_BA_HD void pnp_identity(double* pose) {
    for (int k = 0; k < 12; ++k) pose[k] = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
}

}  // namespace ovs
