// sim3_math.cuh -- FP64 Sim3 arithmetic of the transform optimiser (optimize::transform_optimizer, loop closure):
// the exponential and left update of g2o::Sim3 / transform_vertex, and the residuals and analytic 2 x 7 Jacobians of the
// forward (12) and backward (21) reprojection edges, perspective and equirectangular.
// __host__ __device__ so tests/sim3check can compare the same code with the oracle (oracle/sim3_oracle.c) on the CPU.
//
// Representation: sim3 = {R row-major (9), t (3), s}, S p = s R p + t.  Update xi = [omega (3), upsilon (3), sigma (1)]
// (g2o's Sim3 order); the estimate moves by S <- exp(xi) S.
#pragma once
#include "ba_math.cuh"

namespace ovs {

// exp of the sim(3) generator [[sigma I + [omega]x, upsilon], [0, 0]]:
//   s = e^sigma, R = exp([omega]x) = I + ra O + rb O^2, t = W upsilon with W = int_0^1 e^(sigma u) exp(u O) du = C I + A O + B O^2.
// The small-angle / small-scale branches take the leading terms of the same series (not g2o's I + O + O^2 rotation).
OVS_BA_HD void sim3_exp(const double* u, double* S) {
    const double wx = u[0], wy = u[1], wz = u[2], sigma = u[6];
    const double theta = sqrt(wx * wx + wy * wy + wz * wz);
    const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    double O2[9];
    mat3_mat3(O, O, O2);
    const double es = exp(sigma);
    double C;
    if (fabs(sigma) < 1e-5) C = 1.0 + sigma * (0.5 + sigma * (1.0 / 6.0));
    else C = expm1(sigma) / sigma;
    double ra, rb, A, B;
    if (theta < 1e-5) {
        ra = 1.0; rb = 0.5;
        // A = int u e^(sigma u), B = 1/2 int u^2 e^(sigma u): the theta -> 0 limits
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
    mat3_vec(W, u + 3, S + 9);
    S[12] = es;
}

// transform_vertex::oplusImpl: S <- exp(xi) S; with fix_scale the update's sigma is zeroed first (s stays bit-for-bit).
OVS_BA_HD void sim3_oplus(const double* S, const double* xi, bool fix_scale, double* out) {
    double u[7];
    for (int k = 0; k < 7; ++k) u[k] = xi[k];
    if (fix_scale) u[6] = 0.0;
    double E[13], Rn[9], q[3];
    sim3_exp(u, E);
    mat3_mat3(E, S, Rn);
    mat3_vec(E, S + 9, q);
    for (int k = 0; k < 9; ++k) out[k] = Rn[k];
    for (int k = 0; k < 3; ++k) out[9 + k] = E[12] * q[k] + E[9 + k];
    out[12] = E[12] * S[12];
}

// Projection of a camera-frame point and its Jacobian P = d pi / d p (2 x 3, may be null).
OVS_BA_HD void sim3_project(const CameraD& cam, const double* p, double* uv, double* P) {
    const double x = p[0], y = p[1], z = p[2];
    if (cam.model == kCamEquirectangular) {
        const double L = sqrt(x * x + y * y + z * z);
        const double theta = atan2(x, z);
        const double phi = -asin(y / L);
        uv[0] = cam.cols * (0.5 + theta / (2 * kPi));
        uv[1] = cam.rows * (0.5 - phi / kPi);
        if (P) {
            const double xz2 = x * x + z * z;
            const double c0 = (cam.cols / (2 * kPi)) / xz2;
            const double c1 = (cam.rows / kPi) / (L * sqrt(xz2));
            P[0] = c0 * z; P[1] = 0.0; P[2] = -c0 * x;
            P[3] = -c1 * (y * x / L); P[4] = c1 * (L - y * y / L); P[5] = -c1 * (y * z / L);
        }
        return;
    }
    uv[0] = cam.fx * x / z + cam.cx;
    uv[1] = cam.fy * y / z + cam.cy;
    if (P) {
        const double z_sq = z * z;
        P[0] = cam.fx / z; P[1] = 0.0; P[2] = -cam.fx * x / z_sq;
        P[3] = 0.0; P[4] = cam.fy / z; P[5] = -cam.fy * y / z_sq;
    }
}

// J (2 x 7) = -P D for the point's derivative D (3 x 7, row-major) with respect to the update.
OVS_BA_HD void sim3_chain(const double* P, const double* D, double* J) {
    for (int r = 0; r < 2; ++r)
        for (int k = 0; k < 7; ++k) J[7 * r + k] = -(P[3 * r] * D[k] + P[3 * r + 1] * D[7 + k] + P[3 * r + 2] * D[14 + k]);
}

// Forward edge (12): e = obs_1 - pi_1(S pc2), pc2 = keyframe 2's camera-frame landmark.  J: 2 x 7 or null.
OVS_BA_HD void sim3_edge_forward(const CameraD& cam1, const double* S, const double* pc2, const double* obs, double* e, double* J) {
    double q[3], p[3], uv[2], P[6];
    mat3_vec(S, pc2, q);
    for (int k = 0; k < 3; ++k) p[k] = S[12] * q[k] + S[9 + k];
    sim3_project(cam1, p, uv, J ? P : nullptr);
    e[0] = obs[0] - uv[0];
    e[1] = obs[1] - uv[1];
    if (J) {
        // d(exp(xi) p)/d xi at 0 = [-[p]x, I, p]
        const double x = p[0], y = p[1], z = p[2];
        const double D[21] = {0, z, -y, 1, 0, 0, x,
                              -z, 0, x, 0, 1, 0, y,
                              y, -x, 0, 0, 0, 1, z};
        sim3_chain(P, D, J);
    }
}

// Backward edge (21): e = obs_2 - pi_2(S^-1 pc1), S^-1 p = R^T (p - t) / s, pc1 = keyframe 1's camera-frame landmark.
OVS_BA_HD void sim3_edge_backward(const CameraD& cam2, const double* S, const double* pc1, const double* obs, double* e, double* J) {
    const double is = 1.0 / S[12];
    const double d[3] = {pc1[0] - S[9], pc1[1] - S[10], pc1[2] - S[11]};
    double p[3], uv[2], P[6];
    for (int k = 0; k < 3; ++k) p[k] = (S[k] * d[0] + S[3 + k] * d[1] + S[6 + k] * d[2]) * is;
    sim3_project(cam2, p, uv, J ? P : nullptr);
    e[0] = obs[0] - uv[0];
    e[1] = obs[1] - uv[1];
    if (J) {
        // (exp(xi) S)^-1 pc1 = S^-1 exp(-xi) pc1: d/d xi at 0 = (R^T / s) [[pc1]x, -I, -pc1]
        const double x = pc1[0], y = pc1[1], z = pc1[2];
        const double M[21] = {0, -z, y, -1, 0, 0, -x,
                              z, 0, -x, 0, -1, 0, -y,
                              -y, x, 0, 0, 0, -1, -z};
        double D[21];
        for (int m = 0; m < 3; ++m)
            for (int k = 0; k < 7; ++k) D[7 * m + k] = (S[m] * M[k] + S[3 + m] * M[7 + k] + S[6 + m] * M[14 + k]) * is;
        sim3_chain(P, D, J);
    }
}

// Packed upper-triangle index of element (i, j) of a symmetric 7 x 7.
OVS_BA_HD int sym7(int i, int j) { return i <= j ? (i * 7 - i * (i - 1) / 2 + (j - i)) : (j * 7 - j * (j - 1) / 2 + (i - j)); }

// (H + lambda I) x = b for a packed symmetric 7 x 7 H by Cholesky.  Returns false if not positive definite.
OVS_BA_HD bool solve7(const double* Hs, double lambda, const double* b, double* x) {
    double Lm[7][7];
    for (int i = 0; i < 7; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = Hs[sym7(j, i)] + (i == j ? lambda : 0.0);
            for (int k = 0; k < j; ++k) s -= Lm[i][k] * Lm[j][k];
            if (i == j) {
                if (!(s > 0.0) || !isfinite(s)) return false;
                Lm[i][i] = sqrt(s);
            } else Lm[i][j] = s / Lm[j][j];
        }
    double y[7];
    for (int i = 0; i < 7; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= Lm[i][k] * y[k];
        y[i] = s / Lm[i][i];
    }
    for (int i = 6; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < 7; ++k) s -= Lm[k][i] * x[k];
        x[i] = s / Lm[i][i];
    }
    return true;
}

// ------------------------------------------------------------------ pose graph (optimize::graph_optimizer, loop closure)
// One Sim3 vertex per keyframe (S_iw, camera from world), one relative edge per keyframe pair with the measurement S_ji:
//   e = log(S_ji S_i S_j^-1),  identity information.
// Jacobians with respect to the left updates S <- exp(d) S of both vertices, analytic:
//   J_i = J_l^-1(e) Ad(S_ji),  J_j = -J_l^-1(e) Ad(E),  E = S_ji S_i S_j^-1,  J_l(xi) = phi(ad xi),  phi(x) = (e^x - 1) / x.

// S^-1 = {R', -R' t / s, 1 / s}
OVS_BA_HD void sim3_inverse(const double* S, double* out) {
    const double is = 1.0 / S[12];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) out[3 * i + j] = S[3 * j + i];
    for (int k = 0; k < 3; ++k) out[9 + k] = -(S[k] * S[9] + S[3 + k] * S[10] + S[6 + k] * S[11]) * is;
    out[12] = is;
}

// A B = {R_a R_b, s_a R_a t_b + t_a, s_a s_b}  (out must not alias A or B)
OVS_BA_HD void sim3_compose(const double* A, const double* B, double* out) {
    double q[3];
    mat3_mat3(A, B, out);
    mat3_vec(A, B + 9, q);
    for (int k = 0; k < 3; ++k) out[9 + k] = A[12] * q[k] + A[9 + k];
    out[12] = A[12] * B[12];
}

// The exact inverse of sim3_exp: sigma = log s; omega from R with the angle atan2(|vee(R - R')| / 2, (tr R - 1) / 2) (accurate
// near 0 and near pi; near pi the axis comes from the symmetric part of R); upsilon = W^-1 t with W read from sim3_exp itself
// (its t for upsilon = e_k is W's column k), so that every branch of the exponential is inverted exactly.
OVS_BA_HD void sim3_log(const double* S, double* xi) {
    const double* R = S;
    const double v[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    const double sn = 0.5 * sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
    const double theta = atan2(sn, c);
    if (c > -0.5) {
        // theta < 2 pi / 3: theta / (2 sin theta) is well conditioned
        // below 1e-5 sim3_exp takes R = I + O + O^2 / 2, whose vee(R - R') / 2 is omega itself
        const double f = theta < 1e-5 ? 0.5 : 0.5 * theta / sn;
        for (int k = 0; k < 3; ++k) xi[k] = f * v[k];
    } else {
        // (R + R') / 2 - cos(theta) I = (1 - cos theta) a a'; the axis from its largest diagonal entry, the sign from vee(R - R')
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
        sim3_exp(u, E);
        for (int r = 0; r < 3; ++r) W[3 * r + col] = E[9 + r];
    }
    // upsilon = W^-1 t by the adjugate
    const double c00 = W[4] * W[8] - W[5] * W[7], c01 = W[5] * W[6] - W[3] * W[8], c02 = W[3] * W[7] - W[4] * W[6];
    const double c10 = W[2] * W[7] - W[1] * W[8], c11 = W[0] * W[8] - W[2] * W[6], c12 = W[1] * W[6] - W[0] * W[7];
    const double c20 = W[1] * W[5] - W[2] * W[4], c21 = W[2] * W[3] - W[0] * W[5], c22 = W[0] * W[4] - W[1] * W[3];
    const double id = 1.0 / (W[0] * c00 + W[1] * c01 + W[2] * c02);
    const double* t = S + 9;
    xi[3] = (c00 * t[0] + c10 * t[1] + c20 * t[2]) * id;
    xi[4] = (c01 * t[0] + c11 * t[1] + c21 * t[2]) * id;
    xi[5] = (c02 * t[0] + c12 * t[1] + c22 * t[2]) * id;
}

// Ad(S) (7 x 7 row-major) in the update order (omega, upsilon, sigma): exp(Ad(S) d) = S exp(d) S^-1
//   [[R, 0, 0], [[t]x R, s R, -t], [0, 0, 1]]
OVS_BA_HD void sim3_adjoint(const double* S, double* Ad) {
    for (int k = 0; k < 49; ++k) Ad[k] = 0.0;
    const double* t = S + 9;
    const double T[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    double TR[9];
    mat3_mat3(T, S, TR);
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

// ad(xi) = [[[w]x, 0, 0], [[u]x, sigma I + [w]x, -u], [0, 0, 0]]
OVS_BA_HD void sim3_ad(const double* xi, double* ad) {
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

// C = A B, 7 x 7 row-major (C must not alias A or B)
OVS_BA_HD void mat7_mul(const double* A, const double* B, double* C) {
    for (int i = 0; i < 7; ++i)
        for (int j = 0; j < 7; ++j) {
            double s = 0.0;
            for (int k = 0; k < 7; ++k) s += A[7 * i + k] * B[7 * k + j];
            C[7 * i + j] = s;
        }
}

// phi(A) = sum_k A^k / (k + 1)! of a 7 x 7 matrix by scaling and squaring: A is halved until its infinity norm is <= 1/2,
// a degree-12 Taylor core (Horner) gives phi there, and phi(2X) = phi(X) (2 I + X phi(X)) / 2 undoes the halving.
OVS_BA_HD void sim3_phi7(const double* A, double* F) {
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
    // Horner: F = I / 13!, then F = I / (k + 1)! + X F for k = 11 .. 0
    double inv_fact[13];
    inv_fact[0] = 1.0;
    for (int k = 1; k < 13; ++k) inv_fact[k] = inv_fact[k - 1] / (double)(k + 1);   // inv_fact[k] = 1 / (k + 1)!
    for (int k = 0; k < 49; ++k) F[k] = (k % 8 == 0) ? inv_fact[12] : 0.0;
    for (int k = 11; k >= 0; --k) {
        mat7_mul(X, F, T);
        for (int m = 0; m < 49; ++m) F[m] = T[m] + ((m % 8 == 0) ? inv_fact[k] : 0.0);
    }
    for (int s = 0; s < sq; ++s) {
        mat7_mul(X, F, T);                                             // X phi(X)
        for (int m = 0; m < 49; ++m) T[m] = 0.5 * T[m] + ((m % 8 == 0) ? 1.0 : 0.0);   // I + X phi(X) / 2
        double Fn[49];
        mat7_mul(F, T, Fn);
        for (int m = 0; m < 49; ++m) { F[m] = Fn[m]; X[m] = 2.0 * X[m]; }
    }
}

// X = M^-1 B for a 7 x 7 M and a 7 x nrhs B (row-major, pitch nrhs) by Gaussian elimination with partial pivoting.
// M and B are overwritten.  Returns false for a singular M.
OVS_BA_HD bool solve7_general(double* M, double* B, int nrhs) {
    for (int c = 0; c < 7; ++c) {
        int p = c;
        for (int r = c + 1; r < 7; ++r)
            if (fabs(M[7 * r + c]) > fabs(M[7 * p + c])) p = r;
        if (!(fabs(M[7 * p + c]) > 0.0)) return false;
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
    return true;
}

// The relative Sim3 edge: e = log(S_ji S_i S_j^-1) (7) and, when J is not null, J = [J_i | J_j] (7 x 14 row-major).
OVS_BA_HD void graph_edge(const double* S_ji, const double* S_i, const double* S_j, double* e, double* J) {
    double Sji_i[13], Sj_inv[13], E[13];
    sim3_compose(S_ji, S_i, Sji_i);
    sim3_inverse(S_j, Sj_inv);
    sim3_compose(Sji_i, Sj_inv, E);
    sim3_log(E, e);
    if (!J) return;
    double Jl[49], ad[49], Ad1[49], Ad2[49];
    sim3_ad(e, ad);
    sim3_phi7(ad, Jl);
    sim3_adjoint(S_ji, Ad1);
    sim3_adjoint(E, Ad2);
    for (int r = 0; r < 7; ++r)
        for (int k = 0; k < 7; ++k) { J[14 * r + k] = Ad1[7 * r + k]; J[14 * r + 7 + k] = -Ad2[7 * r + k]; }
    if (!solve7_general(Jl, J, 14))
        for (int k = 0; k < 98; ++k) J[k] = 0.0;   // J_l is singular only at |omega| = 2 pi k: not reached by log's output
}

// ------------------------------------------------------------------ Sim3 RANSAC (solve::sim3_solver, loop detection)
// Per hypothesis k: three distinct pairs from a counter-based sampler, Horn's closed-form Sim3 S_12 on them (S_21 its inverse),
// and the count of pairs whose points reproject through S_21 / S_12 within 9.21 sigma^2 of their own reprojections.
// Only + - * / sqrt are used (and atan2 / asin for the equirectangular projection), so with contraction off the host and the
// device give the same bits.

// splitmix64's output function
OVS_BA_HD uint64_t splitmix64_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// The m distinct indices of hypothesis k of a problem with n >= m entries: w_j = mix(seed + golden * (m k + j + 1)),
// c_j = w_j % (n - j), then c_j steps past the indices drawn before it, visited in ascending order (+1 for each one <= it).
// No rejection loop.  m = 3 is the Sim3 solver's triple, m = 6 the PnP solver's minimal set.
template <int m>
OVS_BA_HD void ransac_sample(uint64_t seed, int k, int n, int* idx) {
    const uint64_t g = 0x9E3779B97F4A7C15ull, base = (uint64_t)m * (uint64_t)k;
    int sorted[m];                                   // the indices drawn so far, ascending
    for (int j = 0; j < m; ++j) {
        int c = (int)(splitmix64_mix(seed + g * (base + (uint64_t)j + 1)) % (uint64_t)(n - j));
        int pos = 0;
        for (; pos < j && c >= sorted[pos]; ++pos) ++c;
        for (int a = j; a > pos; --a) sorted[a] = sorted[a - 1];
        sorted[pos] = c;
        idx[j] = c;
    }
}

// The three distinct pair indices of hypothesis k of a problem with n >= 3 pairs: ransac_sample with m = 3, i.e.
// i0 = w0 % n, i1 = w1 % (n - 1) skipping i0, i2 = w2 % (n - 2) skipping min(i0, i1), then max(i0, i1).
OVS_BA_HD void sim3_ransac_triple(uint64_t seed, int k, int n, int* idx) { ransac_sample<3>(seed, k, n, idx); }

// Cyclic Jacobi on a symmetric N x N A (row-major, overwritten: its diagonal ends as the eigenvalues); V (row-major) gets the
// eigenvectors as columns.  Sweeps visit (p, q) for p < q in row-major order; a sweep starts only while the off-diagonal sum of
// squares exceeds 1e-30 of the matrix's (at entry), at most 16 sweeps.  Rotation: theta = (a_qq - a_pp) / (2 a_pq),
// t = sign(theta) / (|theta| + sqrt(theta^2 + 1)), c = 1 / sqrt(t^2 + 1), s = t c; a_pq is set to zero after it.
template <int N>
OVS_BA_HD void jacobi_sym(double* A, double* V) {
    for (int k = 0; k < N * N; ++k) V[k] = (k % (N + 1) == 0) ? 1.0 : 0.0;
    double frob = 0.0;
    for (int k = 0; k < N * N; ++k) frob += A[k] * A[k];
    for (int sweep = 0; sweep < 16; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) off += A[N * p + q] * A[N * p + q];
        if (!(off > 1e-30 * frob)) break;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[N * p + q];
                if (apq == 0.0) continue;
                const double theta = (A[N * q + q] - A[N * p + p]) / (2.0 * apq);
                double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
                if (theta < 0.0) t = -t;
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int r = 0; r < N; ++r) {      // columns p, q
                    const double arp = A[N * r + p], arq = A[N * r + q];
                    A[N * r + p] = c * arp - s * arq;
                    A[N * r + q] = s * arp + c * arq;
                }
                for (int r = 0; r < N; ++r) {      // rows p, q
                    const double apr = A[N * p + r], aqr = A[N * q + r];
                    A[N * p + r] = c * apr - s * aqr;
                    A[N * q + r] = s * apr + c * aqr;
                }
                A[N * p + q] = 0.0; A[N * q + p] = 0.0;
                for (int r = 0; r < N; ++r) {
                    const double vrp = V[N * r + p], vrq = V[N * r + q];
                    V[N * r + p] = c * vrp - s * vrq;
                    V[N * r + q] = s * vrp + c * vrq;
                }
            }
    }
}

OVS_BA_HD void jacobi4(double* A, double* V) { jacobi_sym<4>(A, V); }

// The rotation of absolute orientation from the correlation M = sum (a - a0)(b - b0)^T of centred source points a and target
// points b (M[3 * r + c]: source coordinate r, target coordinate c): Horn's 4 x 4 N, the quaternion (w, x, y, z) = the
// eigenvector of N's largest eigenvalue (lowest index on ties), R (row-major, b ~ R a) directly from it (divided by |q|^2).
OVS_BA_HD void horn_rotation(const double* M, double* R) {
    const double Sxx = M[0], Sxy = M[1], Sxz = M[2], Syx = M[3], Syy = M[4], Syz = M[5], Szx = M[6], Szy = M[7], Szz = M[8];
    double N[16] = {Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx,
                    Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz,
                    Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy,
                    Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz};
    double V[16];
    jacobi4(N, V);
    int m = 0;
    for (int k = 1; k < 4; ++k)
        if (N[5 * k] > N[5 * m]) m = k;
    const double w = V[m], x = V[4 + m], y = V[8 + m], z = V[12 + m];
    const double nq = w * w + x * x + y * y + z * z;
    R[0] = (w * w + x * x - y * y - z * z) / nq; R[1] = 2.0 * (x * y - w * z) / nq;         R[2] = 2.0 * (x * z + w * y) / nq;
    R[3] = 2.0 * (x * y + w * z) / nq;         R[4] = (w * w - x * x + y * y - z * z) / nq; R[5] = 2.0 * (y * z - w * x) / nq;
    R[6] = 2.0 * (x * z - w * y) / nq;         R[7] = 2.0 * (y * z + w * x) / nq;         R[8] = (w * w - x * x - y * y + z * z) / nq;
}

// compute_Sim3 by Horn's closed form on three point pairs (p1[3 * j + c]: point j in keyframe 1's camera frame, p2 likewise):
// centroids, M = A2 A1^T, R_12 = horn_rotation(M), s = sum A1 . (R A2) / sum |A2|^2 (1 with fix_scale), t = c1 - s R c2.
// S_21 = S_12^-1.  Coincident or collinear points are not special-cased.
OVS_BA_HD void sim3_horn(const double* p1, const double* p2, bool fix_scale, double* S12, double* S21) {
    double c1[3], c2[3], A1[9], A2[9];   // A[3 * r + j]: coordinate r of centred point j
    for (int r = 0; r < 3; ++r) {
        c1[r] = (p1[r] + p1[3 + r] + p1[6 + r]) / 3.0;
        c2[r] = (p2[r] + p2[3 + r] + p2[6 + r]) / 3.0;
        for (int j = 0; j < 3; ++j) { A1[3 * r + j] = p1[3 * j + r] - c1[r]; A2[3 * r + j] = p2[3 * j + r] - c2[r]; }
    }
    double M[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) M[3 * a + b] = A2[3 * a] * A1[3 * b] + A2[3 * a + 1] * A1[3 * b + 1] + A2[3 * a + 2] * A1[3 * b + 2];
    double* R = S12;
    horn_rotation(M, R);
    double s = 1.0;
    if (!fix_scale) {
        double num = 0.0, den = 0.0;
        for (int j = 0; j < 3; ++j) {
            const double a2[3] = {A2[j], A2[3 + j], A2[6 + j]};
            double ra[3];
            mat3_vec(R, a2, ra);
            num += A1[j] * ra[0] + A1[3 + j] * ra[1] + A1[6 + j] * ra[2];
            den += a2[0] * a2[0] + a2[1] * a2[1] + a2[2] * a2[2];
        }
        s = num / den;
    }
    double rc2[3];
    mat3_vec(R, c2, rc2);
    for (int r = 0; r < 3; ++r) S12[9 + r] = c1[r] - s * rc2[r];
    S12[12] = s;
    sim3_inverse(S12, S21);
}

// camera::reproject_to_image(rot_cw, trans_cw, p) as the reference writes it, p_c = rot_cw p + trans_cw; false when the
// perspective point is not in front of the camera (the reference returns before writing the reprojection).  The in-image
// result is not reported.
OVS_BA_HD bool ransac_reproject(const CameraD& cam, const double* rot, const double* trans, const double* p, double* uv) {
    double pc[3];
    mat3_vec(rot, p, pc);
    for (int k = 0; k < 3; ++k) pc[k] += trans[k];
    if (cam.model == kCamEquirectangular) {
        const double L = sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
        const double bx = pc[0] / L, by = pc[1] / L, bz = pc[2] / L;
        const double latitude = -asin(by), longitude = atan2(bx, bz);
        uv[0] = cam.cols * (0.5 + longitude / (2.0 * kPi));
        uv[1] = cam.rows * (0.5 - latitude / kPi);
        return true;
    }
    if (pc[2] <= 0.0) return false;
    const double z_inv = 1.0 / pc[2];
    uv[0] = cam.fx * pc[0] * z_inv + cam.cx;
    uv[1] = cam.fy * pc[1] * z_inv + cam.cy;
    return true;
}

// rot_cw = s R, formed element-wise before the projection (reproject_to_other_image)
OVS_BA_HD void sim3_scaled_rotation(const double* S, double* sR) {
    for (int k = 0; k < 9; ++k) sR[k] = S[12] * S[k];
}

// The bound of one side of a pair: 9.21034f * sigma^2 in float, or -1 (never met) when the pair's own reprojection on that side
// does not exist (a perspective point behind its camera).
OVS_BA_HD float ransac_bound(float sigma_sq, bool own_ok) { return own_ok ? 9.21034f * sigma_sq : -1.0f; }

// count_inliers for one pair: |pi_2(S_21 pc1) - reproj_2|^2 < bound_2 and |pi_1(S_12 pc2) - reproj_1|^2 < bound_1, both strict;
// a projection behind its camera is not an inlier.  sR / t: the scaled rotations and translations of S_12 and S_21.
OVS_BA_HD bool ransac_is_inlier(const CameraD& cam1, const CameraD& cam2, const double* sR12, const double* t12, const double* sR21,
                                const double* t21, const double* pc1, const double* pc2, const double* reproj1, const double* reproj2,
                                float bound1, float bound2) {
    double u2[2], u1[2];
    if (!ransac_reproject(cam2, sR21, t21, pc1, u2)) return false;
    if (!ransac_reproject(cam1, sR12, t12, pc2, u1)) return false;
    const double d2x = u2[0] - reproj2[0], d2y = u2[1] - reproj2[1];
    const double d1x = u1[0] - reproj1[0], d1y = u1[1] - reproj1[1];
    const double e2 = d2x * d2x + d2y * d2y, e1 = d1x * d1x + d1y * d1y;
    return e2 < (double)bound2 && e1 < (double)bound1;
}

}  // namespace ovs
