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

}  // namespace ovs
