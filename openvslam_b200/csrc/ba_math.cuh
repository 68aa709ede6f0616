// ba_math.cuh -- FP64 residual / Jacobian / SE3 arithmetic of the pose optimiser and the local
// bundle adjuster (optimize/g2o/se3/{perspective,equirectangular}_{reproj,pose_opt}_edge.cc,
// shot_vertex.h, g2o se3quat.h / robust_kernel_impl.cpp; names as in SURVEY.md 8a a13-a15).
// __host__ __device__ so tests/hostcheck can compare the same code with the oracle on the CPU.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define OVS_BA_HD __host__ __device__ __forceinline__
#else
#define OVS_BA_HD static inline
#endif

namespace ovs {

constexpr int kCamPerspective = 0;
constexpr int kCamEquirectangular = 1;
constexpr double kPi = 3.14159265358979323846;

struct CameraD {
    int model;
    double fx, fy, cx, cy, fb, cols, rows;
};

OVS_BA_HD void mat3_vec(const double* R, const double* v, double* o) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
OVS_BA_HD void mat3_mat3(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// shot_vertex::oplusImpl: estimate <- SE3Quat::exp(update) * estimate; update = [omega, upsilon];
// pose = {R row-major (9), t (3)}.
OVS_BA_HD void pose_oplus(const double* pose, const double* u, double* out) {
    const double wx = u[0], wy = u[1], wz = u[2];
    const double theta = sqrt(wx * wx + wy * wy + wz * wz);
    const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    double O2[9];
    mat3_mat3(O, O, O2);
    double a, b, c;
    if (theta < 0.00001) { a = 1.0; b = 0.5; c = 1.0 / 6.0; }
    else {
        a = sin(theta) / theta;
        b = (1 - cos(theta)) / (theta * theta);
        c = (theta - sin(theta)) / (theta * theta * theta);
    }
    double Rd[9], V[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i == 0 || i == 4 || i == 8) ? 1.0 : 0.0;
        Rd[i] = I + a * O[i] + b * O2[i];
        V[i] = I + b * O[i] + c * O2[i];
    }
    double td[3], tn[3];
    mat3_vec(V, u + 3, td);
    mat3_mat3(Rd, pose, out);
    mat3_vec(Rd, pose + 9, tn);
    out[9] = tn[0] + td[0]; out[10] = tn[1] + td[1]; out[11] = tn[2] + td[2];
}

// Residual e = obs - project(R pw + t); Jacobians wrt the pose update (Jp: dim x 6) and the
// landmark (Jl: dim x 3), either may be null.  Returns dim (2 mono, 3 stereo).
OVS_BA_HD int edge_eval(const CameraD& cam, const double* pose, const double* pw, const double* obs, bool stereo,
                        double* e, double* Jp, double* Jl) {
    double pc[3];
    mat3_vec(pose, pw, pc);
    pc[0] += pose[9]; pc[1] += pose[10]; pc[2] += pose[11];
    const double x = pc[0], y = pc[1], z = pc[2];
    const double* R = pose;
    if (cam.model == kCamEquirectangular) {
        const double L = sqrt(x * x + y * y + z * z);
        const double theta = atan2(x, z);
        const double phi = -asin(y / L);
        e[0] = obs[0] - cam.cols * (0.5 + theta / (2 * kPi));
        e[1] = obs[1] - cam.rows * (0.5 - phi / kPi);
        if (Jp || Jl) {
            const double dpc[3][9] = {
                {0, z, -y, 1, 0, 0, R[0], R[1], R[2]},
                {-z, 0, x, 0, 1, 0, R[3], R[4], R[5]},
                {y, -x, 0, 0, 0, 1, R[6], R[7], R[8]}};
            const double xz2 = x * x + z * z;
            const double c0 = -(cam.cols / (2 * kPi)) * (1.0 / xz2);
            const double c1 = -(cam.rows / kPi) * (1.0 / (L * sqrt(xz2)));
            for (int k = 0; k < 9; ++k) {
                const double dL = (1.0 / L) * (x * dpc[0][k] + y * dpc[1][k] + z * dpc[2][k]);
                const double j0 = c0 * (z * dpc[0][k] - x * dpc[2][k]);
                const double j1 = c1 * (L * dpc[1][k] - y * dL);
                if (k < 6) { if (Jp) { Jp[k] = j0; Jp[6 + k] = j1; } }
                else if (Jl) { Jl[k - 6] = j0; Jl[3 + k - 6] = j1; }
            }
        }
        return 2;
    }
    const double fx = cam.fx, fy = cam.fy, fb = cam.fb;
    const double z_sq = z * z;
    const double reproj_x = fx * x / z + cam.cx;
    e[0] = obs[0] - reproj_x;
    e[1] = obs[1] - (fy * y / z + cam.cy);
    if (stereo) e[2] = obs[2] - (reproj_x - fb / z);
    if (Jl) {
        for (int k = 0; k < 3; ++k) {
            Jl[k] = -fx * R[k] / z + fx * x * R[6 + k] / z_sq;
            Jl[3 + k] = -fy * R[3 + k] / z + fy * y * R[6 + k] / z_sq;
            if (stereo) Jl[6 + k] = Jl[k] - fb * R[6 + k] / z_sq;
        }
    }
    if (Jp) {
        Jp[0] = x * y / z_sq * fx; Jp[1] = -(1.0 + (x * x / z_sq)) * fx; Jp[2] = y / z * fx;
        Jp[3] = -1.0 / z * fx; Jp[4] = 0.0; Jp[5] = x / z_sq * fx;
        Jp[6] = (1.0 + y * y / z_sq) * fy; Jp[7] = -x * y / z_sq * fy; Jp[8] = -x / z * fy;
        Jp[9] = 0.0; Jp[10] = -1.0 / z * fy; Jp[11] = y / z_sq * fy;
        if (stereo) {
            Jp[12] = Jp[0] - fb * y / z_sq; Jp[13] = Jp[1] + fb * x / z_sq; Jp[14] = Jp[2];
            Jp[15] = Jp[3]; Jp[16] = 0.0; Jp[17] = Jp[5] - fb / z_sq;
        }
    }
    return stereo ? 3 : 2;
}

// g2o::RobustKernelHuber::robustify: rho[0] = robust cost, rho[1] = weight.
OVS_BA_HD void huber(double e2, double delta, double* rho0, double* rho1) {
    const double dsqr = delta * delta;
    if (e2 <= dsqr) { *rho0 = e2; *rho1 = 1.0; }
    else {
        const double sqrte = sqrt(e2);
        *rho0 = 2 * sqrte * delta - dsqr;
        *rho1 = delta / sqrte;
    }
}

// Inverse of a symmetric 3x3 given as {d00, d01, d02, d11, d12, d22}; same packed output.
OVS_BA_HD bool inv3_sym(const double* D, double* Di) {
    const double a = D[0], b = D[1], c = D[2], d = D[3], e = D[4], f = D[5];
    const double c00 = d * f - e * e, c01 = c * e - b * f, c02 = b * e - c * d;
    const double det = a * c00 + b * c01 + c * c02;
    if (det == 0.0 || !isfinite(det)) return false;
    const double id = 1.0 / det;
    Di[0] = c00 * id; Di[1] = c01 * id; Di[2] = c02 * id;
    Di[3] = (a * f - c * c) * id; Di[4] = (b * c - a * e) * id; Di[5] = (a * d - b * b) * id;
    return true;
}

// Index of element (i, j) of a packed symmetric N x N (upper triangle, row-major).
template <int N>
OVS_BA_HD int sym(int i, int j) { return i <= j ? (i * N - i * (i - 1) / 2 + (j - i)) : (j * N - j * (j - 1) / 2 + (i - j)); }
OVS_BA_HD int sym3(int i, int j) { return sym<3>(i, j); }
OVS_BA_HD int sym6(int i, int j) { return sym<6>(i, j); }

// (H + lambda I) x = b for a packed symmetric N x N H by Cholesky (thread-local).  Returns false if not positive definite.
template <int N>
OVS_BA_HD bool solve_spd(const double* Hs, double lambda, const double* b, double* x) {
    double Lm[N][N];
    for (int i = 0; i < N; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = Hs[sym<N>(j, i)] + (i == j ? lambda : 0.0);
            for (int k = 0; k < j; ++k) s -= Lm[i][k] * Lm[j][k];
            if (i == j) {
                if (!(s > 0.0) || !isfinite(s)) return false;
                Lm[i][i] = sqrt(s);
            } else Lm[i][j] = s / Lm[j][j];
        }
    double y[N];
    for (int i = 0; i < N; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= Lm[i][k] * y[k];
        y[i] = s / Lm[i][i];
    }
    for (int i = N - 1; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < N; ++k) s -= Lm[k][i] * x[k];
        x[i] = s / Lm[i][i];
    }
    return true;
}

// ---- per-edge blocks of the normal equations from the edge's Jacobians, residual and robust weight ww (= rho'(chi2) * info)
// The bundle adjusters store only {Jp, Jl, ww, e} per edge and form these blocks where they are read, in several kernels; the
// results must not depend on which kernel forms them, so every product and sum is rounded explicitly, in one fixed order:
// h = 0, then h += (J[d][a] * ww) * J'[d][b] for d < dim.  dim is the edge's own row count (2, or 3 for a stereo edge); rows
// beyond it are never added, not even as zeros (+0.0 would turn a -0.0 sum into +0.0).  R = rows of the arrays (>= dim).
OVS_BA_HD double rn_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
OVS_BA_HD double rn_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
OVS_BA_HD double rn_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}

// Jp' W Jl (6 x 3): out(a, b, element) as each element is formed (a consumer that parks the block elsewhere keeps no copy)
template <int R, class Out>
OVS_BA_HD void edge_hpl_each(const double* Jp, const double* Jl, double ww, int dim, Out&& out) {
    for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 3; ++b) {
            double h = 0;
            for (int d = 0; d < R; ++d)
                if (d < dim) h = rn_add(h, rn_mul(rn_mul(Jp[6 * d + a], ww), Jl[3 * d + b]));
            out(a, b, h);
        }
}
// Jp' W Jl (6 x 3, row-major): W[3 a + b]
template <int R>
OVS_BA_HD void edge_hpl(const double* Jp, const double* Jl, double ww, int dim, double* W) {
    edge_hpl_each<R>(Jp, Jl, ww, dim, [W](int a, int b, double h) { W[3 * a + b] = h; });
}
// Jl' W Jl (3 x 3, packed upper triangle, sym3)
template <int R>
OVS_BA_HD void edge_hll(const double* Jl, double ww, int dim, double* A) {
    for (int a = 0; a < 3; ++a)
        for (int b = a; b < 3; ++b) {
            double h = 0;
            for (int d = 0; d < R; ++d)
                if (d < dim) h = rn_add(h, rn_mul(rn_mul(Jl[3 * d + a], ww), Jl[3 * d + b]));
            A[sym3(a, b)] = h;
        }
}
// Jp' W Jp (6 x 6, packed upper triangle, sym6)
template <int R>
OVS_BA_HD void edge_hpp(const double* Jp, double ww, int dim, double* C) {
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) {
            double h = 0;
            for (int d = 0; d < R; ++d)
                if (d < dim) h = rn_add(h, rn_mul(rn_mul(Jp[6 * d + a], ww), Jp[6 * d + b]));
            C[sym6(a, b)] = h;
        }
}
// -Jp' W e (6)
template <int R>
OVS_BA_HD void edge_bp(const double* Jp, double ww, const double* e, int dim, double* bp) {
    for (int a = 0; a < 6; ++a) {
        double g = 0;
        for (int d = 0; d < R; ++d)
            if (d < dim) g = rn_sub(g, rn_mul(rn_mul(Jp[6 * d + a], ww), e[d]));
        bp[a] = g;
    }
}
// -Jl' W e (3)
template <int R>
OVS_BA_HD void edge_bl(const double* Jl, double ww, const double* e, int dim, double* bl) {
    for (int a = 0; a < 3; ++a) {
        double g = 0;
        for (int d = 0; d < R; ++d)
            if (d < dim) g = rn_sub(g, rn_mul(rn_mul(Jl[3 * d + a], ww), e[d]));
        bl[a] = g;
    }
}

}  // namespace ovs
