/*
 * oracle/sim3_solver_oracle.c -- CPU restatement (FP64) of OpenVSLAM's solve::sim3_solver (loop detection: the Sim3 between the
 * current keyframe and a loop candidate, by RANSAC over Horn's closed form on three landmark pairs), constructor and
 * find_via_ransac(max_num_iter), restated from memory.
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes (the kernel's csrc/sim3_math.cuh follows them operation for operation):
 *  - the sampler is counter-based and seeded per problem (the reference draws from std::random_device);
 *  - N's eigenvector comes from a cyclic Jacobi with a fixed sweep order and stop rule (not Eigen's SelfAdjointEigenSolver);
 *    the lowest index wins among equal eigenvalues;
 *  - R is formed from the quaternion directly (not through atan2 and Rodrigues), the scale is a double;
 *  - a perspective point behind its camera is not an inlier (the reference leaves the reprojection unwritten).
 * Checks: tests/test_sim3_solver_oracle.py (numpy Umeyama / eigh, a numpy sampler and count_inliers, the kernel header
 * compiled for the host).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "sim3_solver_oracle.h"

static const double OS_PI = 3.14159265358979323846;

static void os_mat3_vec(const double* R, const double* v, double* o) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}

uint64_t os_splitmix64_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* w_j = mix(seed + 0x9E3779B97F4A7C15 (3k + j + 1)); i0 = w0 % n; i1 = w1 % (n - 1), stepped past i0; i2 = w2 % (n - 2), stepped
 * past the smaller and then the larger of i0, i1 */
void os_ransac_triple(uint64_t seed, int k, int n, int* idx) {
    const uint64_t golden = 0x9E3779B97F4A7C15ull;
    uint64_t w[3];
    for (int j = 0; j < 3; ++j) w[j] = os_splitmix64_mix(seed + golden * (3ull * (uint64_t)k + (uint64_t)j + 1ull));
    const int a = (int)(w[0] % (uint64_t)n);
    const int c = (int)(w[1] % (uint64_t)(n - 1));
    const int d = (int)(w[2] % (uint64_t)(n - 2));
    const int i1 = c >= a ? c + 1 : c;
    const int lo = a < i1 ? a : i1, hi = a < i1 ? i1 : a;
    int i2 = d;
    if (i2 >= lo) i2 += 1;
    if (i2 >= hi) i2 += 1;
    idx[0] = a; idx[1] = i1; idx[2] = i2;
}

void os_jacobi4(const double* A_in, double* evals, double* V) {
    double A[4][4];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) { A[r][c] = A_in[4 * r + c]; V[4 * r + c] = r == c ? 1.0 : 0.0; }
    double frob = 0.0;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) frob += A[r][c] * A[r][c];
    for (int sweep = 0; sweep < 16; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 3; ++p)
            for (int q = p + 1; q < 4; ++q) off += A[p][q] * A[p][q];
        if (!(off > 1e-30 * frob)) break;
        for (int p = 0; p < 3; ++p)
            for (int q = p + 1; q < 4; ++q) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
                if (theta < 0.0) t = -t;
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int r = 0; r < 4; ++r) {
                    const double arp = A[r][p], arq = A[r][q];
                    A[r][p] = c * arp - s * arq;
                    A[r][q] = s * arp + c * arq;
                }
                for (int r = 0; r < 4; ++r) {
                    const double apr = A[p][r], aqr = A[q][r];
                    A[p][r] = c * apr - s * aqr;
                    A[q][r] = s * apr + c * aqr;
                }
                A[p][q] = 0.0; A[q][p] = 0.0;
                for (int r = 0; r < 4; ++r) {
                    const double vrp = V[4 * r + p], vrq = V[4 * r + q];
                    V[4 * r + p] = c * vrp - s * vrq;
                    V[4 * r + q] = s * vrp + c * vrq;
                }
            }
    }
    for (int k = 0; k < 4; ++k) evals[k] = A[k][k];
}

void os_horn(const double* p1, const double* p2, int fix_scale, double* S12, double* S21) {
    double c1[3], c2[3], A1[3][3], A2[3][3];
    for (int r = 0; r < 3; ++r) {
        c1[r] = (p1[r] + p1[3 + r] + p1[6 + r]) / 3.0;
        c2[r] = (p2[r] + p2[3 + r] + p2[6 + r]) / 3.0;
    }
    for (int r = 0; r < 3; ++r)
        for (int j = 0; j < 3; ++j) { A1[r][j] = p1[3 * j + r] - c1[r]; A2[r][j] = p2[3 * j + r] - c2[r]; }
    double M[3][3];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) M[a][b] = A2[a][0] * A1[b][0] + A2[a][1] * A1[b][1] + A2[a][2] * A1[b][2];
    const double Sxx = M[0][0], Sxy = M[0][1], Sxz = M[0][2], Syx = M[1][0], Syy = M[1][1], Syz = M[1][2];
    const double Szx = M[2][0], Szy = M[2][1], Szz = M[2][2];
    const double N[16] = {Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx,
                          Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz,
                          Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy,
                          Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz};
    double ev[4], V[16];
    os_jacobi4(N, ev, V);
    int m = 0;
    for (int k = 1; k < 4; ++k)
        if (ev[k] > ev[m]) m = k;
    const double w = V[m], x = V[4 + m], y = V[8 + m], z = V[12 + m];
    const double nq = w * w + x * x + y * y + z * z;
    double R[9];
    R[0] = (w * w + x * x - y * y - z * z) / nq; R[1] = 2.0 * (x * y - w * z) / nq; R[2] = 2.0 * (x * z + w * y) / nq;
    R[3] = 2.0 * (x * y + w * z) / nq; R[4] = (w * w - x * x + y * y - z * z) / nq; R[5] = 2.0 * (y * z - w * x) / nq;
    R[6] = 2.0 * (x * z - w * y) / nq; R[7] = 2.0 * (y * z + w * x) / nq; R[8] = (w * w - x * x - y * y + z * z) / nq;
    double s = 1.0;
    if (!fix_scale) {
        double num = 0.0, den = 0.0;
        for (int j = 0; j < 3; ++j) {
            const double a2[3] = {A2[0][j], A2[1][j], A2[2][j]};
            double ra[3];
            os_mat3_vec(R, a2, ra);
            num += A1[0][j] * ra[0] + A1[1][j] * ra[1] + A1[2][j] * ra[2];
            den += a2[0] * a2[0] + a2[1] * a2[1] + a2[2] * a2[2];
        }
        s = num / den;
    }
    double rc2[3];
    os_mat3_vec(R, c2, rc2);
    memcpy(S12, R, sizeof(R));
    for (int r = 0; r < 3; ++r) S12[9 + r] = c1[r] - s * rc2[r];
    S12[12] = s;
    /* S_21 = {R^T, -R^T t / s, 1 / s} */
    const double is = 1.0 / s;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) S21[3 * i + j] = R[3 * j + i];
    for (int k = 0; k < 3; ++k) S21[9 + k] = -(R[k] * S12[9] + R[3 + k] * S12[10] + R[6 + k] * S12[11]) * is;
    S21[12] = is;
}

int os_reproject(const ob_camera* cam, const double* rot, const double* trans, const double* p, double* uv) {
    double pc[3];
    os_mat3_vec(rot, p, pc);
    for (int k = 0; k < 3; ++k) pc[k] += trans[k];
    if (cam->model == 1) {   /* equirectangular: longitude / latitude of the normalised bearing */
        const double L = sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
        const double bx = pc[0] / L, by = pc[1] / L, bz = pc[2] / L;
        const double latitude = -asin(by), longitude = atan2(bx, bz);
        uv[0] = cam->cols * (0.5 + longitude / (2.0 * OS_PI));
        uv[1] = cam->rows * (0.5 - latitude / OS_PI);
        return 1;
    }
    if (pc[2] <= 0.0) return 0;
    const double z_inv = 1.0 / pc[2];
    uv[0] = cam->fx * pc[0] * z_inv + cam->cx;
    uv[1] = cam->fy * pc[1] * z_inv + cam->cy;
    return 1;
}

/* count_inliers: both reprojection errors strictly below their bounds; a reprojection behind its camera is no inlier */
static int os_count_inliers(const ob_camera* cam_1, const ob_camera* cam_2, const double* S12, const double* S21, int n,
                            const double* pc1, const double* pc2, const double* rp1, const double* rp2, const int* own_ok,
                            const float* bound1, const float* bound2, uint8_t* flags) {
    double sR12[9], sR21[9];
    for (int k = 0; k < 9; ++k) { sR12[k] = S12[12] * S12[k]; sR21[k] = S21[12] * S21[k]; }
    int count = 0;
    for (int i = 0; i < n; ++i) {
        double u2[2], u1[2];
        int in = own_ok[i] && os_reproject(cam_2, sR21, S21 + 9, pc1 + 3 * i, u2) && os_reproject(cam_1, sR12, S12 + 9, pc2 + 3 * i, u1);
        if (in) {
            const double d2x = u2[0] - rp2[2 * i], d2y = u2[1] - rp2[2 * i + 1];
            const double d1x = u1[0] - rp1[2 * i], d1y = u1[1] - rp1[2 * i + 1];
            const double e2 = d2x * d2x + d2y * d2y, e1 = d1x * d1x + d1y * d1y;
            in = e2 < (double)bound2[i] && e1 < (double)bound1[i];
        }
        if (flags) flags[i] = (uint8_t)in;
        count += in;
    }
    return count;
}

void os_sim3_solve_ransac(const ob_camera* cam_1, const ob_camera* cam_2, const double* pose_1w, const double* pose_2w, int n,
                          const double* pos_w_1, const float* sigma_sq_1, const double* pos_w_2, const float* sigma_sq_2, int fix_scale,
                          int min_num_inliers, int max_num_iter, uint64_t seed, double* sim3_12, int* valid, int* num_inliers,
                          int* best_iter, uint8_t* inlier_out, int* hyp_idx, int* hyp_count) {
    for (int k = 0; k < 13; ++k) sim3_12[k] = (k == 0 || k == 4 || k == 8 || k == 12) ? 1.0 : 0.0;
    *valid = 0; *num_inliers = 0; *best_iter = -1;
    for (int i = 0; i < n; ++i) inlier_out[i] = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        if (hyp_idx) hyp_idx[3 * k] = hyp_idx[3 * k + 1] = hyp_idx[3 * k + 2] = -1;
        if (hyp_count) hyp_count[k] = 0;
    }
    if (n < 3 || n < min_num_inliers) return;
    /* the constructor: camera-frame points, their own reprojections, chi_sq_2D * sigma^2 in float */
    double* pc1 = malloc(sizeof(double) * 3 * n); double* pc2 = malloc(sizeof(double) * 3 * n);
    double* rp1 = malloc(sizeof(double) * 2 * n); double* rp2 = malloc(sizeof(double) * 2 * n);
    float* b1 = malloc(sizeof(float) * n); float* b2 = malloc(sizeof(float) * n);
    int* own_ok = malloc(sizeof(int) * n);
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
    for (int i = 0; i < n; ++i) {
        os_mat3_vec(pose_1w, pos_w_1 + 3 * i, pc1 + 3 * i);
        os_mat3_vec(pose_2w, pos_w_2 + 3 * i, pc2 + 3 * i);
        for (int k = 0; k < 3; ++k) { pc1[3 * i + k] += pose_1w[9 + k]; pc2[3 * i + k] += pose_2w[9 + k]; }
        const int ok1 = os_reproject(cam_1, I, zero, pc1 + 3 * i, rp1 + 2 * i);
        const int ok2 = os_reproject(cam_2, I, zero, pc2 + 3 * i, rp2 + 2 * i);
        own_ok[i] = ok1 && ok2;
        b1[i] = 9.21034f * sigma_sq_1[i];
        b2[i] = 9.21034f * sigma_sq_2[i];
    }
    int best = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        int idx[3];
        os_ransac_triple(seed, k, n, idx);
        double q1[9], q2[9], S12[13], S21[13];
        for (int j = 0; j < 3; ++j)
            for (int c = 0; c < 3; ++c) { q1[3 * j + c] = pc1[3 * idx[j] + c]; q2[3 * j + c] = pc2[3 * idx[j] + c]; }
        os_horn(q1, q2, fix_scale, S12, S21);
        const int count = os_count_inliers(cam_1, cam_2, S12, S21, n, pc1, pc2, rp1, rp2, own_ok, b1, b2, NULL);
        if (hyp_idx) { hyp_idx[3 * k] = idx[0]; hyp_idx[3 * k + 1] = idx[1]; hyp_idx[3 * k + 2] = idx[2]; }
        if (hyp_count) hyp_count[k] = count;
        if (count > best) {
            best = count;
            *best_iter = k;
            memcpy(sim3_12, S12, sizeof(S12));
            os_count_inliers(cam_1, cam_2, S12, S21, n, pc1, pc2, rp1, rp2, own_ok, b1, b2, inlier_out);
        }
    }
    *num_inliers = best;
    *valid = best >= min_num_inliers;
    free(pc1); free(pc2); free(rp1); free(rp2); free(b1); free(b2); free(own_ok);
}
