/*
 * oracle/pnp_solver_oracle.c -- CPU restatement (FP64) of OpenVSLAM's solve::pnp_solver (relocalisation: the pose of the current
 * frame from its 2D-3D matches with a candidate keyframe's landmarks, by RANSAC over EPnP on minimal sets), constructor and
 * find_via_ransac(max_num_iter, recompute), restated from memory.
 *
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: **parity unpinned** (no reference source here; DESIGN.md 5).
 * Conventions this file fixes (the kernel's csrc/pnp_math.cuh follows them operation for operation):
 *  - the sampler is counter-based and seeded per problem (the reference draws from std::random_device); minimal set of 6;
 *  - EPnP in the bearing form: rows [a_j w, 0, -a_j u] and [0, a_j w, -a_j v]; eigenvectors by a cyclic Jacobi (fixed sweep
 *    order and stop rule), ordered by eigenvalue with the lowest index on ties, each signed so that its entry of largest
 *    magnitude is positive; betas by Householder least squares; R by Horn's quaternion (not an SVD); the sign of the
 *    camera-frame control points from b . p_c of the first correspondence; the error is the mean (1 - cos);
 *  - every sum over points follows one order: 256 strided partials from 0, then their running sum (for n <= 256 the plain
 *    running sum);
 *  - the angular bound cos(pi / 180 * scale_factor) is a fixed polynomial (+ - * / only), so host and device agree.
 * Checks: tests/test_pnp_solver_oracle.py (cv2.solvePnP's EPnP, a numpy restatement, a numpy sampler and check_inliers, the
 * kernel header compiled for the host).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "pnp_solver_oracle.h"

#define OP_MIN_SET 6
#define OP_SLOTS 256

static uint64_t op_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* w_j = mix(seed + 0x9E3779B97F4A7C15 (m k + j + 1)); c_j = w_j % (n - j), then +1 for every earlier index <= it, in ascending
 * order of the earlier indices */
void op_ransac_sample(uint64_t seed, int k, int n, int m, int* idx) {
    const uint64_t golden = 0x9E3779B97F4A7C15ull;
    int sorted[16];
    for (int j = 0; j < m; ++j) {
        int c = (int)(op_mix(seed + golden * ((uint64_t)m * (uint64_t)k + (uint64_t)j + 1ull)) % (uint64_t)(n - j));
        int pos = 0;
        while (pos < j && c >= sorted[pos]) { ++c; ++pos; }
        memmove(sorted + pos + 1, sorted + pos, sizeof(int) * (size_t)(j - pos));
        sorted[pos] = c;
        idx[j] = c;
    }
}

void op_jacobi(int N, const double* A_in, double* evals, double* V) {
    double A[144];
    for (int k = 0; k < N * N; ++k) { A[k] = A_in[k]; V[k] = (k % (N + 1) == 0) ? 1.0 : 0.0; }
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
                for (int r = 0; r < N; ++r) {
                    const double arp = A[N * r + p], arq = A[N * r + q];
                    A[N * r + p] = c * arp - s * arq;
                    A[N * r + q] = s * arp + c * arq;
                }
                for (int r = 0; r < N; ++r) {
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
    for (int k = 0; k < N; ++k) evals[k] = A[(N + 1) * k];
}

/* eigenvector `rank` (descending or ascending eigenvalue, lowest index on ties), signed: largest-magnitude entry positive */
static void op_eigvec(int N, const double* ev, const double* V, int descending, int rank, double* v) {
    int used[12] = {0}, col = 0;
    for (int r = 0; r <= rank; ++r) {
        int m = -1;
        for (int k = 0; k < N; ++k) {
            if (used[k]) continue;
            if (m < 0 || (descending ? ev[k] > ev[m] : ev[k] < ev[m])) m = k;
        }
        used[m] = 1;
        col = m;
    }
    int a = 0;
    for (int r = 1; r < N; ++r)
        if (fabs(V[N * r + col]) > fabs(V[N * a + col])) a = r;
    const double sg = V[N * a + col] < 0.0 ? -1.0 : 1.0;
    for (int r = 0; r < N; ++r) v[r] = sg * V[N * r + col];
}

double op_max_cos(float scale_factor) {
    const double x = 3.14159265358979323846 / 180.0 * (double)scale_factor;
    if (x <= 0.7853981633974483) {   /* Taylor series of cos to x^26 */
        const double x2 = x * x;
        double p = 1.0;
        for (int k = 13; k >= 1; --k) p = 1.0 - x2 / (double)((2 * k - 1) * (2 * k)) * p;
        return p;
    }
    /* sin(pi / 2 - x) to d^25, pi / 2 in two parts: d_hi + (d_lo - d_hi^3 / 6 p) */
    const double dh = 1.5707963267948966 - x, d2 = dh * dh;
    double p = 1.0;
    for (int k = 12; k >= 2; --k) p = 1.0 - d2 / (double)((2 * k) * (2 * k + 1)) * p;
    return dh + (6.123233995736766e-17 - dh * d2 / 6.0 * p);
}

/* the fixed order: out[c] = running sum over the 256 strided partials of vals[i * K + c] */
static void op_sum(int n, int K, const double* vals, double* out) {
    for (int c = 0; c < K; ++c) {
        double acc = 0.0;
        for (int t = 0; t < OP_SLOTS && t < n; ++t) {
            double s = 0.0;
            for (int i = t; i < n; i += OP_SLOTS) s += vals[(size_t)i * K + c];
            acc += s;
        }
        out[c] = acc;
    }
}

static void op_mat3_vec(const double* R, const double* v, double* o) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}

/* Horn: N from M = sum (a - a0)(b - b0)^T, the eigenvector of the largest eigenvalue (lowest index on ties), R from it */
static void op_horn_rotation(const double* M, double* R) {
    const double Sxx = M[0], Sxy = M[1], Sxz = M[2], Syx = M[3], Syy = M[4], Syz = M[5], Szx = M[6], Szy = M[7], Szz = M[8];
    const double N[16] = {Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx,
                          Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz,
                          Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy,
                          Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz};
    double ev[4], V[16];
    op_jacobi(4, N, ev, V);
    int m = 0;
    for (int k = 1; k < 4; ++k)
        if (ev[k] > ev[m]) m = k;
    const double w = V[m], x = V[4 + m], y = V[8 + m], z = V[12 + m];
    const double nq = w * w + x * x + y * y + z * z;
    R[0] = (w * w + x * x - y * y - z * z) / nq; R[1] = 2.0 * (x * y - w * z) / nq; R[2] = 2.0 * (x * z + w * y) / nq;
    R[3] = 2.0 * (x * y + w * z) / nq; R[4] = (w * w - x * x + y * y - z * z) / nq; R[5] = 2.0 * (y * z - w * x) / nq;
    R[6] = 2.0 * (x * z - w * y) / nq; R[7] = 2.0 * (y * z + w * x) / nq; R[8] = (w * w - x * x - y * y + z * z) / nq;
}

/* least squares by Householder QR, m x n (row-major), A and b overwritten */
static void op_lsq(double* A, double* b, int m, int n, double* x) {
    for (int k = 0; k < n; ++k) {
        double nrm2 = 0.0;
        for (int i = k; i < m; ++i) nrm2 += A[n * i + k] * A[n * i + k];
        const double nrm = sqrt(nrm2);
        const double alpha = A[n * k + k] > 0.0 ? -nrm : nrm;
        const double v0 = A[n * k + k] - alpha;
        double vtv = v0 * v0;
        for (int i = k + 1; i < m; ++i) vtv += A[n * i + k] * A[n * i + k];
        if (vtv > 0.0) {
            for (int j = k + 1; j < n; ++j) {
                double dot = v0 * A[n * k + j];
                for (int i = k + 1; i < m; ++i) dot += A[n * i + k] * A[n * i + j];
                const double f = 2.0 * dot / vtv;
                A[n * k + j] -= f * v0;
                for (int i = k + 1; i < m; ++i) A[n * i + j] -= f * A[n * i + k];
            }
            double dot = v0 * b[k];
            for (int i = k + 1; i < m; ++i) dot += A[n * i + k] * b[i];
            const double f = 2.0 * dot / vtv;
            b[k] -= f * v0;
            for (int i = k + 1; i < m; ++i) b[i] -= f * A[n * i + k];
        }
        A[n * k + k] = alpha;
    }
    for (int k = n - 1; k >= 0; --k) {
        double s = b[k];
        for (int j = k + 1; j < n; ++j) s -= A[n * k + j] * x[j];
        x[k] = s / A[n * k + k];
    }
}

void op_epnp(int n, const double* bear, const double* pw, double* pose) {
    const double dn = (double)n;
    double* vals = malloc(sizeof(double) * (size_t)n * 78);
    double* alphas = malloc(sizeof(double) * (size_t)n * 4);
    double* pcs = malloc(sizeof(double) * (size_t)n * 3);
    /* control points */
    double cws[4][3];
    for (int i = 0; i < n; ++i) memcpy(vals + 3 * (size_t)i, pw + 3 * (size_t)i, 3 * sizeof(double));
    op_sum(n, 3, vals, cws[0]);
    for (int k = 0; k < 3; ++k) cws[0][k] = cws[0][k] / dn;
    for (int i = 0; i < n; ++i) {
        const double* p = pw + 3 * (size_t)i;
        const double d0 = p[0] - cws[0][0], d1 = p[1] - cws[0][1], d2 = p[2] - cws[0][2];
        double* v = vals + 6 * (size_t)i;
        v[0] = d0 * d0; v[1] = d0 * d1; v[2] = d0 * d2; v[3] = d1 * d1; v[4] = d1 * d2; v[5] = d2 * d2;
    }
    double c6[6];
    op_sum(n, 6, vals, c6);
    const double C[9] = {c6[0], c6[1], c6[2], c6[1], c6[3], c6[4], c6[2], c6[4], c6[5]};
    double cev[3], CV[9];
    op_jacobi(3, C, cev, CV);
    for (int j = 0; j < 3; ++j) {
        double u[3];
        op_eigvec(3, cev, CV, 1, j, u);
        /* the eigenvalue of rank j, descending */
        double lam = 0.0;
        {
            int used[3] = {0, 0, 0}, col = 0;
            for (int r = 0; r <= j; ++r) {
                int m = -1;
                for (int k = 0; k < 3; ++k)
                    if (!used[k] && (m < 0 || cev[k] > cev[m])) m = k;
                used[m] = 1; col = m;
            }
            lam = cev[col];
        }
        const double kj = sqrt((lam > 0.0 ? lam : 0.0) / dn);
        for (int c = 0; c < 3; ++c) cws[j + 1][c] = cws[0][c] + kj * u[c];
    }
    /* barycentric coordinates through the adjugate inverse of CC */
    double cc[9], ci[9];
    for (int r = 0; r < 3; ++r)
        for (int j = 0; j < 3; ++j) cc[3 * r + j] = cws[j + 1][r] - cws[0][r];
    {
        const double c00 = cc[4] * cc[8] - cc[5] * cc[7], c01 = cc[5] * cc[6] - cc[3] * cc[8], c02 = cc[3] * cc[7] - cc[4] * cc[6];
        const double c10 = cc[2] * cc[7] - cc[1] * cc[8], c11 = cc[0] * cc[8] - cc[2] * cc[6], c12 = cc[1] * cc[6] - cc[0] * cc[7];
        const double c20 = cc[1] * cc[5] - cc[2] * cc[4], c21 = cc[2] * cc[3] - cc[0] * cc[5], c22 = cc[0] * cc[4] - cc[1] * cc[3];
        const double det = cc[0] * c00 + cc[1] * c01 + cc[2] * c02;
        const double adj[9] = {c00, c10, c20, c01, c11, c21, c02, c12, c22};
        for (int k = 0; k < 9; ++k) ci[k] = adj[k] / det;
    }
    for (int i = 0; i < n; ++i) {
        const double* p = pw + 3 * (size_t)i;
        double* a = alphas + 4 * (size_t)i;
        const double d[3] = {p[0] - cws[0][0], p[1] - cws[0][1], p[2] - cws[0][2]};
        for (int j = 0; j < 3; ++j) a[1 + j] = ci[3 * j] * d[0] + ci[3 * j + 1] * d[1] + ci[3 * j + 2] * d[2];
        a[0] = 1.0 - a[1] - a[2] - a[3];
    }
    /* M^T M, upper triangle per point */
    for (int i = 0; i < n; ++i) {
        const double* a = alphas + 4 * (size_t)i;
        const double* b = bear + 3 * (size_t)i;
        double r1[12], r2[12];
        for (int j = 0; j < 4; ++j) {
            r1[3 * j] = a[j] * b[2]; r1[3 * j + 1] = 0.0; r1[3 * j + 2] = -a[j] * b[0];
            r2[3 * j] = 0.0; r2[3 * j + 1] = a[j] * b[2]; r2[3 * j + 2] = -a[j] * b[1];
        }
        double* v = vals + 78 * (size_t)i;
        int q = 0;
        for (int r = 0; r < 12; ++r)
            for (int c = r; c < 12; ++c) v[q++] = r1[r] * r1[c] + r2[r] * r2[c];
    }
    double up[78], MtM[144];
    op_sum(n, 78, vals, up);
    {
        int q = 0;
        for (int r = 0; r < 12; ++r)
            for (int c = r; c < 12; ++c) { MtM[12 * r + c] = up[q]; MtM[12 * c + r] = up[q]; ++q; }
    }
    double mev[12], MV[144], vs[4][12];
    op_jacobi(12, MtM, mev, MV);
    for (int i = 0; i < 4; ++i) op_eigvec(12, mev, MV, 0, i, vs[i]);
    /* L_6x10 and rho (pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3)) */
    static const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
    double L[60], rho[6];
    for (int j = 0; j < 6; ++j) {
        double dv[4][3];
        for (int i = 0; i < 4; ++i)
            for (int c = 0; c < 3; ++c) dv[i][c] = vs[i][3 * pa[j] + c] - vs[i][3 * pb[j] + c];
        double d[4][4];
        for (int x = 0; x < 4; ++x)
            for (int y = 0; y < 4; ++y) d[x][y] = dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2];
        double* row = L + 10 * j;
        row[0] = d[0][0]; row[1] = 2.0 * d[0][1]; row[2] = d[1][1]; row[3] = 2.0 * d[0][2]; row[4] = 2.0 * d[1][2];
        row[5] = d[2][2]; row[6] = 2.0 * d[0][3]; row[7] = 2.0 * d[1][3]; row[8] = 2.0 * d[2][3]; row[9] = d[3][3];
        const double e0 = cws[pa[j]][0] - cws[pb[j]][0], e1 = cws[pa[j]][1] - cws[pb[j]][1], e2 = cws[pa[j]][2] - cws[pb[j]][2];
        rho[j] = e0 * e0 + e1 * e1 + e2 * e2;
    }
    static const int cols[3][5] = {{0, 1, 3, 6, -1}, {0, 1, 2, -1, -1}, {0, 1, 2, 3, 4}};
    double best_err = 0.0;
    for (int ap = 1; ap <= 3; ++ap) {
        const int nc = ap == 1 ? 4 : (ap == 2 ? 3 : 5);
        double A[30], rhs[6], x[5], betas[4];
        for (int j = 0; j < 6; ++j) {
            for (int c = 0; c < nc; ++c) A[nc * j + c] = L[10 * j + cols[ap - 1][c]];
            rhs[j] = rho[j];
        }
        op_lsq(A, rhs, 6, nc, x);
        if (ap == 1) {
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
            betas[2] = ap == 3 ? x[3] / betas[0] : 0.0;
            betas[3] = 0.0;
        }
        for (int it = 0; it < 5; ++it) {
            double G[24], r[6], dx[4];
            const double* bt = betas;
            for (int j = 0; j < 6; ++j) {
                const double* l = L + 10 * j;
                G[4 * j] = 2.0 * l[0] * bt[0] + l[1] * bt[1] + l[3] * bt[2] + l[6] * bt[3];
                G[4 * j + 1] = l[1] * bt[0] + 2.0 * l[2] * bt[1] + l[4] * bt[2] + l[7] * bt[3];
                G[4 * j + 2] = l[3] * bt[0] + l[4] * bt[1] + 2.0 * l[5] * bt[2] + l[8] * bt[3];
                G[4 * j + 3] = l[6] * bt[0] + l[7] * bt[1] + l[8] * bt[2] + 2.0 * l[9] * bt[3];
                r[j] = rho[j] - (l[0] * bt[0] * bt[0] + l[1] * bt[0] * bt[1] + l[2] * bt[1] * bt[1] + l[3] * bt[0] * bt[2] +
                                 l[4] * bt[1] * bt[2] + l[5] * bt[2] * bt[2] + l[6] * bt[0] * bt[3] + l[7] * bt[1] * bt[3] +
                                 l[8] * bt[2] * bt[3] + l[9] * bt[3] * bt[3]);
            }
            op_lsq(G, r, 6, 4, dx);
            for (int k = 0; k < 4; ++k) betas[k] += dx[k];
        }
        double ccs[12];
        for (int k = 0; k < 12; ++k) ccs[k] = 0.0;
        for (int i = 0; i < 4; ++i)
            for (int k = 0; k < 12; ++k) ccs[k] += betas[i] * vs[i][k];
        for (int pass = 0; pass < 2; ++pass) {   /* pass 1 only when the sign flips */
            for (int i = 0; i < n; ++i) {
                const double* a = alphas + 4 * (size_t)i;
                for (int c = 0; c < 3; ++c) pcs[3 * i + c] = a[0] * ccs[c] + a[1] * ccs[3 + c] + a[2] * ccs[6 + c] + a[3] * ccs[9 + c];
            }
            if (pass == 1 || !(pcs[0] * bear[0] + pcs[1] * bear[1] + pcs[2] * bear[2] < 0.0)) break;
            for (int k = 0; k < 12; ++k) ccs[k] = -ccs[k];
        }
        double pc0[3];
        op_sum(n, 3, pcs, pc0);
        for (int c = 0; c < 3; ++c) pc0[c] = pc0[c] / dn;
        for (int i = 0; i < n; ++i) {
            const double* p = pw + 3 * (size_t)i;
            const double dw[3] = {p[0] - cws[0][0], p[1] - cws[0][1], p[2] - cws[0][2]};
            const double dc[3] = {pcs[3 * i] - pc0[0], pcs[3 * i + 1] - pc0[1], pcs[3 * i + 2] - pc0[2]};
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) vals[9 * (size_t)i + 3 * r + c] = dw[r] * dc[c];
        }
        double Mo[9], cand[12], rc[3];
        op_sum(n, 9, vals, Mo);
        op_horn_rotation(Mo, cand);
        op_mat3_vec(cand, cws[0], rc);
        for (int c = 0; c < 3; ++c) cand[9 + c] = pc0[c] - rc[c];
        for (int i = 0; i < n; ++i) {
            const double* b = bear + 3 * (size_t)i;
            double q[3];
            op_mat3_vec(cand, pw + 3 * (size_t)i, q);
            for (int c = 0; c < 3; ++c) q[c] += cand[9 + c];
            vals[i] = 1.0 - (q[0] * b[0] + q[1] * b[1] + q[2] * b[2]) / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        }
        double err;
        op_sum(n, 1, vals, &err);
        err = err / dn;
        if (ap == 1 || err < best_err) {
            best_err = err;
            memcpy(pose, cand, sizeof(cand));
        }
    }
    free(vals); free(alphas); free(pcs);
}

/* check_inliers: (R p_w + t) . b / |R p_w + t| > max_cos, strictly */
static int op_check_inliers(int n, const double* bear, const double* pw, const double* max_cos, const double* pose, uint8_t* flags) {
    int count = 0;
    for (int i = 0; i < n; ++i) {
        double pc[3];
        op_mat3_vec(pose, pw + 3 * (size_t)i, pc);
        for (int k = 0; k < 3; ++k) pc[k] += pose[9 + k];
        const double* b = bear + 3 * (size_t)i;
        const double dot = pc[0] * b[0] + pc[1] * b[1] + pc[2] * b[2];
        const int in = dot / sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]) > max_cos[i];
        if (flags) flags[i] = (uint8_t)in;
        count += in;
    }
    return count;
}

void op_pnp_solve_ransac(int n, const double* bear, const double* pw, const float* scale_factor, int min_num_inliers,
                         int max_num_iter, int recompute, uint64_t seed, double* pose, int* valid, int* num_inliers, int* best_iter,
                         uint8_t* inlier_out, int* hyp_idx, double* hyp_pose, int* hyp_count) {
    for (int k = 0; k < 12; ++k) pose[k] = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
    *valid = 0; *num_inliers = 0; *best_iter = -1;
    for (int i = 0; i < n; ++i) inlier_out[i] = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        for (int j = 0; j < OP_MIN_SET; ++j) if (hyp_idx) hyp_idx[OP_MIN_SET * k + j] = -1;
        for (int j = 0; j < 12; ++j) if (hyp_pose) hyp_pose[12 * k + j] = 0.0;
        if (hyp_count) hyp_count[k] = 0;
    }
    if (n < OP_MIN_SET || n < min_num_inliers) return;
    double* max_cos = malloc(sizeof(double) * (size_t)n);
    for (int i = 0; i < n; ++i) max_cos[i] = op_max_cos(scale_factor[i]);
    int best = 0;
    for (int k = 0; k < max_num_iter; ++k) {
        int idx[OP_MIN_SET];
        op_ransac_sample(seed, k, n, OP_MIN_SET, idx);
        double b6[3 * OP_MIN_SET], p6[3 * OP_MIN_SET], P[12];
        for (int j = 0; j < OP_MIN_SET; ++j)
            for (int c = 0; c < 3; ++c) { b6[3 * j + c] = bear[3 * idx[j] + c]; p6[3 * j + c] = pw[3 * idx[j] + c]; }
        op_epnp(OP_MIN_SET, b6, p6, P);
        const int count = op_check_inliers(n, bear, pw, max_cos, P, NULL);
        if (hyp_idx) memcpy(hyp_idx + OP_MIN_SET * k, idx, sizeof(idx));
        if (hyp_pose) memcpy(hyp_pose + 12 * k, P, sizeof(P));
        if (hyp_count) hyp_count[k] = count;
        if (count > best) {
            best = count;
            *best_iter = k;
            memcpy(pose, P, sizeof(P));
            op_check_inliers(n, bear, pw, max_cos, P, inlier_out);
        }
    }
    *num_inliers = best;
    *valid = best >= min_num_inliers;
    if (*valid && recompute && *best_iter >= 0 && best >= OP_MIN_SET) {
        double* bi = malloc(sizeof(double) * 3 * (size_t)best);
        double* pi = malloc(sizeof(double) * 3 * (size_t)best);
        int m = 0;
        for (int i = 0; i < n; ++i)
            if (inlier_out[i]) {
                memcpy(bi + 3 * m, bear + 3 * (size_t)i, 3 * sizeof(double));
                memcpy(pi + 3 * m, pw + 3 * (size_t)i, 3 * sizeof(double));
                ++m;
            }
        op_epnp(m, bi, pi, pose);
        *num_inliers = op_check_inliers(n, bear, pw, max_cos, pose, inlier_out);
        free(bi); free(pi);
    }
    free(max_cos);
}
