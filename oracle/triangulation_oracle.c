/* triangulation_oracle.c -- module::two_view_triangulator::triangulate (with solve::triangulator::triangulate and
 * keyframe::triangulate_stereo) and the compute step of mapping_module::create_new_landmarks, as recalled (DESIGN.md section 5).
 * The two-camera solve takes the eigenvector of A^T A's smallest eigenvalue from the oracle's cyclic Jacobi (op_jacobi). */
#include "triangulation_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "match_oracle.h"
#include "pnp_solver_oracle.h"
#include "sim3_solver_oracle.h"

#define OTR_PI 3.14159265358979323846

static int otr_is_stereo(const otr_keyframe* k, int i) { return k->stereo_x_right && 0.0f <= k->stereo_x_right[i]; }

/* R^T v (rot_wc = rot_cw^T) */
static void otr_rot_t(const double* pose, const double* v, double* o) {
    for (int r = 0; r < 3; ++r) o[r] = pose[r] * v[0] + pose[3 + r] * v[1] + pose[6 + r] * v[2];
}

/* cam_center = -rot_wc trans_cw */
static void otr_center(const double* pose, double* c) {
    double rt[3];
    otr_rot_t(pose, pose + 9, rt);
    for (int r = 0; r < 3; ++r) c[r] = -rt[r];
}

static double otr_cos_stereo(const otr_keyframe* k, int i) {
    if (!otr_is_stereo(k, i)) return 2.0;
    /* cos(2 atan2(h, d)) in closed form: cos 2a = (1 - tan^2 a) / (1 + tan^2 a), tan a = h / d */
    const double h = k->true_baseline / 2.0, d = (double)k->depths[i];
    return (d * d - h * h) / (d * d + h * h);
}

static void otr_solve_two(const double* b1, const double* b2, const double* P1, const double* P2, double* pos) {
    double A[4][4], M[16], ev[4], V[16];
    for (int c = 0; c < 4; ++c) {
        /* the 3 x 4 [R | t]: element (r, c) */
        const double p1[3] = {c < 3 ? P1[c] : P1[9], c < 3 ? P1[3 + c] : P1[10], c < 3 ? P1[6 + c] : P1[11]};
        const double p2[3] = {c < 3 ? P2[c] : P2[9], c < 3 ? P2[3 + c] : P2[10], c < 3 ? P2[6 + c] : P2[11]};
        A[0][c] = b1[0] * p1[2] - b1[2] * p1[0];
        A[1][c] = b1[1] * p1[2] - b1[2] * p1[1];
        A[2][c] = b2[0] * p2[2] - b2[2] * p2[0];
        A[3][c] = b2[1] * p2[2] - b2[2] * p2[1];
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = A[0][i] * A[0][j];
            for (int r = 1; r < 4; ++r) s += A[r][i] * A[r][j];
            M[4 * i + j] = s;
        }
    op_jacobi(4, M, ev, V);
    int col = 0;
    for (int k = 1; k < 4; ++k) if (ev[k] < ev[col]) col = k;
    int a = 0;
    for (int r = 1; r < 4; ++r) if (fabs(V[4 * r + col]) > fabs(V[4 * a + col])) a = r;
    const double sg = V[4 * a + col] < 0.0 ? -1.0 : 1.0;
    double v[4];
    for (int r = 0; r < 4; ++r) v[r] = sg * V[4 * r + col];
    for (int r = 0; r < 3; ++r) pos[r] = v[r] / v[3];
}

static void otr_stereo(const otr_keyframe* k, int i, double* pos) {
    const float depth = k->depths[i];
    if (!(0.0 < depth)) { pos[0] = pos[1] = pos[2] = 0.0; return; }
    const double fx_inv = 1.0 / k->camera.fx, fy_inv = 1.0 / k->camera.fy;
    const float ux = (float)(((double)k->undist_keypts[i].x - k->camera.cx) * (double)depth * fx_inv);
    const float uy = (float)(((double)k->undist_keypts[i].y - k->camera.cy) * (double)depth * fy_inv);
    const double pc[3] = {ux, uy, depth};
    double rp[3], c[3];
    otr_rot_t(k->pose_cw, pc, rp);
    otr_center(k->pose_cw, c);
    for (int r = 0; r < 3; ++r) pos[r] = rp[r] + c[r];
}

static int otr_depth_ok(const otr_keyframe* k, const double* p) {
    if (k->camera.model == 1) return 1;
    const double* R = k->pose_cw;
    const float z = (float)(R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + R[11]);
    return 0.0f < z;
}

static int otr_reproj_ok(const otr_keyframe* k, int i, const double* p) {
    const float chi_sq_2D = 5.99146f, chi_sq_3D = 7.81473f;
    double uv[2];
    os_reproject(&k->camera, k->pose_cw, k->pose_cw + 9, p, uv);
    const float sigma_sq = k->level_sigma_sq[k->undist_keypts[i].octave];
    const double ex = uv[0] - k->undist_keypts[i].x, ey = uv[1] - k->undist_keypts[i].y;
    if (otr_is_stereo(k, i)) {
        const double* R = k->pose_cw;
        const double z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + R[11];
        const float x_right = (float)(uv[0] - k->camera.focal_x_baseline * (1.0 / z));
        const float exr = x_right - k->stereo_x_right[i];
        return !(chi_sq_3D * sigma_sq < ex * ex + ey * ey + exr * exr);
    }
    return !(chi_sq_2D * sigma_sq < ex * ex + ey * ey);
}

static double otr_dist(const double* p, const double* c) {
    const double d[3] = {p[0] - c[0], p[1] - c[1], p[2] - c[2]};
    return sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
}

int otr_triangulate(const otr_keyframe* k1, const otr_keyframe* k2, int idx_1, int idx_2, double cos_thr, double* pos_w, int* branch) {
    const int st1 = otr_is_stereo(k1, idx_1), st2 = otr_is_stereo(k2, idx_2);
    const double* b1 = k1->bearings + 3 * (size_t)idx_1;
    const double* b2 = k2->bearings + 3 * (size_t)idx_2;
    double r1[3], r2[3];
    otr_rot_t(k1->pose_cw, b1, r1);
    otr_rot_t(k2->pose_cw, b2, r2);
    const double cos_rays = (r1[0] * r2[0] + r1[1] * r2[1] + r1[2] * r2[2]) /
                            (sqrt(r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2]) * sqrt(r2[0] * r2[0] + r2[1] * r2[1] + r2[2] * r2[2]));
    const double cs1 = otr_cos_stereo(k1, idx_1), cs2 = otr_cos_stereo(k2, idx_2);
    const double cs = fmin(cs1, cs2);
    if ((!st1 && !st2 && 0.0 < cos_rays && cos_rays < cos_thr) || ((st1 || st2) && 0.0 < cos_rays && cos_rays < cs)) {
        *branch = 0;
        otr_solve_two(b1, b2, k1->pose_cw, k2->pose_cw, pos_w);
        if (!isfinite(pos_w[0]) || !isfinite(pos_w[1]) || !isfinite(pos_w[2])) return 2;
    } else if (st1 && cs1 < cs2) {
        *branch = 1;
        otr_stereo(k1, idx_1, pos_w);
    } else if (st2 && cs2 < cs1) {
        *branch = 2;
        otr_stereo(k2, idx_2, pos_w);
    } else {
        *branch = -1;
        return 1;
    }
    if (!otr_depth_ok(k1, pos_w)) return 3;
    if (!otr_depth_ok(k2, pos_w)) return 4;
    if (!otr_reproj_ok(k1, idx_1, pos_w)) return 5;
    if (!otr_reproj_ok(k2, idx_2, pos_w)) return 6;
    double c1[3], c2[3];
    otr_center(k1->pose_cw, c1);
    otr_center(k2->pose_cw, c2);
    const double d1 = otr_dist(pos_w, c1), d2 = otr_dist(pos_w, c2);
    if (d1 == 0 || d2 == 0) return 7;
    const float ratio_factor = 1.5f * k1->scale_factor;
    const double ratio_dists = d2 / d1;
    const float ratio_octave = k1->scale_factors[k1->undist_keypts[idx_1].octave] / k2->scale_factors[k2->undist_keypts[idx_2].octave];
    if (ratio_dists * ratio_factor < ratio_octave || ratio_octave * ratio_factor < ratio_dists) return 7;
    return 0;
}

void otr_two_view_triangulate(const otr_keyframe* k1, const otr_keyframe* k2, int m, const int* pairs, double deg_thr, uint8_t* valid,
                              double* pos_w, int* reason, int* branch) {
    const double cos_thr = cos(deg_thr / 180.0 * M_PI);
    for (int i = 0; i < m; ++i) {
        double p[3];
        reason[i] = otr_triangulate(k1, k2, pairs[2 * i], pairs[2 * i + 1], cos_thr, p, &branch[i]);
        valid[i] = reason[i] == 0;
        for (int c = 0; c < 3; ++c) pos_w[3 * i + c] = valid[i] ? p[c] : 0.0;
    }
}

int otr_create_new_landmarks(const otr_keyframe* k1, int B, const otr_keyframe* k2, const double* E_12, const double* epipole_in_2,
                             int check_orientation, double deg_thr, int* rec, double* pos) {
    const int n1 = k1->num_keypts;
    const double cos_thr = cos(deg_thr / 180.0 * M_PI);
    uint8_t* has_lm = (uint8_t*)malloc((size_t)n1 + 1);
    uint8_t* st1 = (uint8_t*)malloc((size_t)n1 + 1);
    int* oct1 = (int*)malloc(sizeof(int) * ((size_t)n1 + 1));
    float* ang1 = (float*)malloc(sizeof(float) * ((size_t)n1 + 1));
    int* matched = (int*)malloc(sizeof(int) * ((size_t)n1 + 1));
    memcpy(has_lm, k1->has_landmark, (size_t)n1);
    for (int i = 0; i < n1; ++i) { st1[i] = otr_is_stereo(k1, i); oct1[i] = k1->undist_keypts[i].octave; ang1[i] = k1->undist_keypts[i].angle; }
    int num = 0;
    for (int b = 0; b < B; ++b) {
        const otr_keyframe* n = &k2[b];
        const int n2 = n->num_keypts;
        uint8_t* st2 = (uint8_t*)malloc((size_t)n2 + 1);
        float* ang2 = (float*)malloc(sizeof(float) * ((size_t)n2 + 1));
        for (int i = 0; i < n2; ++i) { st2[i] = otr_is_stereo(n, i); ang2[i] = n->undist_keypts[i].angle; }
        om_robust_match_for_triangulation(n1, k1->descriptors, k1->bearings, oct1, ang1, has_lm, st1, k1->bow_node, n2, n->descriptors, n->bearings,
                                          ang2, n->has_landmark, st2, n->bow_node, E_12 + 9 * b, epipole_in_2 + 3 * b, k1->scale_factors,
                                          check_orientation, matched);
        for (int i = 0; i < n1; ++i) {
            if (matched[i] < 0) continue;
            double p[3];
            int br;
            if (otr_triangulate(k1, n, i, matched[i], cos_thr, p, &br) != 0) continue;
            rec[3 * num] = b; rec[3 * num + 1] = i; rec[3 * num + 2] = matched[i];
            for (int c = 0; c < 3; ++c) pos[3 * num + c] = p[c];
            has_lm[i] = 1;
            ++num;
        }
        free(st2); free(ang2);
    }
    free(has_lm); free(st1); free(oct1); free(ang1); free(matched);
    return num;
}
