/*
 * oracle/match_oracle.c -- CPU restatement of OpenVSLAM's Hamming matchers.
 * TEST INFRASTRUCTURE ONLY (see orb_oracle.c).  PARITY STATUS: parity unpinned against the
 * real reference (no source under /root/reference; SURVEY.md section 0); the restatement
 * follows match/base.h and match/robust.cc as recalled in SURVEY.md 8(a) a8, a11.
 */
#include <math.h>
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "match_oracle.h"

/* match::compute_descriptor_distance_32 (match/base.h): 8 x 32-bit SWAR popcount. */
unsigned om_hamming(const uint8_t* a, const uint8_t* b) {
    const uint32_t* pa = (const uint32_t*)a;
    const uint32_t* pb = (const uint32_t*)b;
    unsigned dist = 0;
    for (int i = 0; i < 8; ++i, ++pa, ++pb) {
        uint32_t v = *pa ^ *pb;
        v = v - ((v >> 1) & 0x55555555u);
        v = (v & 0x33333333u) + ((v >> 2) & 0x33333333u);
        dist += (((v + (v >> 4)) & 0xF0F0F0Fu) * 0x1010101u) >> 24;
    }
    return dist;
}

/* The sequential nearest / second-nearest scan used by every matcher:
 *   if (d < best) { second = best; best = d; best_idx = i; } else if (d < second) second = d; */
void om_bruteforce(const uint8_t* desc1, int n1, const uint8_t* desc2, int n2,
                   int32_t* best_idx, int32_t* best_dist, int32_t* second_dist) {
    for (int q = 0; q < n1; ++q) {
        unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST;
        int bi = -1;
        for (int t = 0; t < n2; ++t) {
            const unsigned d = om_hamming(desc1 + (size_t)q * 32, desc2 + (size_t)t * 32);
            if (d < best) { second = best; best = d; bi = t; }
            else if (d < second) second = d;
        }
        best_idx[q] = bi; best_dist[q] = (int32_t)best; second_dist[q] = (int32_t)second;
    }
}

/* match::robust::brute_force_match (match/robust.cc). */
int om_robust_brute_force_match(const uint8_t* desc_frm, int n1, const uint8_t* desc_keyfrm, int n2,
                                const uint8_t* lm_valid_2, float lowe_ratio, int32_t* pairs_out) {
    uint8_t* already = (uint8_t*)calloc((size_t)n1 + 1, 1);
    int num = 0;
    for (int idx_2 = 0; idx_2 < n2; ++idx_2) {
        if (lm_valid_2 && !lm_valid_2[idx_2]) continue;
        const uint8_t* d2 = desc_keyfrm + (size_t)idx_2 * 32;
        unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST;
        int best_idx_1 = -1;
        for (int idx_1 = 0; idx_1 < n1; ++idx_1) {
            if (already[idx_1]) continue;
            const unsigned d = om_hamming(d2, desc_frm + (size_t)idx_1 * 32);
            if (d < best) { second = best; best = d; best_idx_1 = idx_1; }
            else if (d < second) second = d;
        }
        if (OM_HAMMING_DIST_THR_LOW < best) continue;
        if (lowe_ratio * second < (float)best) continue;
        pairs_out[2 * num] = best_idx_1; pairs_out[2 * num + 1] = idx_2;
        already[best_idx_1] = 1;
        ++num;
    }
    free(already);
    return num;
}

/* match::robust::check_epipolar_constraint (match/robust.cc, as recalled): angle between bearing_1 and the epipolar plane
 * E_12 * bearing_2, threshold 0.2 deg scaled by the scale factor of keypoint 1's octave. */
int om_check_epipolar_constraint(const double* bearing_1, const double* bearing_2, const double* E_12, float bearing_1_scale_factor) {
    double ep[3];
    for (int i = 0; i < 3; ++i) ep[i] = E_12[3 * i] * bearing_2[0] + E_12[3 * i + 1] * bearing_2[1] + E_12[3 * i + 2] * bearing_2[2];
    const double norm = sqrt(ep[0] * ep[0] + ep[1] * ep[1] + ep[2] * ep[2]);
    const double cos_residual = (ep[0] * bearing_1[0] + ep[1] * bearing_1[1] + ep[2] * bearing_1[2]) / norm;
    const double residual_rad = M_PI / 2.0 - fabs(acos(cos_residual));
    const double residual_rad_thr = 0.2 * M_PI / 180.0;
    return residual_rad < residual_rad_thr * (double)bearing_1_scale_factor;
}

/* match::robust::match_for_triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs) (match/robust.cc, as recalled).
 * The BoW feature vectors are inputs: bow_node_k[i] = vocabulary node of keypoint i (DBoW2 FeatureVector inverted; < 0 =
 * none).  Nodes are visited in ascending id, keypoints of a node in ascending index, exactly like iterating the two
 * std::map<NodeId, std::vector<unsigned>> in lock step.  Only keypoints without a landmark take part; a keyframe-2
 * keypoint is given to the first keyframe-1 keypoint that takes it; among equal distances the LAST candidate wins (the
 * loop skips only strictly larger distances).  epipole_in_2 = bearing of camera centre 1 seen from keyframe 2. */
int om_robust_match_for_triangulation(int n1, const uint8_t* desc_1, const double* bearing_1, const int* octave_1, const float* angle_1,
                                      const uint8_t* has_lm_1, const uint8_t* is_stereo_1, const int* bow_node_1,
                                      int n2, const uint8_t* desc_2, const double* bearing_2, const float* angle_2,
                                      const uint8_t* has_lm_2, const uint8_t* is_stereo_2, const int* bow_node_2,
                                      const double* E_12, const double* epipole_in_2, const float* scale_factors_1,
                                      int check_orientation, int* matched_idx_2_of_1) {
    int max_node = -1;
    for (int i = 0; i < n1; ++i) if (bow_node_1[i] > max_node) max_node = bow_node_1[i];
    for (int i = 0; i < n2; ++i) if (bow_node_2[i] > max_node) max_node = bow_node_2[i];
    uint8_t* taken_2 = (uint8_t*)calloc((size_t)n2 + 1, 1);
    float* deltas = (float*)malloc(sizeof(float) * (n1 + 1)); int* delta_idx = (int*)malloc(sizeof(int) * (n1 + 1)); int nd = 0;
    for (int i = 0; i < n1; ++i) matched_idx_2_of_1[i] = -1;
    int num_matches = 0;
    for (int node = 0; node <= max_node; ++node) {
        for (int idx_1 = 0; idx_1 < n1; ++idx_1) {
            if (bow_node_1[idx_1] != node) continue;
            if (has_lm_1[idx_1]) continue;
            const int stereo_1 = is_stereo_1 ? is_stereo_1[idx_1] : 0;
            unsigned best = OM_HAMMING_DIST_THR_LOW; int best_idx_2 = -1;
            for (int idx_2 = 0; idx_2 < n2; ++idx_2) {
                if (bow_node_2[idx_2] != node) continue;
                if (has_lm_2[idx_2]) continue;
                if (taken_2[idx_2]) continue;
                const int stereo_2 = is_stereo_2 ? is_stereo_2[idx_2] : 0;
                const unsigned d = om_hamming(desc_1 + 32 * (size_t)idx_1, desc_2 + 32 * (size_t)idx_2);
                if (OM_HAMMING_DIST_THR_LOW < d || best < d) continue;
                if (!stereo_1 && !stereo_2) {
                    const double* b2 = bearing_2 + 3 * (size_t)idx_2;
                    const double cos_dist = epipole_in_2[0] * b2[0] + epipole_in_2[1] * b2[1] + epipole_in_2[2] * b2[2];
                    if (0.998 < cos_dist) continue;      /* too close to the epipole */
                }
                if (om_check_epipolar_constraint(bearing_1 + 3 * (size_t)idx_1, bearing_2 + 3 * (size_t)idx_2, E_12, scale_factors_1[octave_1[idx_1]])) {
                    best_idx_2 = idx_2; best = d;
                }
            }
            if (best_idx_2 < 0) continue;
            taken_2[best_idx_2] = 1;
            matched_idx_2_of_1[idx_1] = best_idx_2;
            ++num_matches;
            if (check_orientation) { deltas[nd] = angle_1[idx_1] - angle_2[best_idx_2]; delta_idx[nd] = idx_1; ++nd; }
        }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k) if (invalid[k]) { matched_idx_2_of_1[delta_idx[k]] = -1; --num_matches; }
        free(invalid);
    }
    free(taken_2); free(deltas); free(delta_idx);
    return num_matches;
}

/* ---- match::bow_tree (match/bow_tree.cc, as recalled) -- SURVEY.md 8f rank 2, oracle only so far (no CUDA counterpart).
 * The BoW feature vectors are inputs (per-keypoint vocabulary node ids, < 0 = none); nodes ascending, keypoints of a node
 * in index order, as the lock-step walk over the two std::map<NodeId, std::vector<unsigned>>.
 *
 * match_frame_and_keyframe(keyfrm, frm, matched_lms_in_frm): every keyframe keypoint with a valid landmark looks for its
 * nearest and second nearest descriptor among the still unmatched frame keypoints of the same node; accepted when the
 * distance is <= HAMMING_DIST_THR_LOW and passes the ratio test; the frame keypoint is then taken.
 * matched_keyfrm_idx_of_frm[i] = keyframe keypoint whose landmark frame keypoint i received, or -1. */
int om_bow_tree_match_frame_and_keyframe(int n_kf, const uint8_t* desc_kf, const float* angle_kf, const uint8_t* lm_valid_kf, const int* bow_node_kf,
                                         int n_frm, const uint8_t* desc_frm, const float* angle_frm, const int* bow_node_frm,
                                         float lowe_ratio, int check_orientation, int* matched_keyfrm_idx_of_frm) {
    int max_node = -1;
    for (int i = 0; i < n_kf; ++i) if (bow_node_kf[i] > max_node) max_node = bow_node_kf[i];
    for (int i = 0; i < n_frm; ++i) if (bow_node_frm[i] > max_node) max_node = bow_node_frm[i];
    for (int i = 0; i < n_frm; ++i) matched_keyfrm_idx_of_frm[i] = -1;
    float* deltas = (float*)malloc(sizeof(float) * (n_kf + 1)); int* delta_idx = (int*)malloc(sizeof(int) * (n_kf + 1)); int nd = 0;
    int num_matches = 0;
    for (int node = 0; node <= max_node; ++node) {
        for (int k = 0; k < n_kf; ++k) {
            if (bow_node_kf[k] != node || !lm_valid_kf[k]) continue;
            unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST; int best_f = -1;
            for (int f = 0; f < n_frm; ++f) {
                if (bow_node_frm[f] != node) continue;
                if (matched_keyfrm_idx_of_frm[f] >= 0) continue;
                const unsigned d = om_hamming(desc_kf + 32 * (size_t)k, desc_frm + 32 * (size_t)f);
                if (d < best) { second = best; best = d; best_f = f; }
                else if (d < second) second = d;
            }
            if (OM_HAMMING_DIST_THR_LOW < best) continue;
            if (lowe_ratio * second < (float)best) continue;
            matched_keyfrm_idx_of_frm[best_f] = k;
            ++num_matches;
            if (check_orientation) { deltas[nd] = angle_kf[k] - angle_frm[best_f]; delta_idx[nd] = best_f; ++nd; }
        }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k) if (invalid[k]) { matched_keyfrm_idx_of_frm[delta_idx[k]] = -1; --num_matches; }
        free(invalid);
    }
    free(deltas); free(delta_idx);
    return num_matches;
}

/* match_keyframes(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_1): both keypoints need a valid landmark; a keyframe-2 keypoint
 * is matched at most once.  matched_idx_2_of_1[i1] = keypoint of keyframe 2 or -1. */
int om_bow_tree_match_keyframes(int n1, const uint8_t* desc_1, const float* angle_1, const uint8_t* lm_valid_1, const int* bow_node_1,
                                int n2, const uint8_t* desc_2, const float* angle_2, const uint8_t* lm_valid_2, const int* bow_node_2,
                                float lowe_ratio, int check_orientation, int* matched_idx_2_of_1) {
    int max_node = -1;
    for (int i = 0; i < n1; ++i) if (bow_node_1[i] > max_node) max_node = bow_node_1[i];
    for (int i = 0; i < n2; ++i) if (bow_node_2[i] > max_node) max_node = bow_node_2[i];
    for (int i = 0; i < n1; ++i) matched_idx_2_of_1[i] = -1;
    uint8_t* taken_2 = (uint8_t*)calloc((size_t)n2 + 1, 1);
    float* deltas = (float*)malloc(sizeof(float) * (n1 + 1)); int* delta_idx = (int*)malloc(sizeof(int) * (n1 + 1)); int nd = 0;
    int num_matches = 0;
    for (int node = 0; node <= max_node; ++node) {
        for (int i1 = 0; i1 < n1; ++i1) {
            if (bow_node_1[i1] != node || !lm_valid_1[i1]) continue;
            unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST; int best_2 = -1;
            for (int i2 = 0; i2 < n2; ++i2) {
                if (bow_node_2[i2] != node) continue;
                if (taken_2[i2]) continue;
                if (!lm_valid_2[i2]) continue;
                const unsigned d = om_hamming(desc_1 + 32 * (size_t)i1, desc_2 + 32 * (size_t)i2);
                if (d < best) { second = best; best = d; best_2 = i2; }
                else if (d < second) second = d;
            }
            if (OM_HAMMING_DIST_THR_LOW < best) continue;
            if (lowe_ratio * second < (float)best) continue;
            taken_2[best_2] = 1;
            matched_idx_2_of_1[i1] = best_2;
            ++num_matches;
            if (check_orientation) { deltas[nd] = angle_1[i1] - angle_2[best_2]; delta_idx[nd] = i1; ++nd; }
        }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k) if (invalid[k]) { matched_idx_2_of_1[delta_idx[k]] = -1; --num_matches; }
        free(invalid);
    }
    free(taken_2); free(deltas); free(delta_idx);
    return num_matches;
}

/* ========================================================================================== */
/* Windowed search.  Restates data::frame::get_keypoints_in_cell + data::assign_keypoints_to_grid
 * (data/frame.cc, data/common.cc), match::projection::match_frame_and_landmarks /
 * match_current_and_last_frames (match/projection.cc), match::area::match_in_consistent_area
 * (match/area.cc), match::angle_checker (match/angle_checker.h) and match::stereo (match/stereo.cc);
 * names as recalled in SURVEY.md 8a (a9, a10, a12).  Parity unpinned (no reference source). */

static int cv_floor(double v) { int i = (int)v; return i - (v < i); }
static int cv_ceil(double v) { int i = (int)v; return i + (v > i); }
static int cv_round_f(float v) { return (int)lrintf(v); }

/* data::get_cell_indices */
static int cell_of(const om_grid* g, float x, float y, int* cx, int* cy) {
    *cx = cv_floor((x - g->min_x) * g->inv_cell_width);
    *cy = cv_floor((y - g->min_y) * g->inv_cell_height);
    return 0 <= *cx && *cx < g->num_grid_cols && 0 <= *cy && *cy < g->num_grid_rows;
}

/* Literal restatement: the per-cell lists are rebuilt per call (slow but obviously right). */
int om_get_keypoints_in_cell_literal(const om_frame* f, float ref_x, float ref_y, float margin, int min_level, int max_level, int* out) {
    const om_grid* g = &f->grid;
    int n = 0;
    const int min_cx = cv_floor((ref_x - g->min_x - margin) * g->inv_cell_width) > 0 ? cv_floor((ref_x - g->min_x - margin) * g->inv_cell_width) : 0;
    if (g->num_grid_cols <= min_cx) return 0;
    int max_cx = cv_ceil((ref_x - g->min_x + margin) * g->inv_cell_width);
    if (max_cx > g->num_grid_cols - 1) max_cx = g->num_grid_cols - 1;
    if (max_cx < 0) return 0;
    const int min_cy = cv_floor((ref_y - g->min_y - margin) * g->inv_cell_height) > 0 ? cv_floor((ref_y - g->min_y - margin) * g->inv_cell_height) : 0;
    if (g->num_grid_rows <= min_cy) return 0;
    int max_cy = cv_ceil((ref_y - g->min_y + margin) * g->inv_cell_height);
    if (max_cy > g->num_grid_rows - 1) max_cy = g->num_grid_rows - 1;
    if (max_cy < 0) return 0;
    const int check_level = (0 < min_level) || (0 <= max_level);
    for (int cx = min_cx; cx <= max_cx; ++cx)
        for (int cy = min_cy; cy <= max_cy; ++cy)
            for (int idx = 0; idx < f->n; ++idx) { /* keypt_indices_in_cells_[cx][cy], ascending idx */
                int kx, ky;
                if (!cell_of(g, f->x[idx], f->y[idx], &kx, &ky) || kx != cx || ky != cy) continue;
                if (check_level) {
                    if (f->octave[idx] < min_level) continue;
                    if (0 <= max_level && max_level < f->octave[idx]) continue;
                }
                const float dist_x = f->x[idx] - ref_x, dist_y = f->y[idx] - ref_y;
                if (fabsf(dist_x) < margin && fabsf(dist_y) < margin) out[n++] = idx;
            }
    return n;
}

/* data::frame builds keypt_indices_in_cells_ once (assign_keypoints_to_grid) and every query walks those lists.  The same
 * here: a per-thread cache of the cell lists (CSR: cells in (cx, cy) order, keypoint indices ascending inside a cell), keyed
 * by the frame's arrays and a checksum of the coordinates, so that the CPU baseline pays what the reference pays.  The
 * literal version above stays as the checker of this one (tests/test_match_oracle.py). */
typedef struct {
    const float* x; const float* y; int n; om_grid grid; double checksum;
    int* cell_start; int* cell_idx; int cap_cells, cap_n;
} om_cell_cache;
static __thread om_cell_cache g_cache;

static const om_cell_cache* cell_lists(const om_frame* f) {
    om_cell_cache* c = &g_cache;
    const om_grid* g = &f->grid;
    double cs = 0;
    for (int i = 0; i < f->n; ++i) cs += (double)f->x[i] * 1.000001 + (double)f->y[i] * 0.999983 * (double)((i & 7) + 1);
    if (c->x == f->x && c->y == f->y && c->n == f->n && c->checksum == cs && memcmp(&c->grid, g, sizeof(om_grid)) == 0 && c->cell_start) return c;
    const int ncells = g->num_grid_cols * g->num_grid_rows;
    if (ncells + 1 > c->cap_cells) { free(c->cell_start); c->cell_start = (int*)malloc(sizeof(int) * (size_t)(ncells + 1)); c->cap_cells = ncells + 1; }
    if (f->n + 1 > c->cap_n) { free(c->cell_idx); c->cell_idx = (int*)malloc(sizeof(int) * (size_t)(f->n + 1)); c->cap_n = f->n + 1; }
    memset(c->cell_start, 0, sizeof(int) * (size_t)(ncells + 1));
    for (int i = 0; i < f->n; ++i) {
        int cx, cy;
        if (cell_of(g, f->x[i], f->y[i], &cx, &cy)) c->cell_start[cx * g->num_grid_rows + cy + 1]++;
    }
    for (int k = 0; k < ncells; ++k) c->cell_start[k + 1] += c->cell_start[k];
    int* pos = (int*)malloc(sizeof(int) * (size_t)(ncells + 1));
    memcpy(pos, c->cell_start, sizeof(int) * (size_t)(ncells + 1));
    for (int i = 0; i < f->n; ++i) {
        int cx, cy;
        if (cell_of(g, f->x[i], f->y[i], &cx, &cy)) c->cell_idx[pos[cx * g->num_grid_rows + cy]++] = i;
    }
    free(pos);
    c->x = f->x; c->y = f->y; c->n = f->n; c->grid = *g; c->checksum = cs;
    return c;
}

int om_get_keypoints_in_cell(const om_frame* f, float ref_x, float ref_y, float margin, int min_level, int max_level, int* out) {
    const om_grid* g = &f->grid;
    int n = 0;
    const int min_cx = cv_floor((ref_x - g->min_x - margin) * g->inv_cell_width) > 0 ? cv_floor((ref_x - g->min_x - margin) * g->inv_cell_width) : 0;
    if (g->num_grid_cols <= min_cx) return 0;
    int max_cx = cv_ceil((ref_x - g->min_x + margin) * g->inv_cell_width);
    if (max_cx > g->num_grid_cols - 1) max_cx = g->num_grid_cols - 1;
    if (max_cx < 0) return 0;
    const int min_cy = cv_floor((ref_y - g->min_y - margin) * g->inv_cell_height) > 0 ? cv_floor((ref_y - g->min_y - margin) * g->inv_cell_height) : 0;
    if (g->num_grid_rows <= min_cy) return 0;
    int max_cy = cv_ceil((ref_y - g->min_y + margin) * g->inv_cell_height);
    if (max_cy > g->num_grid_rows - 1) max_cy = g->num_grid_rows - 1;
    if (max_cy < 0) return 0;
    const om_cell_cache* c = cell_lists(f);
    const int check_level = (0 < min_level) || (0 <= max_level);
    for (int cx = min_cx; cx <= max_cx; ++cx)
        for (int cy = min_cy; cy <= max_cy; ++cy) {
            const int cell = cx * g->num_grid_rows + cy;
            for (int p = c->cell_start[cell]; p < c->cell_start[cell + 1]; ++p) { /* keypt_indices_in_cells_[cx][cy], ascending idx */
                const int idx = c->cell_idx[p];
                if (check_level) {
                    if (f->octave[idx] < min_level) continue;
                    if (0 <= max_level && max_level < f->octave[idx]) continue;
                }
                const float dist_x = f->x[idx] - ref_x, dist_y = f->y[idx] - ref_y;
                if (fabsf(dist_x) < margin && fabsf(dist_y) < margin) out[n++] = idx;
            }
        }
    return n;
}

/* match::angle_checker<int>: histogram of delta angles (bin = cvRound(delta / histogram_length)),
 * matches outside the `num_bins_to_retain` fullest bins are invalid; a runner-up bin is dropped when
 * it holds fewer than 10% of the fullest bin's matches. */
void om_angle_checker_invalid(const float* delta_angles, int n, int histogram_length, int num_bins_to_retain, uint8_t* invalid) {
    int* bin_of = (int*)malloc(sizeof(int) * (n + 1));
    int* count = (int*)calloc(histogram_length, sizeof(int));
    const float inv_len = 1.0f / histogram_length;
    for (int i = 0; i < n; ++i) {
        float d = delta_angles[i];
        if (d < 0.0) d += 360.0;
        if (360.0 <= d) d -= 360.0;
        const unsigned bin = (unsigned)cv_round_f(d * inv_len);
        bin_of[i] = (int)(bin % (unsigned)histogram_length);
        count[bin_of[i]]++;
    }
    /* indices of the bins sorted by size, descending (stable) */
    int* order = (int*)malloc(sizeof(int) * histogram_length);
    for (int b = 0; b < histogram_length; ++b) order[b] = b;
    for (int i = 1; i < histogram_length; ++i) {
        const int v = order[i]; int j = i - 1;
        while (j >= 0 && count[order[j]] < count[v]) { order[j + 1] = order[j]; --j; }
        order[j + 1] = v;
    }
    uint8_t* keep = (uint8_t*)calloc(histogram_length, 1);
    const int top = count[order[0]];
    for (int r = 0; r < num_bins_to_retain && r < histogram_length; ++r) {
        const int b = order[r];
        if (r > 0 && (float)count[b] < 0.1f * (float)top) break;
        keep[b] = 1;
    }
    for (int i = 0; i < n; ++i) invalid[i] = !keep[bin_of[i]];
    free(bin_of); free(count); free(order); free(keep);
}

int om_projection_match_frame_and_landmarks(const om_frame* frm, const float* scale_factors, int nlm, const uint8_t* lm_usable,
                                            const float* reproj_xy, const float* x_right_in_tracking, const int* pred_scale_level,
                                            const uint8_t* lm_desc, const uint8_t* kp_has_observed_lm, float margin, float lowe_ratio,
                                            int* matched_lm_of_kp) {
    int* cand = (int*)malloc(sizeof(int) * (frm->n + 1));
    uint8_t* has = (uint8_t*)malloc(frm->n + 1);
    for (int i = 0; i < frm->n; ++i) { has[i] = kp_has_observed_lm ? kp_has_observed_lm[i] : 0; matched_lm_of_kp[i] = -1; }
    int num_matches = 0;
    for (int l = 0; l < nlm; ++l) {
        if (lm_usable && !lm_usable[l]) continue;
        const int lvl = pred_scale_level[l];
        const int nc = om_get_keypoints_in_cell(frm, reproj_xy[2 * l], reproj_xy[2 * l + 1], margin * scale_factors[lvl], lvl - 1, lvl, cand);
        if (nc == 0) continue;
        unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST;
        int best_level = -1, second_level = -1, best_idx = -1;
        for (int c = 0; c < nc; ++c) {
            const int idx = cand[c];
            if (has[idx]) continue;
            if (frm->x_right && 0 < frm->x_right[idx]) {
                const float reproj_error = fabsf(x_right_in_tracking[l] - frm->x_right[idx]);
                if (margin * scale_factors[lvl] < reproj_error) continue;
            }
            const unsigned d = om_hamming(lm_desc + 32 * (size_t)l, frm->desc + 32 * (size_t)idx);
            if (d < best) { second = best; best = d; second_level = best_level; best_level = frm->octave[idx]; best_idx = idx; }
            else if (d < second) { second_level = frm->octave[idx]; second = d; }
        }
        if (best <= OM_HAMMING_DIST_THR_HIGH) {
            if (best_level == second_level && best > lowe_ratio * second) continue;
            matched_lm_of_kp[best_idx] = l;
            has[best_idx] = 1;   /* frm.landmarks_[best_idx] = local_lm (local landmarks have observations) */
            ++num_matches;
        }
    }
    free(cand); free(has);
    return num_matches;
}

int om_projection_match_current_and_last(const om_frame* curr, const float* scale_factors, int num_scale_levels, int n_last,
                                         const uint8_t* last_usable, const float* reproj_xy, const float* reproj_x_right,
                                         const int* last_scale_level, const float* last_angle, const uint8_t* lm_desc,
                                         const uint8_t* kp_has_observed_lm, float margin, int assume_forward, int assume_backward,
                                         int check_orientation, int* matched_last_of_kp) {
    int* cand = (int*)malloc(sizeof(int) * (curr->n + 1));
    uint8_t* has = (uint8_t*)malloc(curr->n + 1);
    float* deltas = (float*)malloc(sizeof(float) * (n_last + 1));
    int* delta_kp = (int*)malloc(sizeof(int) * (n_last + 1));
    int nd = 0;
    for (int i = 0; i < curr->n; ++i) { has[i] = kp_has_observed_lm ? kp_has_observed_lm[i] : 0; matched_last_of_kp[i] = -1; }
    int num_matches = 0;
    for (int i = 0; i < n_last; ++i) {
        if (!last_usable[i]) continue; /* no landmark, outlier, or reprojected outside the image */
        const int lvl = last_scale_level[i];
        const float m = margin * scale_factors[lvl];
        int nc;
        if (assume_forward) nc = om_get_keypoints_in_cell(curr, reproj_xy[2 * i], reproj_xy[2 * i + 1], m, lvl, num_scale_levels - 1, cand);
        else if (assume_backward) nc = om_get_keypoints_in_cell(curr, reproj_xy[2 * i], reproj_xy[2 * i + 1], m, 0, lvl, cand);
        else nc = om_get_keypoints_in_cell(curr, reproj_xy[2 * i], reproj_xy[2 * i + 1], m, lvl - 1, lvl + 1, cand);
        if (nc == 0) continue;
        unsigned best = OM_MAX_HAMMING_DIST; int best_idx = -1;
        for (int c = 0; c < nc; ++c) {
            const int idx = cand[c];
            if (has[idx]) continue;
            if (curr->x_right && curr->x_right[idx] > 0) {
                const float reproj_error = fabsf(reproj_x_right[i] - curr->x_right[idx]);
                if (m < reproj_error) continue;
            }
            const unsigned d = om_hamming(lm_desc + 32 * (size_t)i, curr->desc + 32 * (size_t)idx);
            if (d < best) { best = d; best_idx = idx; }
        }
        if (OM_HAMMING_DIST_THR_HIGH < best) continue;
        matched_last_of_kp[best_idx] = i;
        has[best_idx] = 1;
        ++num_matches;
        if (check_orientation) { deltas[nd] = last_angle[i] - curr->angle[best_idx]; delta_kp[nd] = best_idx; ++nd; }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k)
            if (invalid[k]) { matched_last_of_kp[delta_kp[k]] = -1; --num_matches; }
        free(invalid);
    }
    free(cand); free(has); free(deltas); free(delta_kp);
    return num_matches;
}

/* The search loop shared by the best-only projection matchers (see ovs_projection_match_best_host). */
int om_projection_match_best(const om_frame* f, int nq, const uint8_t* usable, const float* ref_xy, const float* ref_x_right,
                             const float* margin, const int* min_level, const int* max_level, const float* q_angle, const uint8_t* q_desc,
                             const uint8_t* kp_unavailable, unsigned hamm_dist_thr, int check_orientation, int* matched_query_of_kp) {
    int* cand = (int*)malloc(sizeof(int) * (f->n + 1));
    uint8_t* taken = (uint8_t*)malloc(f->n + 1);
    float* deltas = (float*)malloc(sizeof(float) * (nq + 1)); int* delta_kp = (int*)malloc(sizeof(int) * (nq + 1)); int nd = 0;
    for (int i = 0; i < f->n; ++i) { taken[i] = kp_unavailable ? kp_unavailable[i] : 0; matched_query_of_kp[i] = -1; }
    int num_matches = 0;
    for (int q = 0; q < nq; ++q) {
        if (usable && !usable[q]) continue;
        const int nc = om_get_keypoints_in_cell(f, ref_xy[2 * q], ref_xy[2 * q + 1], margin[q], min_level[q], max_level[q], cand);
        if (nc == 0) continue;
        unsigned best = OM_MAX_HAMMING_DIST; int best_idx = -1;
        for (int c = 0; c < nc; ++c) {
            const int idx = cand[c];
            if (taken[idx]) continue;
            if (ref_x_right && f->x_right && f->x_right[idx] > 0) {
                if (margin[q] < fabsf(ref_x_right[q] - f->x_right[idx])) continue;
            }
            const unsigned d = om_hamming(q_desc + 32 * (size_t)q, f->desc + 32 * (size_t)idx);
            if (d < best) { best = d; best_idx = idx; }
        }
        if (hamm_dist_thr < best) continue;
        matched_query_of_kp[best_idx] = q; taken[best_idx] = 1; ++num_matches;
        if (check_orientation) { deltas[nd] = q_angle[q] - f->angle[best_idx]; delta_kp[nd] = best_idx; ++nd; }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k) if (invalid[k]) { matched_query_of_kp[delta_kp[k]] = -1; --num_matches; }
        free(invalid);
    }
    free(cand); free(taken); free(deltas); free(delta_kp);
    return num_matches;
}

/* match::projection::match_keyframes_mutually (match/projection.cc, as recalled; ORB-SLAM2 SearchBySim3): each usable
 * landmark independently takes the nearest keypoint (first in visiting order on ties) of the other keyframe inside
 * its window, levels [pred - 1, pred], distance <= HAMMING_DIST_THR_HIGH; pairs are kept when both directions agree. */
static void om_best_in_window(const om_frame* dst, int nq, const uint8_t* usable, const float* reproj, const int* lvl, const uint8_t* desc,
                              const float* scale_factors, float margin, int* best_out) {
    int* cand = (int*)malloc(sizeof(int) * (dst->n + 1));
    for (int q = 0; q < nq; ++q) {
        best_out[q] = -1;
        if (usable && !usable[q]) continue;
        const int l = lvl[q];
        const int nc = om_get_keypoints_in_cell(dst, reproj[2 * q], reproj[2 * q + 1], margin * scale_factors[l < 0 ? 0 : l], l - 1, l, cand);
        unsigned best = OM_MAX_HAMMING_DIST; int best_idx = -1;
        for (int c = 0; c < nc; ++c) {
            const unsigned d = om_hamming(desc + 32 * (size_t)q, dst->desc + 32 * (size_t)cand[c]);
            if (d < best) { best = d; best_idx = cand[c]; }
        }
        if (best_idx >= 0 && best <= OM_HAMMING_DIST_THR_HIGH) best_out[q] = best_idx;
    }
    free(cand);
}

int om_projection_match_keyframes_mutually(const om_frame* f1, const om_frame* f2, const float* scale_factors, const uint8_t* usable_1,
                                           const float* reproj_1_in_2, const int* pred_level_1_in_2, const uint8_t* lm_desc_1,
                                           const uint8_t* usable_2, const float* reproj_2_in_1, const int* pred_level_2_in_1,
                                           const uint8_t* lm_desc_2, float margin, int* matched_idx_2_of_kp_1) {
    int* b21 = (int*)malloc(sizeof(int) * (f1->n + 1));
    int* b12 = (int*)malloc(sizeof(int) * (f2->n + 1));
    om_best_in_window(f2, f1->n, usable_1, reproj_1_in_2, pred_level_1_in_2, lm_desc_1, scale_factors, margin, b21);
    om_best_in_window(f1, f2->n, usable_2, reproj_2_in_1, pred_level_2_in_1, lm_desc_2, scale_factors, margin, b12);
    int num = 0;
    for (int i1 = 0; i1 < f1->n; ++i1) {
        matched_idx_2_of_kp_1[i1] = -1;
        const int i2 = b21[i1];
        if (i2 >= 0 && b12[i2] == i1) { matched_idx_2_of_kp_1[i1] = i2; ++num; }
    }
    free(b21); free(b12);
    return num;
}

int om_area_match_in_consistent_area(const om_frame* f1, const om_frame* f2, float* prev_matched_xy, int* matched_idx_2_in_1,
                                     int margin, float lowe_ratio, int check_orientation) {
    int num_matches = 0;
    int* cand = (int*)malloc(sizeof(int) * (f2->n + 1));
    unsigned* matched_dists_2 = (unsigned*)malloc(sizeof(unsigned) * (f2->n + 1));
    int* matched_idx_1_in_2 = (int*)malloc(sizeof(int) * (f2->n + 1));
    float* deltas = (float*)malloc(sizeof(float) * (f1->n + 1)); int* delta_idx = (int*)malloc(sizeof(int) * (f1->n + 1)); int nd = 0;
    for (int i = 0; i < f1->n; ++i) matched_idx_2_in_1[i] = -1;
    for (int i = 0; i < f2->n; ++i) { matched_dists_2[i] = OM_MAX_HAMMING_DIST; matched_idx_1_in_2[i] = -1; }
    for (int idx_1 = 0; idx_1 < f1->n; ++idx_1) {
        const int lvl = f1->octave[idx_1];
        if (0 < lvl) continue;
        const int nc = om_get_keypoints_in_cell(f2, prev_matched_xy[2 * idx_1], prev_matched_xy[2 * idx_1 + 1], (float)margin, lvl, lvl, cand);
        if (nc == 0) continue;
        unsigned best = OM_MAX_HAMMING_DIST, second = OM_MAX_HAMMING_DIST; int best_idx_2 = -1;
        for (int c = 0; c < nc; ++c) {
            const int idx_2 = cand[c];
            const unsigned d = om_hamming(f1->desc + 32 * (size_t)idx_1, f2->desc + 32 * (size_t)idx_2);
            if (matched_dists_2[idx_2] <= d) continue;
            if (d < best) { second = best; best = d; best_idx_2 = idx_2; }
            else if (d < second) second = d;
        }
        if (OM_HAMMING_DIST_THR_LOW < best) continue;
        if (second * lowe_ratio < (float)best) continue;
        const int prev_idx_1 = matched_idx_1_in_2[best_idx_2];
        if (0 <= prev_idx_1) { matched_idx_2_in_1[prev_idx_1] = -1; --num_matches; }
        matched_idx_2_in_1[idx_1] = best_idx_2;
        matched_idx_1_in_2[best_idx_2] = idx_1;
        matched_dists_2[best_idx_2] = best;
        ++num_matches;
        if (check_orientation) { deltas[nd] = f1->angle[idx_1] - f2->angle[best_idx_2]; delta_idx[nd] = idx_1; ++nd; }
    }
    if (check_orientation && nd > 0) {
        uint8_t* invalid = (uint8_t*)malloc(nd);
        om_angle_checker_invalid(deltas, nd, 30, 3, invalid);
        for (int k = 0; k < nd; ++k)
            if (invalid[k] && 0 <= matched_idx_2_in_1[delta_idx[k]]) { matched_idx_2_in_1[delta_idx[k]] = -1; --num_matches; }
        free(invalid);
    }
    for (int idx_1 = 0; idx_1 < f1->n; ++idx_1)
        if (0 <= matched_idx_2_in_1[idx_1]) {
            prev_matched_xy[2 * idx_1] = f2->x[matched_idx_2_in_1[idx_1]];
            prev_matched_xy[2 * idx_1 + 1] = f2->y[matched_idx_2_in_1[idx_1]];
        }
    free(cand); free(matched_dists_2); free(matched_idx_1_in_2); free(deltas); free(delta_idx);
    return num_matches;
}

/* match::stereo::compute */
/* cvRound for the SAD window origins, saturating like the kernel's __float2int_rn: a coordinate past the int range lands
 * outside every window instead of wrapping into one. */
static int round_sat(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.f) return INT_MAX;
    if (v < -2147483648.f) return INT_MIN;
    return (int)lrintf(v);
}

typedef struct { unsigned corr; int idx; } corr_idx;
static int corr_cmp(const void* a, const void* b) {
    const corr_idx* A = (const corr_idx*)a; const corr_idx* B = (const corr_idx*)b;
    if (A->corr != B->corr) return A->corr < B->corr ? -1 : 1;
    return A->idx < B->idx ? -1 : (A->idx > B->idx);
}

int om_stereo_compute(const uint8_t* const* left_pyr, const uint8_t* const* right_pyr, const int* pyr_w, const int* pyr_h, const int* pyr_stride,
                      int num_levels, const float* scale_factors, const float* inv_scale_factors,
                      int n_left, const float* lx, const float* ly, const int* loct, const uint8_t* ldesc,
                      int n_right, const float* rx, const float* ry, const int* roct, const uint8_t* rdesc,
                      float focal_x_baseline, float true_baseline, float* stereo_x_right, float* depths) {
    const float min_disp = 0.0f, max_disp = focal_x_baseline / true_baseline;
    const unsigned hamm_dist_thr = (OM_HAMMING_DIST_THR_HIGH + OM_HAMMING_DIST_THR_LOW) / 2;
    const int rows0 = pyr_h[0];
    corr_idx* corr = (corr_idx*)malloc(sizeof(corr_idx) * (n_left + 1));
    int ncorr = 0;
    for (int i = 0; i < n_left; ++i) { stereo_x_right[i] = -1.0f; depths[i] = -1.0f; }
    for (int il = 0; il < n_left; ++il) {
        const int lvl = loct[il];
        const float y_left = ly[il], x_left = lx[il];
        /* a keypoint with a coordinate that is not finite takes no part (the reference's conversions are undefined there) */
        if (!isfinite(x_left) || !isfinite(y_left)) continue;
        if (!(-1.0f < y_left && y_left < (float)rows0)) continue;
        const int row = (int)y_left;   /* indices_right_in_row.at(y_left) */
        const float min_x_right = x_left - max_disp, max_x_right = x_left - min_disp;
        if (max_x_right < 0) continue;
        unsigned best_dist = hamm_dist_thr; int best_ir = 0; int any = 0;
        for (int ir = 0; ir < n_right; ++ir) {
            if (!isfinite(rx[ir]) || !isfinite(ry[ir])) continue;
            /* get_right_keypoint_indices_in_each_row(2.0): rows [floor(y - r), ceil(y + r)] */
            const float r = 2.0f * scale_factors[roct[ir]];
            const int max_r = cv_ceil(ry[ir] + r), min_r = cv_floor(ry[ir] - r);
            if (row < min_r || row > max_r) continue;
            any = 1;
            if (roct[ir] < lvl - 1 || roct[ir] > lvl + 1) continue;
            if (rx[ir] < min_x_right || max_x_right < rx[ir]) continue;
            const unsigned d = om_hamming(ldesc + 32 * (size_t)il, rdesc + 32 * (size_t)ir);
            if (d < best_dist) { best_ir = ir; best_dist = d; }
        }
        if (!any) continue;
        if (hamm_dist_thr <= best_dist) continue;
        /* compute_subpixel_disparity */
        const float inv_s = inv_scale_factors[lvl];
        const int sxl = round_sat(x_left * inv_s), syl = round_sat(y_left * inv_s), sxr = round_sat(rx[best_ir] * inv_s);
        enum { win = 5, slide = 5 };
        const int W = pyr_w[lvl], Hh = pyr_h[lvl], S = pyr_stride[lvl];
        /* ini_x = sxr - slide - win < 0 || W <= end_x = sxr + slide + win + 1, and the left window, without overflow */
        if (sxr < slide + win || W - (slide + win + 1) <= sxr) continue;
        if (sxl < win || W - win <= sxl || syl < win || Hh - win <= syl) continue;
        const uint8_t* Limg = left_pyr[lvl]; const uint8_t* Rimg = right_pyr[lvl];
        const int cl = Limg[(size_t)syl * S + sxl];
        unsigned best_corr = UINT_MAX; int best_off = 0; float corrs[2 * slide + 1];
        for (int off = -slide; off <= slide; ++off) {
            const int cr = Rimg[(size_t)syl * S + sxr + off];
            unsigned sad = 0;
            for (int dy = -win; dy <= win; ++dy)
                for (int dx = -win; dx <= win; ++dx) {
                    const int a = Limg[(size_t)(syl + dy) * S + sxl + dx] - cl;
                    const int b = Rimg[(size_t)(syl + dy) * S + sxr + off + dx] - cr;
                    sad += (unsigned)abs(a - b);
                }
            if (sad < best_corr) { best_corr = sad; best_off = off; }
            corrs[slide + off] = (float)sad;
        }
        if (best_off == -slide || best_off == slide) continue;
        const float c1 = corrs[slide + best_off - 1], c2 = corrs[slide + best_off], c3 = corrs[slide + best_off + 1];
        const float delta = (float)((c1 - c3) / (2.0 * (c1 + c3 - 2.0 * c2)));
        if (delta < -1.0 || 1.0 < delta) continue;
        float best_x_right = scale_factors[lvl] * ((float)sxr + (float)best_off + delta);
        float disp = x_left - best_x_right;
        if (disp < min_disp || max_disp <= disp) continue;
        if (disp <= 0.0f) { disp = 0.01f; best_x_right = x_left - disp; }
        depths[il] = focal_x_baseline / disp;
        stereo_x_right[il] = best_x_right;
        corr[ncorr].corr = best_corr; corr[ncorr].idx = il; ++ncorr;
    }
    if (ncorr > 0) {
        qsort(corr, ncorr, sizeof(corr_idx), corr_cmp);
        const float median = (float)corr[ncorr / 2].corr;
        const float thr = 2.0f * median;
        for (int k = ncorr - 1; k >= 0; --k) {
            if ((float)corr[k].corr < thr) break;
            stereo_x_right[corr[k].idx] = -1; depths[corr[k].idx] = -1;
        }
    }
    free(corr);
    (void)num_levels; (void)ry;
    return ncorr;
}


/* ---- match::fuse (match/fuse.cc, as recalled; ORB-SLAM2 ORBmatcher::Fuse) -- SURVEY.md 8f rank 2, oracle only so far.
 * The matching core of fuse::replace_duplication / detect_duplication: each usable landmark (reprojected into the keyframe by
 * the caller, who also does the depth-range and viewing-angle tests and predict_scale_level) searches the window
 * margin * scale_factors[level] over the levels [level - 1, level]; a candidate keypoint is skipped when its reprojection
 * error exceeds the chi-square bound of its own octave (5.99 monocular, 7.8 stereo with the x_right term); the nearest
 * descriptor wins (first in visiting order on ties) and is accepted at <= HAMMING_DIST_THR_LOW.  No first-taker rule: what
 * happens to a keypoint that already has a landmark (replace / merge) is the caller's data-model decision.
 * best_idx_of_lm[q] = keypoint index or -1. */
int om_fuse_best_keypoints(const om_frame* f, int nq, const uint8_t* usable, const float* reproj_xy, const float* reproj_x_right,
                           const int* pred_level, const uint8_t* lm_desc, const float* scale_factors, const float* inv_level_sigma_sq,
                           float margin, int* best_idx_of_lm) {
    int* cand = (int*)malloc(sizeof(int) * (f->n + 1));
    int num = 0;
    for (int q = 0; q < nq; ++q) {
        best_idx_of_lm[q] = -1;
        if (usable && !usable[q]) continue;
        const int l = pred_level[q];
        const int nc = om_get_keypoints_in_cell(f, reproj_xy[2 * q], reproj_xy[2 * q + 1], margin * scale_factors[l < 0 ? 0 : l], l - 1, l, cand);
        unsigned best = OM_MAX_HAMMING_DIST; int best_idx = -1;
        for (int c = 0; c < nc; ++c) {
            const int idx = cand[c];
            const float ex = reproj_xy[2 * q] - f->x[idx], ey = reproj_xy[2 * q + 1] - f->y[idx];
            const float w = inv_level_sigma_sq[f->octave[idx]];
            if (f->x_right && f->x_right[idx] >= 0 && reproj_x_right) {
                const float er = reproj_x_right[q] - f->x_right[idx];
                if ((ex * ex + ey * ey + er * er) * w > 7.8f) continue;
            } else {
                if ((ex * ex + ey * ey) * w > 5.99f) continue;
            }
            const unsigned d = om_hamming(lm_desc + 32 * (size_t)q, f->desc + 32 * (size_t)idx);
            if (d < best) { best = d; best_idx = idx; }
        }
        if (best_idx >= 0 && best <= OM_HAMMING_DIST_THR_LOW) { best_idx_of_lm[q] = best_idx; ++num; }
    }
    free(cand);
    return num;
}
