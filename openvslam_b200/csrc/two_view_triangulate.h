// two_view_triangulate.h -- the batched two-view triangulation kernel (two_view_triangulate.cu), shared by
// ovs_two_view_triangulate_host and ovs_create_new_landmarks_host (match_window.cu), and the host-side checks of a keyframe view.
#pragma once
#include "ovs_common.h"
#include "triangulation_math.cuh"

namespace ovs {

// The candidate lists of the triangulation matcher: kTriListLen keys per query, key = distance << 16 | (0xffff - rank).
constexpr int kTriListLen = 8;

// One keyframe pair: keyframe 1 and keyframe 2, and 1.5f * keyfrm_1 scale_factor_.
struct TriProblem {
    TriCam c[2];
    float ratio_factor;
};

// n slots, each one keypoint pair of problem p with keypoint records r1 (keyframe 1) and r2 (keyframe 2), given either
//  - explicitly: pairs[s] = {p, r1, r2}, or
//  - by the triangulation matcher's key in keys[s] (0xffffffff: no candidate, invalid): the slot belongs to query
//    q = (s / kTriListLen) % queries_per_prob of problem p = s / (kTriListLen * queries_per_prob), or to (fixed_prob, fixed_query)
//    when fixed_prob >= 0; r1 = q, r2 = rec_2_base + rank_base[p] + rank.
// valid[s] = 1 where the pair makes a landmark; pos[3 s] = its pos_w, zero where it does not.
struct TriLaunch {
    int n;
    double cos_thr;
    const TriProblem* prob;
    const TriKeypt* kp;
    const int3* pairs;
    const unsigned* keys;
    int queries_per_prob, fixed_prob, fixed_query, rec_2_base;
    const int* rank_base;
    uint8_t* valid;
    double* pos;
};

int launch_two_view_triangulate(const TriLaunch& L, cudaStream_t st);
// out[3 i] = pos[3 slot[i]], i < n
int launch_gather_pos(int n, const int* slot, const double* pos, double* out, cudaStream_t st);

// Host side: what a keyframe view contributes, after check_keyframe_view / check_tri_keypt accepted it.
TriCam tri_cam(const ovs_keyframe_view& k);
TriKeypt tri_keypt(const ovs_keyframe_view& k, int i);
// the keyframe's own fields (pose, camera, scale tables, null arrays); matching: descriptors, has_landmark and bow_node too
int check_keyframe_view(const ovs_keyframe_view* k, bool matching, const char* what, int b);
// keypoint i: octave inside the scale table, finite unit bearing, finite x_right and, for a stereo keypoint, finite depth
int check_tri_keypt(const ovs_keyframe_view& k, int i, const char* what, int b);
// cos(rays_parallax_deg_thr / 180 * pi), as the reference's constructor computes it
int tri_cos_thr(double rays_parallax_deg_thr, double* cos_thr);

}  // namespace ovs
