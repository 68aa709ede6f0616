// two_view_triangulate.cu -- module::two_view_triangulator (local mapping) on the device: k_two_view_triangulate, one thread per
// keypoint pair, batched over keyframe pairs; the arithmetic is triangulation_math.cuh.  ovs_two_view_triangulate_host stages
// one keypoint record per pair end; ovs_create_new_landmarks_host (match_window.cu) runs the same kernel on the triangulation
// matcher's candidate lists.
#include <cmath>
#include <cstring>
#include <vector>

#include "match_common.h"
#include "ransac.cuh"
#include "two_view_triangulate.h"

namespace ovs {

namespace {

__global__ void __launch_bounds__(128) k_two_view_triangulate(TriLaunch A) {
    const int s = blockIdx.x * 128 + threadIdx.x;
    if (s >= A.n) return;
    int p, r1, r2;
    if (A.pairs) {
        const int3 q = A.pairs[s];
        p = q.x; r1 = q.y; r2 = q.z;
    } else {
        const unsigned key = A.keys[s];
        if (key == 0xffffffffu) {
            A.valid[s] = 0;
            for (int k = 0; k < 3; ++k) A.pos[3 * (size_t)s + k] = 0.0;
            return;
        }
        int q;
        if (A.fixed_prob >= 0) { p = A.fixed_prob; q = A.fixed_query; }
        else { const int qs = s / kTriListLen; p = qs / A.queries_per_prob; q = qs - p * A.queries_per_prob; }
        r1 = q;
        r2 = A.rec_2_base + A.rank_base[p] + (0xffff - (int)(key & 0xffffu));
    }
    const TriProblem& P = A.prob[p];
    double pos[3];
    int branch;
    const bool ok = tri_two_view(P.c[0], P.c[1], A.kp[r1], A.kp[r2], A.cos_thr, P.ratio_factor, pos, &branch) == kTriOk;
    A.valid[s] = ok ? 1 : 0;
    for (int k = 0; k < 3; ++k) A.pos[3 * (size_t)s + k] = ok ? pos[k] : 0.0;
}

__global__ void __launch_bounds__(128) k_gather_pos(int n, const int* __restrict__ slot, const double* __restrict__ pos, double* __restrict__ out) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < 3; ++k) out[3 * (size_t)i + k] = pos[3 * (size_t)slot[i] + k];
}

}  // namespace

int launch_two_view_triangulate(const TriLaunch& L, cudaStream_t st) {
    k_two_view_triangulate<<<(L.n + 127) / 128, 128, 0, st>>>(L);
    OVS_LAUNCH_CHECK();
    return OVS_OK;
}

int launch_gather_pos(int n, const int* slot, const double* pos, double* out, cudaStream_t st) {
    k_gather_pos<<<(n + 127) / 128, 128, 0, st>>>(n, slot, pos, out);
    OVS_LAUNCH_CHECK();
    return OVS_OK;
}

TriCam tri_cam(const ovs_keyframe_view& k) {
    TriCam c;
    for (int i = 0; i < 12; ++i) c.pose[i] = k.pose_cw[i];
    c.cam.model = k.camera.model; c.cam.fx = k.camera.fx; c.cam.fy = k.camera.fy; c.cam.cx = k.camera.cx; c.cam.cy = k.camera.cy;
    c.cam.fb = k.camera.focal_x_baseline; c.cam.cols = k.camera.cols; c.cam.rows = k.camera.rows;
    c.true_baseline = k.true_baseline;
    return c;
}

TriKeypt tri_keypt(const ovs_keyframe_view& k, int i) {
    TriKeypt r;
    for (int c = 0; c < 3; ++c) r.bearing[c] = k.bearings[3 * (size_t)i + c];
    r.x = k.undist_keypts[i].x; r.y = k.undist_keypts[i].y;
    r.x_right = k.stereo_x_right ? k.stereo_x_right[i] : -1.0f;
    r.depth = k.depths ? k.depths[i] : -1.0f;
    r.sigma_sq = k.level_sigma_sq[k.undist_keypts[i].octave];
    r.scale_factor = k.scale_factors[k.undist_keypts[i].octave];
    return r;
}

int check_keyframe_view(const ovs_keyframe_view* k, bool matching, const char* what, int b) {
    OVS_REQUIRE(k, OVS_ERR_INVALID_ARG, "null %s (%d)", what, b);
    for (int i = 0; i < 12; ++i) OVS_REQUIRE(std::isfinite(k->pose_cw[i]), OVS_ERR_INVALID_ARG, "pose of %s %d is not finite", what, b);
    const ovs_camera& c = k->camera;
    OVS_REQUIRE(c.model == OVS_CAMERA_PERSPECTIVE || c.model == OVS_CAMERA_EQUIRECTANGULAR, OVS_ERR_INVALID_ARG,
                "unknown camera model of %s %d", what, b);
    OVS_REQUIRE(k->num_keypts >= 0 && k->num_scale_levels >= 1, OVS_ERR_INVALID_ARG, "bad sizes of %s %d", what, b);
    OVS_REQUIRE(k->scale_factors && k->level_sigma_sq, OVS_ERR_INVALID_ARG, "null scale table of %s %d", what, b);
    for (int l = 0; l < k->num_scale_levels; ++l)
        OVS_REQUIRE(std::isfinite(k->scale_factors[l]) && k->scale_factors[l] > 0.0f && std::isfinite(k->level_sigma_sq[l]) &&
                    k->level_sigma_sq[l] > 0.0f, OVS_ERR_INVALID_ARG, "scale table of %s %d is not positive and finite", what, b);
    OVS_REQUIRE(std::isfinite(k->scale_factor) && k->scale_factor > 0.0f, OVS_ERR_INVALID_ARG, "scale_factor of %s %d", what, b);
    OVS_REQUIRE((k->stereo_x_right == nullptr) == (k->depths == nullptr), OVS_ERR_INVALID_ARG,
                "%s %d: stereo_x_right and depths come together", what, b);
    OVS_REQUIRE(k->num_keypts == 0 || (k->undist_keypts && k->bearings), OVS_ERR_INVALID_ARG, "null keypoint array of %s %d", what, b);
    if (matching)
        OVS_REQUIRE(k->num_keypts == 0 || (k->descriptors && k->has_landmark && k->bow_node), OVS_ERR_INVALID_ARG,
                    "null descriptor, landmark or node array of %s %d", what, b);
    return OVS_OK;
}

int check_tri_keypt(const ovs_keyframe_view& k, int i, const char* what, int b) {
    OVS_REQUIRE(i >= 0 && i < k.num_keypts, OVS_ERR_INVALID_ARG, "keypoint %d outside %s %d", i, what, b);
    const int o = k.undist_keypts[i].octave;
    OVS_REQUIRE(o >= 0 && o < k.num_scale_levels, OVS_ERR_INVALID_ARG, "octave %d of keypoint %d of %s %d outside the scale table", o, i,
                what, b);
    const double* v = k.bearings + 3 * (size_t)i;
    OVS_REQUIRE(std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]) && std::fabs(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] - 1.0) <= 1e-6,
                OVS_ERR_INVALID_ARG, "bearing of keypoint %d of %s %d is not a finite unit vector", i, what, b);
    OVS_REQUIRE(std::isfinite(k.undist_keypts[i].x) && std::isfinite(k.undist_keypts[i].y), OVS_ERR_INVALID_ARG,
                "keypoint %d of %s %d is not finite", i, what, b);
    if (k.stereo_x_right) {
        const float xr = k.stereo_x_right[i];
        OVS_REQUIRE(std::isfinite(xr), OVS_ERR_INVALID_ARG, "x_right of keypoint %d of %s %d is not finite", i, what, b);
        if (0.0f <= xr) {
            OVS_REQUIRE(k.camera.model == OVS_CAMERA_PERSPECTIVE, OVS_ERR_INVALID_ARG, "stereo keypoint %d on the equirectangular %s %d", i,
                        what, b);
            OVS_REQUIRE(std::isfinite(k.depths[i]), OVS_ERR_INVALID_ARG, "depth of stereo keypoint %d of %s %d is not finite", i, what, b);
        }
    }
    return OVS_OK;
}

int tri_cos_thr(double deg, double* cos_thr) {
    OVS_REQUIRE(std::isfinite(deg), OVS_ERR_INVALID_ARG, "rays_parallax_deg_thr must be finite");
    *cos_thr = std::cos(deg / 180.0 * M_PI);
    return OVS_OK;
}

}  // namespace ovs

extern "C" int ovs_two_view_triangulate_host(ovs_matcher* h, int B, const ovs_keyframe_view* keyfrms_1, const ovs_keyframe_view* keyfrms_2,
                                             const int32_t* pair_offsets, const int32_t* pairs, double rays_parallax_deg_thr, uint8_t* valid,
                                             double* pos_w) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    double cos_thr;
    int rc;
    if ((rc = ovs::tri_cos_thr(rays_parallax_deg_thr, &cos_thr)) != OVS_OK) return rc;
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(keyfrms_1 && keyfrms_2 && pair_offsets, OVS_ERR_INVALID_ARG, "null argument");
    if ((rc = ovs::check_offsets(pair_offsets, B, "pair_offsets")) != OVS_OK) return rc;
    const int M = pair_offsets[B];
    OVS_REQUIRE(M == 0 || (pairs && valid && pos_w), OVS_ERR_INVALID_ARG, "null argument");
    // two keypoint records per pair, indexed by int
    OVS_REQUIRE(M <= INT32_MAX / 2, OVS_ERR_UNSUPPORTED, "%d pairs: more than one call holds (2^30 - 1)", M);
    for (int b = 0; b < B; ++b) {
        if ((rc = ovs::check_keyframe_view(&keyfrms_1[b], false, "keyframe 1 of problem", b)) != OVS_OK) return rc;
        if ((rc = ovs::check_keyframe_view(&keyfrms_2[b], false, "keyframe 2 of problem", b)) != OVS_OK) return rc;
        for (int m = pair_offsets[b]; m < pair_offsets[b + 1]; ++m) {
            if ((rc = ovs::check_tri_keypt(keyfrms_1[b], pairs[2 * (size_t)m], "keyframe 1 of problem", b)) != OVS_OK) return rc;
            if ((rc = ovs::check_tri_keypt(keyfrms_2[b], pairs[2 * (size_t)m + 1], "keyframe 2 of problem", b)) != OVS_OK) return rc;
        }
    }
    if (M == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    const size_t NM = (size_t)M, NB = (size_t)B;
    ovs::TriLaunch L{};
    ovs::TriProblem* hprob; ovs::TriKeypt* hkp; int3* hpairs; uint8_t* hvalid; double* hpos;
    ovs::Staging S;
    rc = ovs::stage(S, h->h_tri, h->h_tri_cap, h->d_tri, h->d_tri_cap, [&](ovs::Staging& S) {
        L.prob = S.in(hprob, NB); L.kp = S.in(hkp, 2 * NM); L.pairs = S.in(hpairs, NM);
        L.valid = S.out(hvalid, NM); L.pos = S.out(hpos, 3 * NM);
    });
    if (rc != OVS_OK) return rc;
    for (int b = 0; b < B; ++b) {
        hprob[b].c[0] = ovs::tri_cam(keyfrms_1[b]); hprob[b].c[1] = ovs::tri_cam(keyfrms_2[b]);
        hprob[b].ratio_factor = 1.5f * keyfrms_1[b].scale_factor;
        for (int m = pair_offsets[b]; m < pair_offsets[b + 1]; ++m) {
            hkp[2 * (size_t)m] = ovs::tri_keypt(keyfrms_1[b], pairs[2 * (size_t)m]);
            hkp[2 * (size_t)m + 1] = ovs::tri_keypt(keyfrms_2[b], pairs[2 * (size_t)m + 1]);
            hpairs[m] = make_int3(b, 2 * m, 2 * m + 1);
        }
    }
    L.n = M; L.cos_thr = cos_thr; L.fixed_prob = -1;
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    if ((rc = ovs::launch_two_view_triangulate(L, st)) != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
    h->last_kernel_us = ms * 1000.f;
    memcpy(valid, hvalid, NM);
    memcpy(pos_w, hpos, 24 * NM);
    return OVS_OK;
}
