// fuse.cu -- the compute of match::fuse::replace_duplication (match/fuse.cc) for many target keyframes in one call: the
// per-landmark geometry (fuse_observe, tracking_math.cuh) and the windowed search of the fuse matching core (window_walk.cuh, the
// walk k_window_topk runs), without the data-model updates, which the caller replays in the reference's order.
//
// k_fuse_geometry  one FP64 thread per query: reprojection into its target, the two gates, the predicted level.
// k_fuse_search    one warp per query that passed: the window margin * scale_factors[level] over the levels [level - 1, level] of
//                  its target's keypoints with the chi-square gate, nearest descriptor (first in visiting order on ties).
//
// Every target's cell index (data::assign_keypoints_to_grid, rank_keypoints of match_window.cu) is built on the host and staged with
// the queries and landmarks through one pinned arena and one device arena of the matcher: one copy up, one copy down, one wait.
#include <cmath>
#include <cstring>
#include <vector>

#include "match_common.h"
#include "tracking_math.cuh"
#include "window_walk.cuh"

namespace ovs {

namespace {

// one target as the kernels read it: its geometry, scale tables, grid and where its keypoints and cell starts are in the staged
// concatenation
struct FuseTarget {
    CameraD cam;
    ImgBounds b;
    double rot[9], trans[3], center[3];
    float log_scale_factor;
    int num_levels;
    float scale_factors[16], inv_sigma_sq[16];
    float grid_min_x, grid_min_y, inv_w, inv_h;
    int cols, rows;
    int kp_off, cell_off, has_xr;
};

struct FuseArgs {
    int nu;
    float margin;
    const FuseTarget* tgt;
    const int* q_tgt; const int* q_lm;
    const double* pos; const double* normal; const float* min_dist; const float* max_dist; const uint4* desc;
    const float* kx; const float* ky; const float* kxr; const signed char* koct; const uint4* kdesc; const int* cell;
    uint8_t* ok; float2* uv; float* xr; int* level; unsigned* key;
};

__global__ void __launch_bounds__(128) k_fuse_geometry(FuseArgs A) {
    const int k = blockIdx.x * 128 + threadIdx.x;
    if (k >= A.nu) return;
    const FuseTarget& T = A.tgt[A.q_tgt[k]];
    const size_t l = (size_t)A.q_lm[k];
    double p[3], nrm[3], uv[2] = {0.0, 0.0};
    for (int c = 0; c < 3; ++c) { p[c] = A.pos[3 * l + c]; nrm[c] = A.normal[3 * l + c]; }
    float xr = 0.0f;
    int level = 0;
    const bool ok = fuse_observe(T.cam, T.b, T.rot, T.trans, T.center, p, nrm, A.min_dist[l], A.max_dist[l], T.log_scale_factor, T.num_levels,
                                 uv, &xr, &level);
    A.ok[k] = ok ? 1 : 0;
    A.uv[k] = ok ? make_float2((float)uv[0], (float)uv[1]) : make_float2(0.0f, 0.0f);
    A.xr[k] = ok ? xr : 0.0f;
    A.level[k] = ok ? level : 0;
}

__global__ void __launch_bounds__(128) k_fuse_search(FuseArgs A) {
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (k >= A.nu) return;
    unsigned best = 0xffffffffu;
    if (A.ok[k]) {   // the same for the whole warp
        const FuseTarget& T = A.tgt[A.q_tgt[k]];
        WindowFrame F;
        F.min_x = T.grid_min_x; F.min_y = T.grid_min_y; F.inv_w = T.inv_w; F.inv_h = T.inv_h; F.cols = T.cols; F.rows = T.rows;
        F.x = A.kx + T.kp_off; F.y = A.ky + T.kp_off; F.xr = T.has_xr ? A.kxr + T.kp_off : nullptr; F.oct = A.koct + T.kp_off;
        F.desc = A.kdesc + 2 * (size_t)T.kp_off; F.cell_start = A.cell + T.cell_off; F.cap = nullptr;
        const int level = A.level[k];
        window_walk(F, A.uv[k], __fmul_rn(A.margin, T.scale_factors[level]), level - 1, level, true, [&] { return A.xr[k]; }, A.desc + 2 * (size_t)A.q_lm[k], true,
                    [&](int o) { return T.inv_sigma_sq[o & 15]; }, lane, [&](unsigned key) { best = min(best, key); });
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (lane == 0) A.key[k] = best;
}

int check_fuse_args(int B, const ovs_fuse_target* targets, int nlm, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                    const float* max_valid_dist, const uint8_t* lm_desc, const int32_t* q_off, const int32_t* q_lm, float margin,
                    const int32_t* best_idx, const int* num_fused) {
    OVS_REQUIRE(B >= 0 && nlm >= 0, OVS_ERR_INVALID_ARG, "B and nlm must be >= 0");
    OVS_REQUIRE(B <= OVS_FUSE_MAX_ITEMS && nlm <= OVS_FUSE_MAX_ITEMS, OVS_ERR_UNSUPPORTED, "more than %d targets or landmarks", OVS_FUSE_MAX_ITEMS);
    OVS_REQUIRE(q_off && num_fused && (B == 0 || targets), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(std::isfinite(margin) && margin > 0.0f, OVS_ERR_INVALID_ARG, "margin must be positive and finite");
    OVS_REQUIRE(q_off[0] == 0, OVS_ERR_INVALID_ARG, "q_off[0] must be 0");
    for (int t = 0; t < B; ++t) OVS_REQUIRE(q_off[t + 1] >= q_off[t], OVS_ERR_INVALID_ARG, "q_off decreases at target %d", t);
    const int Q = q_off[B];
    OVS_REQUIRE(Q <= OVS_FUSE_MAX_ITEMS, OVS_ERR_UNSUPPORTED, "more than %d queries", OVS_FUSE_MAX_ITEMS);
    OVS_REQUIRE(Q == 0 || (q_lm && best_idx), OVS_ERR_INVALID_ARG, "null query or output array");
    OVS_REQUIRE(nlm == 0 || (pos_w && mean_normal && min_valid_dist && max_valid_dist && lm_desc), OVS_ERR_INVALID_ARG, "null landmark array");
    long long kps = 0, cells = 0;
    for (int t = 0; t < B; ++t) {
        const ovs_fuse_target& T = targets[t];
        int rc;
        if ((rc = check_geometry(&T.geometry)) != OVS_OK) return rc;
        OVS_REQUIRE(T.num_keypts >= 0, OVS_ERR_INVALID_ARG, "target %d: num_keypts < 0", t);
        OVS_REQUIRE(T.num_keypts < 65536, OVS_ERR_UNSUPPORTED, "target %d: more than 65535 keypoints", t);
        OVS_REQUIRE(T.scale_factors && T.inv_level_sigma_sq, OVS_ERR_INVALID_ARG, "target %d: null scale table", t);
        OVS_REQUIRE(T.num_keypts == 0 || (T.x && T.y && T.octave && T.descriptors), OVS_ERR_INVALID_ARG, "target %d: null keypoint array", t);
        const ovs_grid& g = T.grid;
        OVS_REQUIRE(g.num_grid_cols > 0 && g.num_grid_rows > 0 && (long long)g.num_grid_cols * g.num_grid_rows <= 1 << 20, OVS_ERR_INVALID_ARG,
                    "target %d: bad grid", t);
        kps += T.num_keypts;
        cells += (long long)g.num_grid_cols * g.num_grid_rows + 1;
        OVS_REQUIRE(kps <= OVS_FUSE_MAX_ITEMS && cells <= OVS_FUSE_MAX_ITEMS, OVS_ERR_UNSUPPORTED, "more than %d keypoints or grid cells in all",
                    OVS_FUSE_MAX_ITEMS);
        const int L = T.geometry.num_scale_levels;
        for (int i = 0; i < T.num_keypts; ++i)
            OVS_REQUIRE(T.octave[i] >= 0 && T.octave[i] < L, OVS_ERR_INVALID_ARG, "target %d: octave %d of keypoint %d outside the scale table (%d levels)",
                        t, T.octave[i], i, L);
    }
    for (int q = 0; q < Q; ++q)
        OVS_REQUIRE(q_lm[q] >= -1 && q_lm[q] < nlm, OVS_ERR_INVALID_ARG, "q_lm[%d] = %d outside [-1, %d)", q, q_lm[q], nlm);
    return OVS_OK;
}

}  // namespace

}  // namespace ovs

extern "C" int ovs_fuse_replace_duplication_host(ovs_matcher* m, int B, const ovs_fuse_target* targets, int nlm, const double* pos_w,
                                                 const double* mean_normal, const float* min_valid_dist, const float* max_valid_dist,
                                                 const uint8_t* lm_desc, const int32_t* q_off, const int32_t* q_lm, float margin, int32_t* best_idx,
                                                 int* num_fused, uint8_t* passed, float* reproj_xy, float* x_right, int32_t* pred_level) {
    using namespace ovs;
    OVS_REQUIRE(m, OVS_ERR_INVALID_ARG, "null matcher");
    int rc = check_fuse_args(B, targets, nlm, pos_w, mean_normal, min_valid_dist, max_valid_dist, lm_desc, q_off, q_lm, margin, best_idx, num_fused);
    if (rc != OVS_OK) return rc;
    const int Q = q_off[B];
    *num_fused = 0;
    for (int q = 0; q < Q; ++q) best_idx[q] = -1;
    if (passed) memset(passed, 0, (size_t)Q);
    if (reproj_xy) memset(reproj_xy, 0, 8 * (size_t)Q);
    if (x_right) memset(x_right, 0, 4 * (size_t)Q);
    if (pred_level) memset(pred_level, 0, 4 * (size_t)Q);
    // the queries with a landmark, and the target of each
    std::vector<int> qi, qt;
    for (int t = 0; t < B; ++t)
        for (int q = q_off[t]; q < q_off[t + 1]; ++q)
            if (q_lm[q] >= 0) { qi.push_back(q); qt.push_back(t); }
    const int nu = (int)qi.size();
    if (nu == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    // every target's cell index, in the order get_keypoints_in_cell visits the keypoints
    std::vector<std::vector<int>> rank_to_idx(B), start(B);
    std::vector<int> nranked(B), kp_off(B + 1, 0), cell_off(B + 1, 0);
    std::vector<int> idx_to_rank;
    for (int t = 0; t < B; ++t) {
        const ovs_fuse_target& T = targets[t];
        start[t] = rank_keypoints(T.grid, T.num_keypts, T.x, T.y, rank_to_idx[t], idx_to_rank, &nranked[t]);
        kp_off[t + 1] = kp_off[t] + nranked[t];
        cell_off[t + 1] = cell_off[t] + (int)start[t].size();
    }
    const size_t N = (size_t)nu, L = (size_t)std::max(nlm, 1), K = (size_t)std::max(kp_off[B], 1);
    FuseArgs A{};
    A.nu = nu; A.margin = margin;
    FuseTarget* htgt; int *hqt, *hql; double *hpos, *hnrm; float *hlo, *hhi; uint4* hdesc;
    float *hkx, *hky, *hkxr; signed char* hkoct; uint4* hkdesc; int* hcell;
    uint8_t* hok; float2* huv; float* hxr; int* hlevel; unsigned* hkey;
    Staging S;
    rc = stage(S, m->h_fuse, m->h_fuse_cap, m->d_fuse, m->d_fuse_cap, [&](Staging& S) {
        A.tgt = S.in(htgt, (size_t)B); A.q_tgt = S.in(hqt, N); A.q_lm = S.in(hql, N);
        A.pos = S.in(hpos, 3 * L); A.normal = S.in(hnrm, 3 * L); A.min_dist = S.in(hlo, L); A.max_dist = S.in(hhi, L); A.desc = S.in(hdesc, 2 * L);
        A.kx = S.in(hkx, K); A.ky = S.in(hky, K); A.kxr = S.in(hkxr, K); A.koct = S.in(hkoct, K); A.kdesc = S.in(hkdesc, 2 * K);
        A.cell = S.in(hcell, (size_t)cell_off[B]);
        A.ok = S.out(hok, N); A.uv = S.out(huv, N); A.xr = S.out(hxr, N); A.level = S.out(hlevel, N); A.key = S.out(hkey, N);
    });
    if (rc != OVS_OK) return rc;
    for (int t = 0; t < B; ++t) {
        const ovs_fuse_target& T = targets[t];
        const ovs_frame_geometry& g = T.geometry;
        FuseTarget D{};
        D.cam.model = g.camera.model == OVS_CAMERA_EQUIRECTANGULAR ? kCamEquirectangular : kCamPerspective;
        D.cam.fx = g.camera.fx; D.cam.fy = g.camera.fy; D.cam.cx = g.camera.cx; D.cam.cy = g.camera.cy; D.cam.fb = g.camera.focal_x_baseline;
        D.cam.cols = g.camera.cols; D.cam.rows = g.camera.rows;
        D.b = ImgBounds{g.min_x, g.max_x, g.min_y, g.max_y};
        for (int k = 0; k < 9; ++k) D.rot[k] = g.rot_cw[k];
        for (int k = 0; k < 3; ++k) { D.trans[k] = g.trans_cw[k]; D.center[k] = g.cam_center[k]; }
        D.log_scale_factor = g.log_scale_factor; D.num_levels = g.num_scale_levels;
        for (int l = 0; l < g.num_scale_levels; ++l) { D.scale_factors[l] = T.scale_factors[l]; D.inv_sigma_sq[l] = T.inv_level_sigma_sq[l]; }
        D.grid_min_x = T.grid.min_x; D.grid_min_y = T.grid.min_y; D.inv_w = T.grid.inv_cell_width; D.inv_h = T.grid.inv_cell_height;
        D.cols = T.grid.num_grid_cols; D.rows = T.grid.num_grid_rows;
        D.kp_off = kp_off[t]; D.cell_off = cell_off[t]; D.has_xr = T.x_right != nullptr;
        htgt[t] = D;
        for (int r = 0; r < nranked[t]; ++r) {
            const int i = rank_to_idx[t][r], o = kp_off[t] + r;
            hkx[o] = T.x[i]; hky[o] = T.y[i]; hkxr[o] = T.x_right ? T.x_right[i] : -1.0f; hkoct[o] = (signed char)T.octave[i];
            memcpy(&hkdesc[2 * (size_t)o], T.descriptors + 32 * (size_t)i, 32);
        }
        memcpy(hcell + cell_off[t], start[t].data(), 4 * start[t].size());
    }
    for (int k = 0; k < nu; ++k) { hqt[k] = qt[k]; hql[k] = q_lm[qi[k]]; }
    if (nlm > 0) {
        memcpy(hpos, pos_w, 24 * (size_t)nlm); memcpy(hnrm, mean_normal, 24 * (size_t)nlm);
        memcpy(hlo, min_valid_dist, 4 * (size_t)nlm); memcpy(hhi, max_valid_dist, 4 * (size_t)nlm);
        memcpy(hdesc, lm_desc, 32 * (size_t)nlm);
    }
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_fuse_geometry<<<(nu + 127) / 128, 128, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    k_fuse_search<<<(nu + 3) / 4, 128, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    int num = 0;
    for (int k = 0; k < nu; ++k) {
        const int q = qi[k];
        const unsigned key = hkey[k];
        if (key != 0xffffffffu && (int)(key >> 16) <= OVS_HAMMING_DIST_THR_LOW) { best_idx[q] = rank_to_idx[qt[k]][key & 0xffffu]; ++num; }
        if (passed) passed[q] = hok[k];
        if (reproj_xy) { reproj_xy[2 * (size_t)q] = huv[k].x; reproj_xy[2 * (size_t)q + 1] = huv[k].y; }
        if (x_right) x_right[q] = hxr[k];
        if (pred_level) pred_level[q] = hlevel[k];
    }
    *num_fused = num;
    return OVS_OK;
}
