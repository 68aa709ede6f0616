// match_window.cu -- grid-windowed Hamming search for openvslam::match::{projection, area} and the
// rectified-row search + SAD sub-pixel refinement of openvslam::match::stereo
// (match/projection.cc, match/area.cc, match/stereo.cc, data/frame.cc get_keypoints_in_cell,
// data/common.cc assign_keypoints_to_grid; names as in SURVEY.md 8a a9, a10, a12).
//
// Frame index (ovs_frame_index): the frame's keypoints re-ordered by (cell_x, cell_y, index) -- the
// order get_keypoints_in_cell visits them -- with a CSR of cell starts, resident on the device.
//
// k_window_topk     one warp per query (landmark / keypoint): the cell range and the box, level,
//                   x_right and per-keypoint distance-cap tests exactly as the reference, 256-bit
//                   Hamming by __popc, per-lane sorted top-4 of (distance << 16 | rank), merged
//                   across the warp with __reduce_min_sync.  Rank order == candidate order, so the
//                   sorted keys reproduce the reference's first-wins tie-breaking.
// k_stereo_match    one thread per left keypoint, right keypoints staged through shared memory:
//                   row band / octave / disparity tests + Hamming -> best right keypoint.
// k_stereo_subpixel one warp per left keypoint: 11 SAD windows (11 x 11, centre-normalised) on the
//                   extractor's device pyramids, warp-reduced with __reduce_add_sync, parabola fit.
//
// The sequential parts of the reference (greedy "a keypoint is matched once" bookkeeping and the angle histogram,
// greedy_replay.h; the median test of stereo) run on the host over these results.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <new>
#include <vector>

#include "greedy_replay.h"
#include "match_common.h"
#include "two_view_triangulate.h"
#include "window_walk.cuh"

// ------------------------------------------------------------------------------- frame index
struct ovs_frame_index {
    ovs_matcher* m = nullptr;
    int n = 0, nranked = 0;
    ovs_grid grid{};
    std::vector<int> rank_to_idx, idx_to_rank;   // host
    std::vector<float> hx, hy, hxr, hangle; std::vector<int> hoct;
    // device, rank order
    float* d_x = nullptr; float* d_y = nullptr; float* d_xr = nullptr; signed char* d_oct = nullptr;
    uint4* d_desc = nullptr; int* d_cell_start = nullptr; unsigned short* d_cap = nullptr; int* d_rank = nullptr;
    ovs_index_buf buf;          // all of the above are carved from this one allocation (recycled through the matcher's pool)
    bool has_xr = false;
};

ovs_matcher* ovs::frame_index_matcher(const ovs_frame_index* f) { return f->m; }

namespace {

constexpr int kTopK = 4;

__device__ __forceinline__ void topk_insert(unsigned (&k)[kTopK], unsigned key) {
    if (key < k[3]) {
        k[3] = key;
        if (k[3] < k[2]) { const unsigned t = k[2]; k[2] = k[3]; k[3] = t; }
        if (k[2] < k[1]) { const unsigned t = k[1]; k[1] = k[2]; k[2] = t; }
        if (k[1] < k[0]) { const unsigned t = k[0]; k[0] = k[1]; k[1] = t; }
    }
}

using ovs::cv_ceil_f;
using ovs::cv_floor_f;
using ovs::hamming256;
using ovs::WindowFrame;

// One chunk of a warp's running top-K (k_triangulation_topk, k_node_topk): lane r < K carries entry r in `extra`, every lane
// holds up to K keys of the chunk in mine[]; returns lane r's entry r of the K smallest keys of both.  Keys are unique (they
// carry the candidate's rank).
template <int K>
__device__ __forceinline__ unsigned warp_merge_topk(unsigned extra, unsigned (&mine)[K], int lane) {
    unsigned next_extra = 0xffffffffu;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        unsigned lmin = extra;
#pragma unroll
        for (int k = 0; k < K; ++k) lmin = min(lmin, mine[k]);
        const unsigned wmin = __reduce_min_sync(0xffffffffu, lmin);
        if (wmin != 0xffffffffu) {
            if (extra == wmin) extra = 0xffffffffu;
#pragma unroll
            for (int k = 0; k < K; ++k) if (mine[k] == wmin) mine[k] = 0xffffffffu;
        }
        if (lane == r) next_extra = wmin;
    }
    return next_extra;
}

struct WindowQueries {
    int nq;
    const float2* ref; const float* margin; const int* min_level; const int* max_level; const float* xr; const uint4* desc;
    // match::fuse: instead of the x_right window test, a candidate is skipped when its reprojection error exceeds the
    // chi-square bound of its own octave (5.99 monocular, 7.8 with the x_right term)
    int fuse_gate;
    float inv_sigma_sq[16];
};

__global__ void __launch_bounds__(128) k_window_topk(WindowFrame F, WindowQueries Q, unsigned* __restrict__ out) {
    const int q = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= Q.nq) return;
    unsigned best[kTopK] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    ovs::window_walk(F, Q.ref[q], Q.margin[q], Q.min_level[q], Q.max_level[q], Q.xr != nullptr, [&] { return Q.xr ? Q.xr[q] : -1.0f; }, Q.desc + 2 * (size_t)q,
                     Q.fuse_gate != 0, [&](int o) { return Q.inv_sigma_sq[o & 15]; }, lane,
                     [&](unsigned key) { topk_insert(best, key); });
    // merge the 32 sorted lists: 4 rounds of warp-wide minimum
#pragma unroll
    for (int k = 0; k < kTopK; ++k) {
        const unsigned m = __reduce_min_sync(0xffffffffu, best[0]);
        if (best[0] == m && m != 0xffffffffu) { best[0] = best[1]; best[1] = best[2]; best[2] = best[3]; best[3] = 0xffffffffu; }
        if (lane == 0) out[(size_t)q * kTopK + k] = m;
    }
}

// ------------------------------------------------------------------------------------ stereo
struct StereoArgs {
    int n_left, n_right;
    const float* lx; const float* ly; const int* loct; const uint4* ldesc;
    const float* rx; const float* ry; const int* roct; const uint4* rdesc;
    float min_disp, max_disp; int hamm_thr; int rows0;
    float scale[16], inv_scale[16];
    const uint8_t* lpyr[16]; const uint8_t* rpyr[16]; int pw[16], ph[16], pitch[16];
    float focal_x_baseline;
};

// best[il] = (dist << 16 | idx_right) or 0xFFFFFFFF; flag bit 31 of any[il] unused.
__global__ void __launch_bounds__(128) k_stereo_match(StereoArgs A, unsigned* __restrict__ best_out) {
    __shared__ float s_rx[256], s_lo[256], s_hi[256];
    __shared__ int s_oct[256];
    __shared__ uint4 s_desc[512];
    const int il = blockIdx.x * 128 + threadIdx.x;
    const bool act = il < A.n_left;
    float x_left = 0, y_left = 0; int lvl = 0; uint4 qa = make_uint4(0, 0, 0, 0), qb = qa;
    if (act) { x_left = A.lx[il]; y_left = A.ly[il]; lvl = A.loct[il]; qa = __ldg(A.ldesc + 2 * (size_t)il); qb = __ldg(A.ldesc + 2 * (size_t)il + 1); }
    const int row = (int)y_left;
    const float min_x_right = __fsub_rn(x_left, A.max_disp), max_x_right = __fsub_rn(x_left, A.min_disp);
    // a keypoint with a coordinate that is not finite takes no part (the reference's conversions are undefined there)
    const bool usable = act && isfinite(x_left) && isfinite(y_left) && row >= 0 && row < A.rows0 && !(max_x_right < 0);
    unsigned best = ((unsigned)A.hamm_thr << 16) | 0xffffu;   // sentinel: distance == threshold
    for (int t0 = 0; t0 < A.n_right; t0 += 256) {
        const int n = min(256, A.n_right - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += 128) {
            const int ir = t0 + i;
            const int o = A.roct[ir];
            const float r = __fmul_rn(2.0f, A.scale[o]);
            const float yy = A.ry[ir];
            s_rx[i] = A.rx[ir]; s_oct[i] = o;
            const bool finite = isfinite(yy) && isfinite(A.rx[ir]);   // else an empty band: no candidate
            s_lo[i] = finite ? (float)cv_floor_f(__fsub_rn(yy, r)) : INFINITY; s_hi[i] = finite ? (float)cv_ceil_f(__fadd_rn(yy, r)) : -INFINITY;
            s_desc[2 * i] = __ldg(A.rdesc + 2 * (size_t)ir); s_desc[2 * i + 1] = __ldg(A.rdesc + 2 * (size_t)ir + 1);
        }
        __syncthreads();
        if (!usable) continue;
        for (int j = 0; j < n; ++j) {
            if ((float)row < s_lo[j] || (float)row > s_hi[j]) continue;
            const int o = s_oct[j];
            if (o < lvl - 1 || o > lvl + 1) continue;
            const float xr = s_rx[j];
            if (xr < min_x_right || max_x_right < xr) continue;
            const uint4 ta = s_desc[2 * j], tb = s_desc[2 * j + 1];
            const int d = hamming256(qa, qb, ta, tb);
            const unsigned key = ((unsigned)d << 16) | (unsigned)(t0 + j);
            if ((key >> 16) < (best >> 16)) best = key;   // strict '<' on the distance: first (lowest index) wins ties
        }
    }
    if (act) best_out[il] = (usable && (best >> 16) < (unsigned)A.hamm_thr) ? best : 0xffffffffu;
}

// One warp per left keypoint with a Hamming match: SAD over 11 horizontal offsets, parabola fit,
// disparity checks.  Writes x_right / depth (-1 if rejected) and the best SAD (for the median test).
__global__ void __launch_bounds__(128) k_stereo_subpixel(StereoArgs A, const unsigned* __restrict__ best_in, float* __restrict__ x_right_out,
                                                          float* __restrict__ depth_out, unsigned* __restrict__ corr_out) {
    const int il = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (il >= A.n_left) return;
    float xr_res = -1.0f, depth_res = -1.0f; unsigned corr_res = 0xffffffffu;
    const unsigned key = best_in[il];
    if (key != 0xffffffffu) {
        const int ir = (int)(key & 0xffffu);
        const int lvl = A.loct[il];
        const float x_left = A.lx[il], y_left = A.ly[il];
        const float inv_s = A.inv_scale[lvl];
        const int sxl = __float2int_rn(__fmul_rn(x_left, inv_s)), syl = __float2int_rn(__fmul_rn(y_left, inv_s));
        const int sxr = __float2int_rn(__fmul_rn(A.rx[ir], inv_s));
        constexpr int win = 5, slide = 5;
        const int W = A.pw[lvl], Hh = A.ph[lvl], S = A.pitch[lvl];
        // ini_x = sxr - slide - win >= 0, end_x = sxr + slide + win + 1 < W and the left window, without overflow: the
        // conversions saturate, so a coordinate past the int range lands outside every window
        const bool fits = !(sxr < slide + win || W - (slide + win + 1) <= sxr) && !(sxl < win || W - win <= sxl || syl < win || Hh - win <= syl);
        if (fits) {
            const uint8_t* L = A.lpyr[lvl]; const uint8_t* R = A.rpyr[lvl];
            const int cl = L[(size_t)syl * S + sxl];
            // each lane owns up to 4 of the 121 window pixels
            int lv[4], py[4], px[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int p = lane + 32 * k;
                py[k] = p / 11 - win; px[k] = p % 11 - win;
                lv[k] = (p < 121) ? (int)L[(size_t)(syl + py[k]) * S + sxl + px[k]] - cl : 0;
            }
            unsigned best_corr = 0xffffffffu; int best_off = 0;
            unsigned sads[2 * slide + 1];
#pragma unroll
            for (int off = -slide; off <= slide; ++off) {
                const int cr = R[(size_t)syl * S + sxr + off];
                unsigned sad = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int p = lane + 32 * k;
                    if (p < 121) {
                        const int b = (int)R[(size_t)(syl + py[k]) * S + sxr + off + px[k]] - cr;
                        sad += (unsigned)abs(lv[k] - b);
                    }
                }
                sad = __reduce_add_sync(0xffffffffu, sad);
                sads[off + slide] = sad;
                if (sad < best_corr) { best_corr = sad; best_off = off; }
            }
            if (!(best_off == -slide || best_off == slide)) {
                float c1 = 0, c2 = 0, c3 = 0;
#pragma unroll
                for (int k = 1; k < 2 * slide; ++k)
                    if (k == best_off + slide) { c1 = (float)sads[k - 1]; c2 = (float)sads[k]; c3 = (float)sads[k + 1]; }
                const float delta = (float)((double)__fsub_rn(c1, c3) / (2.0 * ((double)__fadd_rn(c1, c3) - 2.0 * (double)c2)));
                if (!(delta < -1.0f || 1.0f < delta)) {
                    float best_x_right = __fmul_rn(A.scale[lvl], __fadd_rn((float)(sxr + best_off), delta));
                    float disp = __fsub_rn(x_left, best_x_right);
                    if (!(disp < A.min_disp || A.max_disp <= disp)) {
                        if (disp <= 0.0f) { disp = 0.01f; best_x_right = __fsub_rn(x_left, disp); }
                        depth_res = __fdiv_rn(A.focal_x_baseline, disp);
                        xr_res = best_x_right;
                        corr_res = best_corr;
                    }
                }
            }
        }
    }
    if (lane == 0) { x_right_out[il] = xr_res; depth_out[il] = depth_res; corr_out[il] = corr_res; }
}

using ovs::key_dist;
inline int key_rank(unsigned key) { return key == 0xffffffffu ? -1 : (int)(key & 0xffffu); }

// data::get_cell_indices
inline bool cell_of(const ovs_grid& g, float x, float y, int* cx, int* cy) {
    *cx = (int)std::floor((double)((x - g.min_x) * g.inv_cell_width));
    *cy = (int)std::floor((double)((y - g.min_y) * g.inv_cell_height));
    return 0 <= *cx && *cx < g.num_grid_cols && 0 <= *cy && *cy < g.num_grid_rows;
}

// Runs k_window_topk for nq host queries; keys land in m->h_keys[0 .. nq*4).  `cap` (rank order, n
// entries) or nullptr.  use_xr: the keypoints' x_right take part (the x_right test, or the fuse gate's x_right term).
int window_topk(const ovs_frame_index* f, bool use_xr, int nq, const float* ref_xy, const float* margin, const int* min_level,
                const int* max_level, const float* xr_q, const uint8_t* qdesc, const unsigned short* cap_rank_order,
                const float* fuse_inv_sigma_sq = nullptr, int fuse_levels = 0) {
    ovs_matcher* m = f->m;
    cudaStream_t st = m->stream;
    const size_t N = (size_t)nq;
    WindowQueries Q;
    uint8_t* hdesc; float2* href; float *hm, *hxr; int *hlo, *hhi; float* dxr;
    ovs::Staging S;
    int rc = ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_q, m->d_q_cap, [&](ovs::Staging& S) {
        Q.desc = (const uint4*)S.in(hdesc, 32 * N); Q.ref = S.in(href, N); Q.margin = S.in(hm, N);
        Q.min_level = S.in(hlo, N); Q.max_level = S.in(hhi, N); dxr = S.in(hxr, N);
    });
    if (rc != OVS_OK) return rc;
    if ((rc = ovs::grow_dev(&m->d_keys, &m->d_keys_cap, (N + 1) * kTopK)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&m->h_keys, &m->h_keys_cap, (N + 1) * kTopK)) != OVS_OK) return rc;
    memcpy(hdesc, qdesc, 32 * N); memcpy(href, ref_xy, 8 * N); memcpy(hm, margin, 4 * N);
    memcpy(hlo, min_level, 4 * N); memcpy(hhi, max_level, 4 * N);
    if (xr_q) memcpy(hxr, xr_q, 4 * N);
    OVS_CUDA_CHECK(S.upload(st));
    if (cap_rank_order) OVS_CUDA_CHECK(cudaMemcpyAsync(f->d_cap, cap_rank_order, 2 * (size_t)std::max(f->nranked, 1), cudaMemcpyHostToDevice, st));
    WindowFrame F;
    F.min_x = f->grid.min_x; F.min_y = f->grid.min_y; F.inv_w = f->grid.inv_cell_width; F.inv_h = f->grid.inv_cell_height;
    F.cols = f->grid.num_grid_cols; F.rows = f->grid.num_grid_rows;
    F.x = f->d_x; F.y = f->d_y; F.xr = use_xr ? f->d_xr : nullptr; F.oct = f->d_oct; F.desc = f->d_desc;
    F.cell_start = f->d_cell_start; F.cap = cap_rank_order ? f->d_cap : nullptr;
    Q.nq = nq; Q.xr = xr_q ? dxr : nullptr;
    Q.fuse_gate = fuse_inv_sigma_sq ? 1 : 0;
    for (int l = 0; l < 16; ++l) Q.inv_sigma_sq[l] = (fuse_inv_sigma_sq && l < fuse_levels) ? fuse_inv_sigma_sq[l] : 0.0f;
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_window_topk<<<(nq + 3) / 4, 128, 0, st>>>(F, Q, m->d_keys);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys, m->d_keys, N * kTopK * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    return OVS_OK;
}

// Re-runs one query with a distance cap per keypoint (cap[idx]: candidate valid iff d < cap[idx]).
int requery(const ovs_frame_index* f, bool use_xr, const float* ref_xy, float margin, int min_level, int max_level, const float* xr_q,
            const uint8_t* qdesc, const std::vector<unsigned short>& cap_by_idx, unsigned* keys_out) {
    ++f->m->num_requeries;
    std::vector<unsigned short> cap((size_t)std::max(f->nranked, 1));
    for (int r = 0; r < f->nranked; ++r) cap[r] = cap_by_idx[f->rank_to_idx[r]];
    int rc = window_topk(f, use_xr, 1, ref_xy, &margin, &min_level, &max_level, xr_q, qdesc, cap.data());
    if (rc != OVS_OK) return rc;
    memcpy(keys_out, f->m->h_keys, kTopK * sizeof(unsigned));
    return OVS_OK;
}

}  // namespace

// data::assign_keypoints_to_grid: counting sort by cell (cx major, cy minor), index order kept inside a cell.  Fills rank_to_idx /
// idx_to_rank / nranked and returns the cell CSR.
std::vector<int> ovs::rank_keypoints(const ovs_grid& grid, int n, const float* x, const float* y, std::vector<int>& rank_to_idx,
                                     std::vector<int>& idx_to_rank, int* nranked) {
    const int ncells = grid.num_grid_cols * grid.num_grid_rows;
    std::vector<int> cell(n, -1), start(ncells + 1, 0);
    for (int i = 0; i < n; ++i) {
        int cx, cy;
        if (cell_of(grid, x[i], y[i], &cx, &cy)) { cell[i] = cx * grid.num_grid_rows + cy; start[cell[i] + 1]++; }
    }
    for (int c = 0; c < ncells; ++c) start[c + 1] += start[c];
    *nranked = start[ncells];
    rank_to_idx.assign(std::max(*nranked, 1), 0); idx_to_rank.assign(std::max(n, 1), -1);
    std::vector<int> pos(start.begin(), start.end() - 1);
    for (int i = 0; i < n; ++i) if (cell[i] >= 0) { const int r = pos[cell[i]]++; rank_to_idx[r] = i; idx_to_rank[i] = r; }
    return start;
}

namespace {

std::vector<int> rank_keypoints(ovs_frame_index* f) {
    return ovs::rank_keypoints(f->grid, f->n, f->hx.data(), f->hy.data(), f->rank_to_idx, f->idx_to_rank, &f->nranked);
}

bool alloc_index_arrays(ovs_frame_index* f, size_t R, int ncells) {
    auto carve = [&](ovs::Arena& A) {
        f->d_desc = A.take<uint4>(2 * R); f->d_x = A.take<float>(R); f->d_y = A.take<float>(R); f->d_xr = A.take<float>(R);
        f->d_rank = A.take<int>(R); f->d_cell_start = A.take<int>((size_t)ncells + 1); f->d_cap = A.take<unsigned short>(R);
        f->d_oct = A.take<signed char>(R);
    };
    ovs::Arena A{nullptr, 0};
    carve(A);
    const size_t need = A.off;
    ovs_matcher* m = f->m;
    int pick = -1;
    for (int i = 0; i < (int)m->index_pool.size(); ++i)
        if (m->index_pool[i].cap >= need && (pick < 0 || m->index_pool[i].cap < m->index_pool[pick].cap)) pick = i;
    if (pick >= 0) {
        f->buf = m->index_pool[pick];
        m->index_pool.erase(m->index_pool.begin() + pick);
    } else {
        const size_t cap = need + need / 4;
        if (cudaMalloc(&f->buf.base, cap) != cudaSuccess) { f->buf = ovs_index_buf(); return false; }
        f->buf.cap = cap;
    }
    A = ovs::Arena{f->buf.base, 0};
    carve(A);
    return true;
}

// rank-ordered SoA of the index straight from the extractor's device output (ovs_keypoint AoS + descriptors)
__global__ void __launch_bounds__(128) k_index_gather(int nranked, const int* __restrict__ rank_to_idx, const ovs_keypoint* __restrict__ kps,
                                                      const uint4* __restrict__ desc, const float* __restrict__ x_right,
                                                      float* __restrict__ ox, float* __restrict__ oy, float* __restrict__ oxr,
                                                      signed char* __restrict__ ooct, uint4* __restrict__ odesc) {
    const int r = blockIdx.x * 128 + threadIdx.x;
    if (r >= nranked) return;
    const int i = rank_to_idx[r];
    const ovs_keypoint k = kps[i];
    ox[r] = k.x; oy[r] = k.y; ooct[r] = (signed char)k.octave;
    oxr[r] = x_right ? x_right[i] : -1.0f;
    odesc[2 * (size_t)r] = desc[2 * (size_t)i];
    odesc[2 * (size_t)r + 1] = desc[2 * (size_t)i + 1];
}

}  // namespace

extern "C" int ovs_frame_index_create(ovs_matcher* m, int n, const float* x, const float* y, const int32_t* octave, const float* angle,
                                      const float* x_right, const uint8_t* desc, const ovs_grid* grid, ovs_frame_index** out) {
    OVS_REQUIRE(m && grid && out && n >= 0 && (n == 0 || (x && y && octave && desc)), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 keypoints");
    OVS_REQUIRE(grid->num_grid_cols > 0 && grid->num_grid_rows > 0 && grid->num_grid_cols * grid->num_grid_rows <= 1 << 20,
                OVS_ERR_INVALID_ARG, "bad grid");
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    ovs_frame_index* f = new (std::nothrow) ovs_frame_index();
    OVS_REQUIRE(f, OVS_ERR_CUDA, "out of host memory");
    f->m = m; f->n = n; f->grid = *grid; f->has_xr = x_right != nullptr;
    f->hx.assign(x, x + n); f->hy.assign(y, y + n); f->hoct.assign(octave, octave + n);
    if (angle) f->hangle.assign(angle, angle + n); else f->hangle.assign(n, 0.f);
    if (x_right) f->hxr.assign(x_right, x_right + n); else f->hxr.assign(n, -1.0f);
    const int ncells = grid->num_grid_cols * grid->num_grid_rows;
    const std::vector<int> start = rank_keypoints(f);
    const size_t R = (size_t)std::max(f->nranked, 1);
    std::vector<float> rx(R), ry(R), rxr(R); std::vector<signed char> roct(R); std::vector<uint8_t> rdesc(R * 32);
    for (int r = 0; r < f->nranked; ++r) {
        const int i = f->rank_to_idx[r];
        rx[r] = x[i]; ry[r] = y[i]; rxr[r] = f->hxr[i]; roct[r] = (signed char)octave[i];
        memcpy(&rdesc[(size_t)r * 32], desc + (size_t)i * 32, 32);
    }
    bool ok = alloc_index_arrays(f, R, ncells);
    if (ok) {
        cudaStream_t st = m->stream;
        ok = cudaMemcpyAsync(f->d_x, rx.data(), R * 4, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_y, ry.data(), R * 4, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_xr, rxr.data(), R * 4, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_oct, roct.data(), R, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_desc, rdesc.data(), R * 32, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_cell_start, start.data(), (size_t)(ncells + 1) * 4, cudaMemcpyHostToDevice, st) == cudaSuccess
             && ovs::sync_stream(st) == cudaSuccess;
    }
    if (!ok) {
        ovs::set_error("frame index allocation/upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        ovs_frame_index_destroy(f);
        return OVS_ERR_CUDA;
    }
    *out = f;
    return OVS_OK;
}

// The same index from the extractor's DEVICE output (ovs_extract_device): the descriptors never leave the GPU.  Only the
// keypoint records (28 B each; the host side of the matchers needs positions, octaves and angles anyway) come to the
// host, where assign_keypoints_to_grid is a counting sort; the rank-ordered arrays are then gathered on the device.
extern "C" int ovs_frame_index_create_device(ovs_matcher* m, int n, const ovs_keypoint* d_keypts, const uint8_t* d_desc,
                                             const float* d_x_right, const ovs_grid* grid, ovs_frame_index** out) {
    OVS_REQUIRE(m && grid && out && n >= 0 && (n == 0 || (d_keypts && d_desc)), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 keypoints");
    OVS_REQUIRE(grid->num_grid_cols > 0 && grid->num_grid_rows > 0 && grid->num_grid_cols * grid->num_grid_rows <= 1 << 20,
                OVS_ERR_INVALID_ARG, "bad grid");
    OVS_REQUIRE((reinterpret_cast<uintptr_t>(d_desc) & 15) == 0, OVS_ERR_INVALID_ARG, "descriptors must be 16-byte aligned");
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    cudaStream_t st = m->stream;
    const size_t N = (size_t)std::max(n, 1);
    ovs_keypoint* hk; float* hxr;
    auto carve = [&](ovs::Arena& H) { hk = H.take<ovs_keypoint>(N); hxr = H.take<float>(N); };
    ovs::Arena H{nullptr, 0};
    carve(H);
    const int rc = ovs::grow_host(&m->h_stage, &m->h_stage_cap, H.off);
    if (rc != OVS_OK) return rc;
    H = ovs::Arena{m->h_stage, 0};
    carve(H);
    if (n) OVS_CUDA_CHECK(cudaMemcpyAsync(hk, d_keypts, (size_t)n * sizeof(ovs_keypoint), cudaMemcpyDeviceToHost, st));
    if (n && d_x_right) OVS_CUDA_CHECK(cudaMemcpyAsync(hxr, d_x_right, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    ovs_frame_index* f = new (std::nothrow) ovs_frame_index();
    OVS_REQUIRE(f, OVS_ERR_CUDA, "out of host memory");
    f->m = m; f->n = n; f->grid = *grid; f->has_xr = d_x_right != nullptr;
    f->hx.resize(n); f->hy.resize(n); f->hoct.resize(n); f->hangle.resize(n); f->hxr.assign(n, -1.0f);
    for (int i = 0; i < n; ++i) {
        f->hx[i] = hk[i].x; f->hy[i] = hk[i].y; f->hoct[i] = hk[i].octave; f->hangle[i] = hk[i].angle;
        if (d_x_right) f->hxr[i] = hxr[i];
    }
    const int ncells = grid->num_grid_cols * grid->num_grid_rows;
    const std::vector<int> start = rank_keypoints(f);
    const size_t R = (size_t)std::max(f->nranked, 1);
    bool ok = alloc_index_arrays(f, R, ncells);
    int* const d_rank = f->d_rank;
    if (ok) {
        ok = cudaMemcpyAsync(d_rank, f->rank_to_idx.data(), R * 4, cudaMemcpyHostToDevice, st) == cudaSuccess
             && cudaMemcpyAsync(f->d_cell_start, start.data(), (size_t)(ncells + 1) * 4, cudaMemcpyHostToDevice, st) == cudaSuccess;
        if (ok && f->nranked) {
            k_index_gather<<<(f->nranked + 127) / 128, 128, 0, st>>>(f->nranked, d_rank, d_keypts, reinterpret_cast<const uint4*>(d_desc), d_x_right,
                                                                     f->d_x, f->d_y, f->d_xr, f->d_oct, f->d_desc);
            ovs::count_launch();
            ok = cudaGetLastError() == cudaSuccess;
        }
        ok = ok && ovs::sync_stream(st) == cudaSuccess;
    }
    if (!ok) {
        ovs::set_error("frame index allocation/gather failed: %s", cudaGetErrorString(cudaGetLastError()));
        ovs_frame_index_destroy(f);
        return OVS_ERR_CUDA;
    }
    *out = f;
    return OVS_OK;
}

extern "C" void ovs_frame_index_destroy(ovs_frame_index* f) {
    if (!f) return;
    if (f->m) cudaSetDevice(f->m->device);
    if (f->buf.base) {
        // every call on the index returned with the matcher's stream drained, so the buffer is idle: keep it for the next frame
        if (f->m && f->m->index_pool.size() < 8) f->m->index_pool.push_back(f->buf);
        else cudaFree(f->buf.base);
    }
    delete f;
}

// get_keypoints_in_cell + nearest-descriptor search for nq queries: the 4 best candidates of each
// query in the reference's visiting order.  idx_out / dist_out [nq * 4], -1 / 256 where absent.
extern "C" int ovs_match_window_topk_host(ovs_frame_index* f, int nq, const float* ref_xy, const float* margin, const int32_t* min_level,
                                          const int32_t* max_level, const float* x_right_q, const uint8_t* qdesc,
                                          int32_t* idx_out, int32_t* dist_out) {
    OVS_REQUIRE(f && nq >= 0 && (nq == 0 || (ref_xy && margin && min_level && max_level && qdesc && idx_out && dist_out)), OVS_ERR_INVALID_ARG, "bad argument");
    if (nq == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(f->m->device));
    int rc = window_topk(f, f->has_xr, nq, ref_xy, margin, min_level, max_level, x_right_q, qdesc, nullptr);
    if (rc != OVS_OK) return rc;
    for (size_t i = 0; i < (size_t)nq * kTopK; ++i) {
        const unsigned k = f->m->h_keys[i];
        idx_out[i] = k == 0xffffffffu ? -1 : f->rank_to_idx[key_rank(k)];
        dist_out[i] = key_dist(k);
    }
    return OVS_OK;
}

// match::projection::match_keyframes_mutually(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, Sim3s, margin): every usable
// landmark of keyframe 1 (index = its keypoint in keyframe 1) looks for its nearest keypoint of keyframe 2 inside the
// window around its reprojection, levels [pred - 1, pred], distance <= HAMMING_DIST_THR_HIGH -- independently of the
// other landmarks (no first-taker rule in this matcher) -- and vice versa; a pair is kept when both directions agree.
extern "C" int ovs_projection_match_keyframes_mutually_host(ovs_frame_index* f1, ovs_frame_index* f2, const float* scale_factors,
                                                            const uint8_t* usable_1, const float* reproj_1_in_2, const int32_t* pred_level_1_in_2,
                                                            const uint8_t* lm_desc_1, const uint8_t* usable_2, const float* reproj_2_in_1,
                                                            const int32_t* pred_level_2_in_1, const uint8_t* lm_desc_2, float margin,
                                                            int32_t* matched_idx_2_of_kp_1, int* num_matches) {
    OVS_REQUIRE(f1 && f2 && scale_factors && matched_idx_2_of_kp_1 && num_matches, OVS_ERR_INVALID_ARG, "bad argument");
    const int n1 = f1->n, n2 = f2->n;
    OVS_REQUIRE((n1 == 0 || (reproj_1_in_2 && pred_level_1_in_2 && lm_desc_1)) && (n2 == 0 || (reproj_2_in_1 && pred_level_2_in_1 && lm_desc_2)),
                OVS_ERR_INVALID_ARG, "null argument");
    *num_matches = 0;
    for (int i = 0; i < n1; ++i) matched_idx_2_of_kp_1[i] = -1;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    // one direction: best keypoint of `dst` for every usable landmark of the other keyframe
    auto one_way = [&](ovs_frame_index* dst, int nq, const uint8_t* usable, const float* reproj, const int32_t* lvl, const uint8_t* desc,
                       std::vector<int>& best) -> int {
        OVS_CUDA_CHECK(cudaSetDevice(dst->m->device));
        std::vector<float> mg(nq); std::vector<int32_t> lo(nq), hi(nq);
        for (int q = 0; q < nq; ++q) {
            const int l = lvl[q];
            mg[q] = margin * scale_factors[l < 0 ? 0 : l];
            lo[q] = l - 1; hi[q] = l;
            if (usable && !usable[q]) { lo[q] = 1; hi[q] = 0; }   // empty level range: no candidates
        }
        const int rc = window_topk(dst, dst->has_xr, nq, reproj, mg.data(), lo.data(), hi.data(), nullptr, desc, nullptr);
        if (rc != OVS_OK) return rc;
        best.assign(nq, -1);
        for (int q = 0; q < nq; ++q) {
            if (usable && !usable[q]) continue;
            const unsigned k = dst->m->h_keys[(size_t)q * kTopK];
            if (k != 0xffffffffu && key_dist(k) <= OVS_HAMMING_DIST_THR_HIGH) best[q] = dst->rank_to_idx[key_rank(k)];
        }
        return OVS_OK;
    };
    std::vector<int> best_2_of_1, best_1_of_2;
    int rc = one_way(f2, n1, usable_1, reproj_1_in_2, pred_level_1_in_2, lm_desc_1, best_2_of_1);
    if (rc != OVS_OK) return rc;
    rc = one_way(f1, n2, usable_2, reproj_2_in_1, pred_level_2_in_1, lm_desc_2, best_1_of_2);
    if (rc != OVS_OK) return rc;
    for (int i1 = 0; i1 < n1; ++i1) {
        const int i2 = best_2_of_1[i1];
        if (i2 >= 0 && best_1_of_2[i2] == i1) { matched_idx_2_of_kp_1[i1] = i2; ++*num_matches; }
    }
    return OVS_OK;
}

// match::projection::match_frame_and_landmarks(frm, local_landmarks, margin)
extern "C" int ovs_projection_match_frame_and_landmarks_host(ovs_frame_index* f, const float* scale_factors, int num_scale_levels, int nlm, const uint8_t* lm_usable,
                                                             const float* reproj_xy, const float* x_right_in_tracking,
                                                             const int32_t* pred_scale_level, const uint8_t* lm_desc,
                                                             const uint8_t* kp_has_observed_lm, float margin, float lowe_ratio,
                                                             int32_t* matched_lm_of_kp, int* num_matches) {
    OVS_REQUIRE(f && scale_factors && num_matches && matched_lm_of_kp && nlm >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(nlm == 0 || (reproj_xy && pred_scale_level && lm_desc), OVS_ERR_INVALID_ARG, "null argument");
    OVS_CUDA_CHECK(cudaSetDevice(f->m->device));
    const int n = f->n;
    for (int i = 0; i < n; ++i) matched_lm_of_kp[i] = -1;
    *num_matches = 0;
    if (nlm == 0 || n == 0) return OVS_OK;
    // queries = usable landmarks
    OVS_REQUIRE(num_scale_levels >= 1, OVS_ERR_INVALID_ARG, "bad scale table");
    std::vector<int> qlm; qlm.reserve(nlm);
    for (int l = 0; l < nlm; ++l) {
        if (lm_usable && !lm_usable[l]) continue;
        // the reference indexes scale_factors_.at(pred_scale_level): out of range throws there, is an error here
        OVS_REQUIRE(pred_scale_level[l] >= 0 && pred_scale_level[l] < num_scale_levels, OVS_ERR_INVALID_ARG,
                    "predicted scale level %d of landmark %d outside the scale table (%d levels)", pred_scale_level[l], l, num_scale_levels);
        qlm.push_back(l);
    }
    const int nq = (int)qlm.size();
    if (nq == 0) return OVS_OK;
    std::vector<float> ref(2 * (size_t)nq), mg(nq), xr(nq); std::vector<int> lo(nq), hi(nq); std::vector<uint8_t> qd(32 * (size_t)nq);
    for (int q = 0; q < nq; ++q) {
        const int l = qlm[q], lvl = pred_scale_level[l];
        ref[2 * q] = reproj_xy[2 * l]; ref[2 * q + 1] = reproj_xy[2 * l + 1];
        mg[q] = margin * scale_factors[lvl]; lo[q] = lvl - 1; hi[q] = lvl;
        xr[q] = x_right_in_tracking ? x_right_in_tracking[l] : -1.0f;
        memcpy(&qd[32 * (size_t)q], lm_desc + 32 * (size_t)l, 32);
    }
    std::vector<unsigned short> cap(std::max(n, 1), 0xffff);   // 0 = keypoint unavailable
    if (kp_has_observed_lm) for (int i = 0; i < n; ++i) if (kp_has_observed_lm[i]) cap[i] = 0;
    int rc;
    {
        std::vector<unsigned short> cap_rank((size_t)std::max(f->nranked, 1));
        for (int r = 0; r < f->nranked; ++r) cap_rank[r] = cap[f->rank_to_idx[r]];
        rc = window_topk(f, f->has_xr, nq, ref.data(), mg.data(), lo.data(), hi.data(), f->has_xr ? xr.data() : nullptr, qd.data(), cap_rank.data());
        if (rc != OVS_OK) return rc;
    }
    std::vector<unsigned> keys(f->m->h_keys, f->m->h_keys + (size_t)nq * kTopK);   // a re-query overwrites h_keys
    const auto decode = [&](unsigned key) { return f->rank_to_idx[key_rank(key)]; };
    const auto available = [&](int idx, int) { return cap[idx] != 0; };
    // the reference's ratio test applies only when the best and the second best share a level; against a lower bound it
    // always applies (only the true second could pass it)
    const auto ratio = [&](const ovs::ReplayList<kTopK>& L, int second, ovs::Second kind) {
        if (kind == ovs::Second::bound) return !((float)L.dist[0] > lowe_ratio * (float)second);
        const int second_level = kind == ovs::Second::listed ? f->hoct[L.id[1]] : -1;
        return !(f->hoct[L.id[0]] == second_level && (float)L.dist[0] > lowe_ratio * (float)second);
    };
    int nm = 0;
    for (int q = 0; q < nq; ++q) {
        const auto requery_q = [&](unsigned* fresh) {
            return requery(f, f->has_xr, &ref[2 * q], mg[q], lo[q], hi[q], f->has_xr ? &xr[q] : nullptr, &qd[32 * (size_t)q], cap, fresh);
        };
        ovs::ReplayPick p;
        rc = ovs::replay_query<kTopK>(&keys[(size_t)q * kTopK], OVS_HAMMING_DIST_THR_HIGH, ovs::kNeverComplete, decode, available, ratio,
                                      requery_q, &p);
        if (rc != OVS_OK) return rc;
        if (p.id >= 0) { matched_lm_of_kp[p.id] = qlm[q]; cap[p.id] = 0; ++nm; }
    }
    *num_matches = nm;
    return OVS_OK;
}

// match::fuse (match/fuse.cc; ORB-SLAM2 ORBmatcher::Fuse): the matching core of fuse::replace_duplication /
// detect_duplication.  Every usable landmark (reprojected into the keyframe by the caller, who also does the depth-range and
// viewing-angle tests and predict_scale_level) searches the window margin * scale_factors[level] over the levels
// [level - 1, level]; candidates whose reprojection error exceeds the chi-square bound of their own octave are skipped;
// the nearest descriptor wins (first in visiting order on ties), accepted at <= HAMMING_DIST_THR_LOW.  There is no
// first-taker rule in this matcher, so the whole search is one kernel and no replay.  best_idx_of_lm[q] = keypoint or -1.
extern "C" int ovs_fuse_best_keypoints_host(ovs_frame_index* f, int nq, const uint8_t* usable, const float* reproj_xy, const float* reproj_x_right,
                                            const int32_t* pred_level, const uint8_t* lm_desc, const float* scale_factors,
                                            const float* inv_level_sigma_sq, int num_scale_levels, float margin,
                                            int32_t* best_idx_of_lm, int* num_matches) {
    OVS_REQUIRE(f && num_matches && nq >= 0 && (nq == 0 || (reproj_xy && pred_level && lm_desc && best_idx_of_lm)), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(scale_factors && inv_level_sigma_sq && num_scale_levels >= 1 && num_scale_levels <= 16, OVS_ERR_INVALID_ARG, "bad scale tables");
    *num_matches = 0;
    for (int q = 0; q < nq; ++q) best_idx_of_lm[q] = -1;
    if (nq == 0 || f->n == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(f->m->device));
    for (int i = 0; i < f->n; ++i)
        OVS_REQUIRE(f->hoct[i] >= 0 && f->hoct[i] < num_scale_levels, OVS_ERR_INVALID_ARG, "octave %d of keypoint %d outside the scale tables", f->hoct[i], i);
    std::vector<int> ql; ql.reserve(nq);
    for (int q = 0; q < nq; ++q) {
        if (usable && !usable[q]) continue;
        OVS_REQUIRE(pred_level[q] < num_scale_levels, OVS_ERR_INVALID_ARG, "predicted level %d of landmark %d outside the scale tables", pred_level[q], q);
        ql.push_back(q);
    }
    const int nu = (int)ql.size();
    if (nu == 0) return OVS_OK;
    std::vector<float> ref(2 * (size_t)nu), mg(nu), xr(nu); std::vector<int> lo(nu), hi(nu); std::vector<uint8_t> qd(32 * (size_t)nu);
    for (int k = 0; k < nu; ++k) {
        const int q = ql[k], l = pred_level[q];
        ref[2 * k] = reproj_xy[2 * q]; ref[2 * k + 1] = reproj_xy[2 * q + 1];
        mg[k] = margin * scale_factors[l < 0 ? 0 : l]; lo[k] = l - 1; hi[k] = l;
        xr[k] = reproj_x_right ? reproj_x_right[q] : -1.0f;
        memcpy(&qd[32 * (size_t)k], lm_desc + 32 * (size_t)q, 32);
    }
    const int rc = window_topk(f, f->has_xr, nu, ref.data(), mg.data(), lo.data(), hi.data(), reproj_x_right ? xr.data() : nullptr, qd.data(), nullptr,
                               inv_level_sigma_sq, num_scale_levels);
    if (rc != OVS_OK) return rc;
    int num = 0;
    for (int k = 0; k < nu; ++k) {
        const unsigned key = f->m->h_keys[(size_t)k * kTopK];
        if (key != 0xffffffffu && key_dist(key) <= OVS_HAMMING_DIST_THR_LOW) { best_idx_of_lm[ql[k]] = f->rank_to_idx[key_rank(key)]; ++num; }
    }
    *num_matches = num;
    return OVS_OK;
}

// The loop shared by projection::match_current_and_last_frames, match_frame_and_keyframe,
// match_by_Sim3_transform and each direction of match_keyframes_mutually (match/projection.cc): for
// every usable query (a landmark reprojected into this frame by the caller) search the window
// [min_level, max_level] x margin for the nearest descriptor among the keypoints that are still
// available, accept it when the distance is <= hamm_dist_thr, mark the keypoint taken; finally drop
// the matches that disagree with the dominant rotation (angle_checker) when check_orientation.
extern "C" int ovs_projection_match_best_host(ovs_frame_index* f, int nq, const uint8_t* usable, const float* ref_xy, const float* ref_x_right,
                                              const float* margin, const int32_t* min_level, const int32_t* max_level, const float* q_angle,
                                              const uint8_t* q_desc, const uint8_t* kp_unavailable, unsigned hamm_dist_thr, int check_orientation,
                                              int32_t* matched_query_of_kp, int* num_matches) {
    OVS_REQUIRE(f && num_matches && matched_query_of_kp && nq >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(nq == 0 || (ref_xy && margin && min_level && max_level && q_desc && (!check_orientation || q_angle)), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(hamm_dist_thr <= OVS_MAX_HAMMING_DIST, OVS_ERR_INVALID_ARG, "hamm_dist_thr out of range");
    OVS_CUDA_CHECK(cudaSetDevice(f->m->device));
    const int n = f->n;
    for (int i = 0; i < n; ++i) matched_query_of_kp[i] = -1;
    *num_matches = 0;
    std::vector<int> ql; ql.reserve(nq);
    for (int i = 0; i < nq; ++i) if (!usable || usable[i]) ql.push_back(i);
    const int nu = (int)ql.size();
    if (nu == 0 || n == 0) return OVS_OK;
    std::vector<float> ref(2 * (size_t)nu), mg(nu), xr(nu); std::vector<int> lo(nu), hi(nu); std::vector<uint8_t> qd(32 * (size_t)nu);
    for (int q = 0; q < nu; ++q) {
        const int i = ql[q];
        ref[2 * q] = ref_xy[2 * i]; ref[2 * q + 1] = ref_xy[2 * i + 1];
        mg[q] = margin[i]; lo[q] = min_level[i]; hi[q] = max_level[i];
        xr[q] = ref_x_right ? ref_x_right[i] : -1.0f;
        memcpy(&qd[32 * (size_t)q], q_desc + 32 * (size_t)i, 32);
    }
    const bool use_xr = f->has_xr && ref_x_right != nullptr;
    std::vector<unsigned short> cap(std::max(n, 1), 0xffff);
    if (kp_unavailable) for (int i = 0; i < n; ++i) if (kp_unavailable[i]) cap[i] = 0;
    int rc;
    {
        std::vector<unsigned short> cap_rank((size_t)std::max(f->nranked, 1));
        for (int r = 0; r < f->nranked; ++r) cap_rank[r] = cap[f->rank_to_idx[r]];
        // without reprojected x_right the x_right test of the reference is not part of this matcher
        rc = window_topk(f, use_xr, nu, ref.data(), mg.data(), lo.data(), hi.data(), use_xr ? xr.data() : nullptr, qd.data(), cap_rank.data());
        if (rc != OVS_OK) return rc;
    }
    std::vector<unsigned> keys(f->m->h_keys, f->m->h_keys + (size_t)nu * kTopK);   // a re-query overwrites h_keys
    const auto decode = [&](unsigned key) { return f->rank_to_idx[key_rank(key)]; };
    const auto available = [&](int idx, int) { return cap[idx] != 0; };
    int nm = 0;
    ovs::OrientationCheck orientation;
    for (int q = 0; q < nu; ++q) {
        const auto requery_q = [&](unsigned* fresh) {
            return requery(f, use_xr, &ref[2 * q], mg[q], lo[q], hi[q], use_xr ? &xr[q] : nullptr, &qd[32 * (size_t)q], cap, fresh);
        };
        ovs::ReplayPick p;
        rc = ovs::replay_query<kTopK>(&keys[(size_t)q * kTopK], (int)hamm_dist_thr, ovs::kNeverComplete, decode, available, ovs::no_ratio_test,
                                      requery_q, &p);
        if (rc != OVS_OK) return rc;
        if (p.id < 0) continue;
        matched_query_of_kp[p.id] = ql[q]; cap[p.id] = 0; ++nm;
        if (check_orientation) orientation.add(q_angle[ql[q]] - f->hangle[p.id], p.id);
    }
    orientation.unset_invalid([&](int kp) { matched_query_of_kp[kp] = -1; --nm; });
    *num_matches = nm;
    return OVS_OK;
}

// match::projection::match_current_and_last_frames(curr_frm, last_frm, margin)
extern "C" int ovs_projection_match_current_and_last_host(ovs_frame_index* curr, const float* scale_factors, int num_scale_levels, int n_last,
                                                          const uint8_t* last_usable, const float* reproj_xy, const float* reproj_x_right,
                                                          const int32_t* last_scale_level, const float* last_angle, const uint8_t* lm_desc,
                                                          const uint8_t* kp_has_observed_lm, float margin, int assume_forward, int assume_backward,
                                                          int check_orientation, int32_t* matched_last_of_kp, int* num_matches) {
    OVS_REQUIRE(curr && scale_factors && num_matches && matched_last_of_kp && n_last >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n_last == 0 || (last_usable && reproj_xy && last_scale_level && lm_desc), OVS_ERR_INVALID_ARG, "null argument");
    std::vector<float> mg(std::max(n_last, 1)); std::vector<int32_t> lo(std::max(n_last, 1)), hi(std::max(n_last, 1));
    for (int i = 0; i < n_last; ++i) {
        const int lvl = last_scale_level[i];
        OVS_REQUIRE((last_usable && !last_usable[i]) || (lvl >= 0 && lvl < num_scale_levels), OVS_ERR_INVALID_ARG,
                    "scale level %d of last-frame keypoint %d outside the scale table (%d levels)", lvl, i, num_scale_levels);
        mg[i] = (lvl >= 0 && lvl < num_scale_levels) ? margin * scale_factors[lvl] : 0.0f;
        if (assume_forward) { lo[i] = lvl; hi[i] = num_scale_levels - 1; }
        else if (assume_backward) { lo[i] = 0; hi[i] = lvl; }
        else { lo[i] = lvl - 1; hi[i] = lvl + 1; }
    }
    // the reference applies the x_right test whenever the current keypoint has one; a NULL reproj_x_right means -1
    std::vector<float> xr;
    if (!reproj_x_right && curr->has_xr) { xr.assign(std::max(n_last, 1), -1.0f); reproj_x_right = xr.data(); }
    return ovs_projection_match_best_host(curr, n_last, last_usable, reproj_xy, reproj_x_right, mg.data(), lo.data(), hi.data(), last_angle, lm_desc,
                                          kp_has_observed_lm, OVS_HAMMING_DIST_THR_HIGH, check_orientation, matched_last_of_kp, num_matches);
}

// match::area::match_in_consistent_area(frm_1, frm_2, prev_matched_pts, matched_indices_2_in_frm_1, margin)
extern "C" int ovs_area_match_in_consistent_area_host(ovs_frame_index* f2, int n1, const int32_t* octave_1, const float* angle_1, const uint8_t* desc_1,
                                                      float* prev_matched_xy, int32_t* matched_idx_2_in_1, int margin, float lowe_ratio,
                                                      int check_orientation, int* num_matches) {
    OVS_REQUIRE(f2 && num_matches && n1 >= 0 && (n1 == 0 || (octave_1 && desc_1 && prev_matched_xy && matched_idx_2_in_1)), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(!check_orientation || angle_1 || n1 == 0, OVS_ERR_INVALID_ARG, "angles required for the orientation check");
    OVS_CUDA_CHECK(cudaSetDevice(f2->m->device));
    const ovs_frame_index* f = f2;
    const int n2 = f->n;
    for (int i = 0; i < n1; ++i) matched_idx_2_in_1[i] = -1;
    *num_matches = 0;
    std::vector<int> q1; q1.reserve(n1);
    for (int i = 0; i < n1; ++i) if (!(0 < octave_1[i])) q1.push_back(i);   // level-0 keypoints only
    const int nq = (int)q1.size();
    if (nq == 0 || n2 == 0) return OVS_OK;
    std::vector<float> ref(2 * (size_t)nq), mg(nq, (float)margin); std::vector<int> lo(nq), hi(nq); std::vector<uint8_t> qd(32 * (size_t)nq);
    for (int q = 0; q < nq; ++q) {
        const int i = q1[q];
        ref[2 * q] = prev_matched_xy[2 * i]; ref[2 * q + 1] = prev_matched_xy[2 * i + 1];
        lo[q] = octave_1[i]; hi[q] = octave_1[i];
        memcpy(&qd[32 * (size_t)q], desc_1 + 32 * (size_t)i, 32);
    }
    // the area matcher has no x_right test: a stereo frame's index searches here as a monocular one
    int rc = window_topk(f, false, nq, ref.data(), mg.data(), lo.data(), hi.data(), nullptr, qd.data(), nullptr);
    if (rc != OVS_OK) return rc;
    std::vector<unsigned> keys(f->m->h_keys, f->m->h_keys + (size_t)nq * kTopK);   // a re-query overwrites h_keys
    // matched_dists_in_frm_2 doubles as the per-keypoint distance cap (candidate valid iff d < cap)
    std::vector<unsigned short> cap(std::max(n2, 1), (unsigned short)OVS_MAX_HAMMING_DIST);
    std::vector<int> matched_idx_1_in_2(std::max(n2, 1), -1);
    const auto decode = [&](unsigned key) { return f->rank_to_idx[key_rank(key)]; };
    const auto closer = [&](int idx, int d) { return d < (int)cap[idx]; };
    const auto ratio = [&](const ovs::ReplayList<kTopK>& L, int second, ovs::Second) { return !((float)second * lowe_ratio < (float)L.dist[0]); };
    ovs::OrientationCheck orientation;
    int nm = 0;
    for (int q = 0; q < nq; ++q) {
        const int idx_1 = q1[q];
        const auto requery_q = [&](unsigned* fresh) {
            return requery(f, false, &ref[2 * q], mg[q], lo[q], hi[q], nullptr, &qd[32 * (size_t)q], cap, fresh);
        };
        ovs::ReplayPick p;
        rc = ovs::replay_query<kTopK>(&keys[(size_t)q * kTopK], OVS_HAMMING_DIST_THR_LOW, ovs::kNeverComplete, decode, closer, ratio, requery_q, &p);
        if (rc != OVS_OK) return rc;
        if (p.id < 0) continue;
        const int prev_idx_1 = matched_idx_1_in_2[p.id];
        if (0 <= prev_idx_1) { matched_idx_2_in_1[prev_idx_1] = -1; --nm; }
        matched_idx_2_in_1[idx_1] = p.id;
        matched_idx_1_in_2[p.id] = idx_1;
        cap[p.id] = (unsigned short)p.dist;
        ++nm;
        if (check_orientation) orientation.add(angle_1[idx_1] - f->hangle[p.id], idx_1);
    }
    orientation.unset_invalid([&](int i1) {
        if (0 <= matched_idx_2_in_1[i1]) { matched_idx_2_in_1[i1] = -1; --nm; }
    });
    for (int i = 0; i < n1; ++i)
        if (0 <= matched_idx_2_in_1[i]) { prev_matched_xy[2 * i] = f->hx[matched_idx_2_in_1[i]]; prev_matched_xy[2 * i + 1] = f->hy[matched_idx_2_in_1[i]]; }
    *num_matches = nm;
    return OVS_OK;
}

// match::stereo(left_pyr, right_pyr, ...).compute(stereo_x_right, depths); the pyramids are the
// device-resident image_pyramid_ of the two extractors (after their extract() of this stereo pair).
extern "C" int ovs_stereo_compute_host(ovs_matcher* m, const ovs_extractor* left, const ovs_extractor* right,
                                       int n_left, const float* lx, const float* ly, const int32_t* loct, const uint8_t* ldesc,
                                       int n_right, const float* rx, const float* ry, const int32_t* roct, const uint8_t* rdesc,
                                       float focal_x_baseline, float true_baseline, float* stereo_x_right, float* depths, int* num_matched) {
    OVS_REQUIRE(m && left && right && n_left >= 0 && n_right >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n_left == 0 || (lx && ly && loct && ldesc && stereo_x_right && depths), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(n_right == 0 || (rx && ry && roct && rdesc), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(n_right < 65535, OVS_ERR_UNSUPPORTED, "more than 65534 right keypoints");
    OVS_REQUIRE(true_baseline > 0, OVS_ERR_INVALID_ARG, "true_baseline must be positive");
    for (int i = 0; i < n_left; ++i) { stereo_x_right[i] = -1.0f; depths[i] = -1.0f; }
    if (num_matched) *num_matched = 0;
    if (n_left == 0 || n_right == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    StereoArgs A;
    memset(&A, 0, sizeof(A));
    float sf[16], isf[16];
    int rc = ovs_extractor_scale_factors(left, sf, isf, nullptr, nullptr);
    if (rc != OVS_OK) return rc;
    int L = 0;
    for (; L < 16; ++L) {
        const uint8_t *pl, *pr; size_t pitl, pitr; int wl, hl, wr, hr;
        if (ovs_extractor_pyramid_level(left, L, &pl, &pitl, &wl, &hl) != OVS_OK) break;
        if (ovs_extractor_pyramid_level(right, L, &pr, &pitr, &wr, &hr) != OVS_OK) break;
        OVS_REQUIRE(wl == wr && hl == hr && pitl == pitr, OVS_ERR_INVALID_ARG, "left/right pyramids differ at level %d", L);
        A.lpyr[L] = pl; A.rpyr[L] = pr; A.pw[L] = wl; A.ph[L] = hl; A.pitch[L] = (int)pitl; A.scale[L] = sf[L]; A.inv_scale[L] = isf[L];
    }
    OVS_REQUIRE(L > 0, OVS_ERR_INVALID_ARG, "extractors hold no pyramid (call extract first)");
    for (int i = 0; i < n_left; ++i) OVS_REQUIRE(loct[i] >= 0 && loct[i] < L, OVS_ERR_INVALID_ARG, "left octave out of range");
    for (int i = 0; i < n_right; ++i) OVS_REQUIRE(roct[i] >= 0 && roct[i] < L, OVS_ERR_INVALID_ARG, "right octave out of range");
    const size_t NL = (size_t)n_left, NR = (size_t)n_right;
    uint8_t *hld, *hrd; float *hlx, *hly, *hrx, *hry, *hxr, *hdp, *dxr, *ddp; int *hlo, *hro; unsigned *hco, *dco, *dbest;
    ovs::Staging S;
    rc = ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_t, m->d_t_cap, [&](ovs::Staging& S) {
        A.ldesc = (const uint4*)S.in(hld, 32 * NL); A.rdesc = (const uint4*)S.in(hrd, 32 * NR);
        A.lx = S.in(hlx, NL); A.ly = S.in(hly, NL); A.loct = S.in(hlo, NL); A.rx = S.in(hrx, NR); A.ry = S.in(hry, NR); A.roct = S.in(hro, NR);
        dxr = S.out(hxr, NL); ddp = S.out(hdp, NL); dco = S.out(hco, NL);
        dbest = S.dev<unsigned>(NL);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hld, ldesc, 32 * NL); memcpy(hrd, rdesc, 32 * NR);
    memcpy(hlx, lx, 4 * NL); memcpy(hly, ly, 4 * NL); memcpy(hlo, loct, 4 * NL);
    memcpy(hrx, rx, 4 * NR); memcpy(hry, ry, 4 * NR); memcpy(hro, roct, 4 * NR);
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    A.n_left = n_left; A.n_right = n_right;
    A.min_disp = 0.0f; A.max_disp = focal_x_baseline / true_baseline;
    A.hamm_thr = (OVS_HAMMING_DIST_THR_HIGH + OVS_HAMMING_DIST_THR_LOW) / 2;
    A.rows0 = A.ph[0]; A.focal_x_baseline = focal_x_baseline;
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_stereo_match<<<(n_left + 127) / 128, 128, 0, st>>>(A, dbest);
    OVS_LAUNCH_CHECK();
    k_stereo_subpixel<<<(n_left + 3) / 4, 128, 0, st>>>(A, dbest, dxr, ddp, dco);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    // median test on the SAD of the accepted matches (sorted (correlation, idx_left) pairs)
    std::vector<std::pair<unsigned, int>> corr;
    for (int i = 0; i < n_left; ++i) {
        if (hco[i] == 0xffffffffu) continue;
        stereo_x_right[i] = hxr[i]; depths[i] = hdp[i];
        corr.emplace_back(hco[i], i);
    }
    if (!corr.empty()) {
        std::sort(corr.begin(), corr.end());
        const float median = (float)corr[corr.size() / 2].first;
        const float thr = 2.0f * median;
        for (int k = (int)corr.size() - 1; k >= 0; --k) {
            if ((float)corr[k].first < thr) break;
            stereo_x_right[corr[k].second] = -1; depths[corr[k].second] = -1;
        }
    }
    if (num_matched) *num_matched = (int)corr.size();
    return OVS_OK;
}

// ====================================================================================================================
// match::robust::match_for_triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs) (match/robust.cc): BoW-node-guided
// candidate pairs + epipole and epipolar-plane tests.  The BoW feature vectors are inputs (bow_node_k[i] = vocabulary
// node of keypoint i); keyframe-2 keypoints are laid out node by node on the device, each eligible keyframe-1 keypoint is
// one query (one warp) over its node's segment.  The kernel returns the 8 best admissible candidates per query in the
// order the sequential loop prefers them (smallest distance; among equal distances the LAST one); the host replays the
// "a keyframe-2 keypoint is given to its first taker" rule and the orientation histogram.
namespace {

constexpr int kTriK = 8;

struct TriArgs {
    int nq;
    const uint4* qdesc;        // [nq][2]
    const double* qbearing;    // [nq][3]
    const float* qscale;       // [nq] scale factor of the keypoint's octave
    const unsigned char* qstereo;
    const int2* qseg;          // [nq] candidate rank range [begin, end)
    const uint4* tdesc;        // rank order (node major, index minor)
    const double* tbearing;
    const unsigned char* tstereo;
    double E[9];
    double epipole[3];
    // re-query of one keypoint whose candidate list was exhausted by earlier takers: queries [q0, nq) only, keyframe-2
    // keypoints with taken[rank] != 0 are skipped, results go to slot q + out_shift
    int q0, out_shift;
    const unsigned char* taken;   // [R] or null
    // several keyframe pairs in one launch (create_new_landmarks, k_triangulation_topk<true>): query q belongs to problem
    // p = q / queries_per_prob and reads keyframe-1 entry q - p * queries_per_prob, its problem's E_12 (prob_E[9 p]) and
    // epipole (prob_epipole[3 p]), and the keyframe-2 arrays (and taken) from entry prob_tbase[p] on; ranks stay per problem
    int queries_per_prob;
    const double* prob_E;
    const double* prob_epipole;
    const int* prob_tbase;
};

__device__ __forceinline__ bool epipolar_inlier(const double* E, const double b1x, const double b1y, const double b1z, const double b2x,
                                                const double b2y, const double b2z, const float scale) {
    const double ex = E[0] * b2x + E[1] * b2y + E[2] * b2z;
    const double ey = E[3] * b2x + E[4] * b2y + E[5] * b2z;
    const double ez = E[6] * b2x + E[7] * b2y + E[8] * b2z;
    const double norm = sqrt(ex * ex + ey * ey + ez * ez);
    const double cos_residual = (ex * b1x + ey * b1y + ez * b1z) / norm;
    const double residual_rad = 3.14159265358979323846 / 2.0 - fabs(acos(cos_residual));
    const double thr = 0.2 * 3.14159265358979323846 / 180.0;
    return residual_rad < thr * (double)scale;
}

// one warp per query; keys = distance << 16 | (0xffff - rank): ascending order = the sequential loop's preference
template <bool kBatched>
__global__ void __launch_bounds__(128) k_triangulation_topk(TriArgs A, unsigned* __restrict__ keys_out) {
    const int q = A.q0 + blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= A.nq) return;
    int qk = q;
    const double* E = A.E;
    const double* epipole = A.epipole;
    const uint4* tdesc = A.tdesc;
    const double* tbearing = A.tbearing;
    const unsigned char* tstereo = A.tstereo;
    const unsigned char* taken = A.taken;
    if (kBatched) {
        const int p = q / A.queries_per_prob, base = A.prob_tbase[p];
        qk = q - p * A.queries_per_prob;
        E = A.prob_E + 9 * (size_t)p; epipole = A.prob_epipole + 3 * (size_t)p;
        tdesc += 2 * (size_t)base; tbearing += 3 * (size_t)base; tstereo += base;
        if (taken) taken += base;
    }
    const uint4 qa = A.qdesc[2 * (size_t)qk], qb = A.qdesc[2 * (size_t)qk + 1];
    const double b1x = A.qbearing[3 * (size_t)qk], b1y = A.qbearing[3 * (size_t)qk + 1], b1z = A.qbearing[3 * (size_t)qk + 2];
    const float scale = A.qscale[qk];
    const bool stereo_1 = A.qstereo[qk] != 0;
    const int2 seg = A.qseg[q];
    unsigned extra = 0xffffffffu;   // lane r < 8 carries entry r of the running top-8 from one chunk of candidates to the next
    for (int c0 = seg.x; c0 < seg.y; c0 += 32 * kTriK) {
        // each lane evaluates up to kTriK candidates of this chunk
        unsigned mine[kTriK];
#pragma unroll
        for (int k = 0; k < kTriK; ++k) {
            mine[k] = 0xffffffffu;
            const int c = c0 + k * 32 + lane;
            if (c < seg.y && !(taken && taken[c])) {
                const uint4 ta = tdesc[2 * (size_t)c], tb = tdesc[2 * (size_t)c + 1];
                const int d = hamming256(qa, qb, ta, tb);
                if (d <= OVS_HAMMING_DIST_THR_LOW) {
                    const double b2x = tbearing[3 * (size_t)c], b2y = tbearing[3 * (size_t)c + 1], b2z = tbearing[3 * (size_t)c + 2];
                    bool ok = true;
                    if (!stereo_1 && !tstereo[c]) {
                        const double cos_dist = epipole[0] * b2x + epipole[1] * b2y + epipole[2] * b2z;
                        if (0.998 < cos_dist) ok = false;
                    }
                    if (ok && epipolar_inlier(E, b1x, b1y, b1z, b2x, b2y, b2z, scale)) mine[k] = ((unsigned)d << 16) | (0xffffu - (unsigned)c);
                }
            }
        }
        extra = warp_merge_topk(extra, mine, lane);
    }
    if (lane < kTriK) keys_out[(size_t)(q + A.out_shift) * kTriK + lane] = extra;
}

// The keypoints of a keyframe that take part (keep(i), a vocabulary node), node by node and in index order inside a node:
// the reference's walk over the BoW feature vector.
template <class Keep>
void node_order(int n, const int32_t* bow_node, Keep&& keep, std::vector<int>& out) {
    out.clear();
    for (int i = 0; i < n; ++i) if (keep(i) && bow_node[i] >= 0) out.push_back(i);
    std::stable_sort(out.begin(), out.end(), [&](int a, int b) { return bow_node[a] < bow_node[b]; });
}

// seg[k] = the range of rank2 in the node of query q1[k]
void node_segments(const std::vector<int>& q1, const int32_t* bow_node_1, const std::vector<int>& rank2, const int32_t* bow_node_2, int2* seg) {
    size_t lo = 0;
    for (size_t k = 0; k < q1.size(); ++k) {
        const int node = bow_node_1[q1[k]];
        while (lo < rank2.size() && bow_node_2[rank2[lo]] < node) ++lo;
        size_t hi = lo;
        while (hi < rank2.size() && bow_node_2[rank2[hi]] == node) ++hi;
        seg[k] = make_int2((int)lo, (int)hi);
    }
}

// The sequential part of match_for_triangulation on one keyframe pair, given each query's candidate list (keys[kTriK k]): the
// queries k = 0 .. Q - 1 (keyframe-1 keypoint q1[k], in the reference's visiting order; skipped where skip_1[q1[k]] is set, as
// a keypoint that holds a landmark is no query) each take the first listed candidate not taken yet (taken[rank], all zero on
// entry).  The device already applied the distance and epipolar tests, so there is no threshold and no ratio test: only a
// list of kTriK entries that are all taken may be truncated, and then requery(k, keys) asks the device again with the taken
// candidates excluded (rare: needs 8 earlier keypoints of the same node to have claimed them).  Then the orientation
// histogram, if requested.  matched_idx_2_of_1[n1] (all -1 on entry) gets rank2[rank] of each match; slot_of_1 (may be null)
// the list entry kTriK k + j it came from, or -1 - k for a re-query.
template <class Requery>
int tri_replay(int Q, const int* q1, const int* rank2, const unsigned* keys, unsigned char* taken, const uint8_t* skip_1,
               const float* angle_1, const float* angle_2, int check_orientation, Requery&& requery, int32_t* matched_idx_2_of_1,
               int32_t* slot_of_1, int* num_matches) {
    const auto decode = [](unsigned key) { return 0xffff - (int)(key & 0xffffu); };
    const auto not_taken = [&](int r, int) { return !taken[r]; };
    ovs::OrientationCheck orientation;
    int num = 0;
    for (int k = 0; k < Q; ++k) {
        const int i1 = q1[k];
        if (skip_1 && skip_1[i1]) continue;
        ovs::ReplayPick p;
        const int rc = ovs::replay_query<kTriK>(keys + (size_t)k * kTriK, OVS_MAX_HAMMING_DIST, ovs::kNeverComplete, decode, not_taken,
                                                ovs::no_ratio_test, [&](unsigned* fresh) { return requery(k, fresh); }, &p);
        if (rc != OVS_OK) return rc;
        if (p.id < 0) continue;
        taken[p.id] = 1;
        matched_idx_2_of_1[i1] = rank2[p.id];
        if (slot_of_1) slot_of_1[i1] = p.requeried ? -1 - k : kTriK * k + p.pos;
        ++num;
        if (check_orientation) orientation.add(angle_1[i1] - angle_2[rank2[p.id]], i1);
    }
    orientation.unset_invalid([&](int i1) { matched_idx_2_of_1[i1] = -1; --num; });
    *num_matches = num;
    return OVS_OK;
}

}  // namespace

extern "C" int ovs_robust_match_for_triangulation_host(ovs_matcher* m, int n1, const uint8_t* desc_1, const double* bearing_1, const int32_t* octave_1,
                                                       const float* angle_1, const uint8_t* has_lm_1, const uint8_t* is_stereo_1,
                                                       const int32_t* bow_node_1, int n2, const uint8_t* desc_2, const double* bearing_2,
                                                       const float* angle_2, const uint8_t* has_lm_2, const uint8_t* is_stereo_2,
                                                       const int32_t* bow_node_2, const double* E_12, const double* epipole_in_2,
                                                       const float* scale_factors_1, int num_scale_levels, int check_orientation,
                                                       int32_t* matched_idx_2_of_1, int* num_matches) {
    OVS_REQUIRE(m && E_12 && epipole_in_2 && scale_factors_1 && matched_idx_2_of_1 && num_matches && n1 >= 0 && n2 >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n1 == 0 || (desc_1 && bearing_1 && octave_1 && angle_1 && has_lm_1 && bow_node_1), OVS_ERR_INVALID_ARG, "null keyframe-1 array");
    OVS_REQUIRE(n2 == 0 || (desc_2 && bearing_2 && angle_2 && has_lm_2 && bow_node_2), OVS_ERR_INVALID_ARG, "null keyframe-2 array");
    OVS_REQUIRE(n2 < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 keypoints");
    *num_matches = 0;
    for (int i = 0; i < n1; ++i) matched_idx_2_of_1[i] = -1;
    if (n1 == 0 || n2 == 0) return OVS_OK;
    for (int i = 0; i < n1; ++i)
        OVS_REQUIRE(octave_1[i] >= 0 && octave_1[i] < num_scale_levels, OVS_ERR_INVALID_ARG, "octave %d of keypoint %d outside the scale table", octave_1[i], i);
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    // keyframe 2: candidates; keyframe 1: queries in the order the reference visits them
    std::vector<int> rank2, q1;
    node_order(n2, bow_node_2, [&](int i) { return !has_lm_2[i]; }, rank2);
    node_order(n1, bow_node_1, [&](int i) { return !has_lm_1[i]; }, q1);
    const int R = (int)rank2.size(), Q = (int)q1.size();
    if (R == 0 || Q == 0) return OVS_OK;
    std::vector<int2> seg(Q);
    node_segments(q1, bow_node_1, rank2, bow_node_2, seg.data());
    const size_t sQ = (size_t)Q, sR = (size_t)R;
    TriArgs A{};
    uint8_t *hqd, *htd, *hq8, *ht8, *taken, *dtaken; double *hqb, *htb; int2* hsg; float* hqs;
    ovs::Staging S;
    int rc = ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_q, m->d_q_cap, [&](ovs::Staging& S) {
        A.qdesc = (const uint4*)S.in(hqd, 32 * sQ); A.tdesc = (const uint4*)S.in(htd, 32 * sR);
        A.qbearing = S.in(hqb, 3 * sQ); A.tbearing = S.in(htb, 3 * sR); A.qseg = S.in(hsg, sQ); A.qscale = S.in(hqs, sQ);
        A.qstereo = S.in(hq8, sQ); A.tstereo = S.in(ht8, sR);
        dtaken = S.out(taken, sR);   // uploaded a node's slice at a time by the re-queries
    });
    if (rc != OVS_OK) return rc;
    if ((rc = ovs::grow_dev(&m->d_keys, &m->d_keys_cap, (size_t)(Q + 1) * kTriK)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&m->h_keys, &m->h_keys_cap, (size_t)(Q + 1) * kTriK)) != OVS_OK) return rc;
    for (int k = 0; k < Q; ++k) {
        const int i = q1[k];
        memcpy(hqd + 32 * (size_t)k, desc_1 + 32 * (size_t)i, 32);
        memcpy(hqb + 3 * (size_t)k, bearing_1 + 3 * (size_t)i, 24);
        hqs[k] = scale_factors_1[octave_1[i]];
        hsg[k] = seg[k];
        hq8[k] = is_stereo_1 ? is_stereo_1[i] : 0;
    }
    for (int r = 0; r < R; ++r) {
        const int i = rank2[r];
        memcpy(htd + 32 * (size_t)r, desc_2 + 32 * (size_t)i, 32);
        memcpy(htb + 3 * (size_t)r, bearing_2 + 3 * (size_t)i, 24);
        ht8[r] = is_stereo_2 ? is_stereo_2[i] : 0;
    }
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    A.nq = Q;
    for (int k = 0; k < 9; ++k) A.E[k] = E_12[k];
    for (int k = 0; k < 3; ++k) A.epipole[k] = epipole_in_2[k];
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_triangulation_topk<false><<<(Q + 3) / 4, 128, 0, st>>>(A, m->d_keys);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys, m->d_keys, (size_t)Q * kTriK * 4, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    // the flags live in the pinned staging area so that a re-query can upload the slice of a node
    memset(taken, 0, (size_t)R);
    auto requery = [&](int k, unsigned* fresh) -> int {
        ++m->num_requeries;
        const size_t len = (size_t)(seg[k].y - seg[k].x);
        OVS_CUDA_CHECK(cudaMemcpyAsync(dtaken + seg[k].x, taken + seg[k].x, len, cudaMemcpyHostToDevice, st));
        TriArgs B = A;
        B.q0 = k; B.nq = k + 1; B.out_shift = Q - k; B.taken = dtaken;
        k_triangulation_topk<false><<<1, 128, 0, st>>>(B, m->d_keys);
        OVS_LAUNCH_CHECK();
        OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys + (size_t)Q * kTriK, m->d_keys + (size_t)Q * kTriK, kTriK * 4, cudaMemcpyDeviceToHost, st));
        OVS_CUDA_CHECK(ovs::sync_stream(st));
        memcpy(fresh, m->h_keys + (size_t)Q * kTriK, kTriK * 4);
        return OVS_OK;
    };
    return tri_replay(Q, q1.data(), rank2.data(), m->h_keys, taken, nullptr, angle_1, angle_2, check_orientation, requery,
                      matched_idx_2_of_1, nullptr, num_matches);
}

// mapping_module::create_new_landmarks' compute step (ovs_b200.h): the candidate lists of every (neighbour, query) in one launch
// and the triangulation of every listed candidate in another (a list does not depend on the other queries and a pair's
// triangulation only on keyframe data), then the neighbour-by-neighbour replay on the host, where a keyframe-1 keypoint that got a
// landmark from an earlier neighbour is no query any more, and one gather of the chosen points.
extern "C" int ovs_create_new_landmarks_host(ovs_matcher* m, const ovs_keyframe_view* keyfrm_1, int B, const ovs_keyframe_view* keyfrms_2,
                                             const double* E_12, const double* epipole_in_2, int check_orientation, double rays_parallax_deg_thr,
                                             ovs_new_landmark* out, int capacity, int* num_out) {
    OVS_REQUIRE(m && num_out && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    int rc;
    double cos_thr;
    if ((rc = ovs::tri_cos_thr(rays_parallax_deg_thr, &cos_thr)) != OVS_OK) return rc;
    if ((rc = ovs::check_keyframe_view(keyfrm_1, true, "keyframe", 1)) != OVS_OK) return rc;
    const ovs_keyframe_view& K1 = *keyfrm_1;
    const int n1 = K1.num_keypts;
    OVS_REQUIRE(capacity >= n1 && (n1 == 0 || out), OVS_ERR_CAPACITY, "capacity %d below the %d keypoints of keyframe 1", capacity, n1);
    OVS_REQUIRE(B == 0 || (keyfrms_2 && E_12 && epipole_in_2), OVS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n1; ++i)
        if ((rc = ovs::check_tri_keypt(K1, i, "keyframe", 1)) != OVS_OK) return rc;
    for (int b = 0; b < B; ++b) {
        const ovs_keyframe_view& K2 = keyfrms_2[b];
        if ((rc = ovs::check_keyframe_view(&K2, true, "neighbour", b)) != OVS_OK) return rc;
        OVS_REQUIRE(K2.num_keypts < 65536, OVS_ERR_UNSUPPORTED, "neighbour %d has more than 65535 keypoints", b);
        for (int i = 0; i < K2.num_keypts; ++i)
            if ((rc = ovs::check_tri_keypt(K2, i, "neighbour", b)) != OVS_OK) return rc;
        for (int k = 0; k < 9; ++k) OVS_REQUIRE(std::isfinite(E_12[9 * (size_t)b + k]), OVS_ERR_INVALID_ARG, "E_12 of neighbour %d is not finite", b);
        for (int k = 0; k < 3; ++k)
            OVS_REQUIRE(std::isfinite(epipole_in_2[3 * (size_t)b + k]), OVS_ERR_INVALID_ARG, "epipole of neighbour %d is not finite", b);
    }
    *num_out = 0;
    std::vector<int> q1;
    node_order(n1, K1.bow_node, [&](int i) { return !K1.has_landmark[i]; }, q1);
    const int Q = (int)q1.size();
    std::vector<std::vector<int>> rank2((size_t)B);
    std::vector<int> tbase((size_t)B + 1, 0);
    for (int b = 0; b < B; ++b) {
        node_order(keyfrms_2[b].num_keypts, keyfrms_2[b].bow_node, [&](int i) { return !keyfrms_2[b].has_landmark[i]; }, rank2[b]);
        tbase[b + 1] = tbase[b] + (int)rank2[b].size();
    }
    const int R = tbase[B];
    // every (neighbour, query) has a list of kTriK slots, plus one re-query slot: the slot index of the kernels is an int
    OVS_REQUIRE(((int64_t)B * Q + 1) * kTriK <= INT32_MAX, OVS_ERR_UNSUPPORTED,
                "%d neighbours x %d queries: more candidate slots than one call holds (2^31 - 1)", B, Q);
    if (Q == 0 || R == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    // queries of all neighbours, then one re-query slot; keypoint records: the Q queries of keyframe 1, then every candidate
    const size_t sQ = (size_t)Q, sR = (size_t)R, NB = (size_t)B, NQ = NB * sQ, NS = (NQ + 1) * kTriK;
    TriArgs A{};
    ovs::TriLaunch L{};
    uint8_t *hqd, *htd, *hq8, *ht8, *taken, *dtaken, *hvalid; double *hqb, *htb, *hE, *hep, *hrq, *drq, *hgpos, *dgpos; int2* hsg;
    float* hqs; int *htb0, *hchosen, *dchosen; unsigned* hkeys; unsigned* dkeys; ovs::TriProblem* hprob; ovs::TriKeypt* hkp;
    ovs::Staging S;
    rc = ovs::stage(S, m->h_tri, m->h_tri_cap, m->d_tri, m->d_tri_cap, [&](ovs::Staging& S) {
        A.qdesc = (const uint4*)S.in(hqd, 32 * sQ); A.tdesc = (const uint4*)S.in(htd, 32 * sR);
        A.qbearing = S.in(hqb, 3 * sQ); A.tbearing = S.in(htb, 3 * sR); A.qseg = S.in(hsg, NQ); A.qscale = S.in(hqs, sQ);
        A.qstereo = S.in(hq8, sQ); A.tstereo = S.in(ht8, sR);
        A.prob_E = S.in(hE, 9 * NB); A.prob_epipole = S.in(hep, 3 * NB); A.prob_tbase = S.in(htb0, NB);
        L.prob = S.in(hprob, NB); L.kp = S.in(hkp, sQ + sR); L.rank_base = A.prob_tbase;
        dkeys = S.out(hkeys, NS); L.valid = S.out(hvalid, NS);
        // host and device halves of the replay's own transfers, each copied explicitly when it is needed (the lists' download
        // below stops before them): the taken flags (a node's slice per re-query), a re-query's point, the gather's slots and points
        dtaken = S.out(taken, sR);
        drq = S.out(hrq, 3);
        dchosen = S.out(hchosen, (size_t)n1); dgpos = S.out(hgpos, 3 * (size_t)n1);
        L.pos = S.dev<double>(3 * NS);
    });
    if (rc != OVS_OK) return rc;
    for (int k = 0; k < Q; ++k) {
        const int i = q1[k];
        memcpy(hqd + 32 * (size_t)k, K1.descriptors + 32 * (size_t)i, 32);
        memcpy(hqb + 3 * (size_t)k, K1.bearings + 3 * (size_t)i, 24);
        hqs[k] = K1.scale_factors[K1.undist_keypts[i].octave];
        hq8[k] = K1.stereo_x_right && 0.0f <= K1.stereo_x_right[i];
        hkp[k] = ovs::tri_keypt(K1, i);
    }
    for (int b = 0; b < B; ++b) {
        const ovs_keyframe_view& K2 = keyfrms_2[b];
        const std::vector<int>& rk = rank2[b];
        for (size_t r = 0; r < rk.size(); ++r) {
            const int i = rk[r];
            const size_t g = (size_t)tbase[b] + r;
            memcpy(htd + 32 * g, K2.descriptors + 32 * (size_t)i, 32);
            memcpy(htb + 3 * g, K2.bearings + 3 * (size_t)i, 24);
            ht8[g] = K2.stereo_x_right && 0.0f <= K2.stereo_x_right[i];
            hkp[sQ + g] = ovs::tri_keypt(K2, i);
        }
        node_segments(q1, K1.bow_node, rk, K2.bow_node, hsg + sQ * b);
        memcpy(hE + 9 * b, E_12 + 9 * (size_t)b, 72); memcpy(hep + 3 * b, epipole_in_2 + 3 * (size_t)b, 24);
        htb0[b] = tbase[b];
        hprob[b].c[0] = ovs::tri_cam(K1); hprob[b].c[1] = ovs::tri_cam(K2);
        hprob[b].ratio_factor = 1.5f * K1.scale_factor;
    }
    A.nq = (int)NQ; A.queries_per_prob = Q;
    L.n = (int)(NQ * kTriK); L.cos_thr = cos_thr; L.keys = dkeys; L.queries_per_prob = Q; L.fixed_prob = -1; L.rec_2_base = Q;
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_triangulation_topk<true><<<(A.nq + 3) / 4, 128, 0, st>>>(A, dkeys);
    OVS_LAUNCH_CHECK();
    if ((rc = ovs::launch_two_view_triangulate(L, st)) != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    // the keys and the valid flags, carved one after the other: one copy
    const size_t list_bytes = (size_t)((const uint8_t*)(hvalid + NS) - (const uint8_t*)hkeys);
    OVS_CUDA_CHECK(cudaMemcpyAsync(hkeys, dkeys, list_bytes, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;

    std::vector<uint8_t> got((size_t)n1, 0);           // keyframe-1 keypoints that got a landmark in this call
    std::vector<int32_t> match((size_t)n1), slot((size_t)n1);
    std::vector<float> angle_1((size_t)n1), angle_2;
    for (int i = 0; i < n1; ++i) angle_1[i] = K1.undist_keypts[i].angle;
    std::vector<int> list_rec;                           // records whose point comes from a list slot, in record order
    int num = 0;
    for (int b = 0; b < B; ++b) {
        const ovs_keyframe_view& K2 = keyfrms_2[b];
        const size_t qoff = sQ * b;
        std::vector<double> rq_pos((size_t)3 * Q);       // a re-queried pair's point, by query
        std::vector<uint8_t> rq_valid((size_t)Q, 0);
        auto requery = [&](int k, unsigned* fresh) -> int {
            ++m->num_requeries;
            const int2 sg = hsg[qoff + k];
            OVS_CUDA_CHECK(cudaMemcpyAsync(dtaken + tbase[b] + sg.x, taken + tbase[b] + sg.x, (size_t)(sg.y - sg.x), cudaMemcpyHostToDevice, st));
            TriArgs Aq = A;
            Aq.q0 = (int)qoff + k; Aq.nq = Aq.q0 + 1; Aq.out_shift = (int)NQ - Aq.q0; Aq.taken = dtaken;
            k_triangulation_topk<true><<<1, 128, 0, st>>>(Aq, dkeys);
            OVS_LAUNCH_CHECK();
            ovs::TriLaunch Lq = L;
            Lq.n = 1; Lq.keys = dkeys + NQ * kTriK; Lq.fixed_prob = b; Lq.fixed_query = k; Lq.valid = L.valid + NQ * kTriK; Lq.pos = drq;
            const int rc2 = ovs::launch_two_view_triangulate(Lq, st);
            if (rc2 != OVS_OK) return rc2;
            OVS_CUDA_CHECK(cudaMemcpyAsync(hkeys + NQ * kTriK, dkeys + NQ * kTriK, kTriK * 4, cudaMemcpyDeviceToHost, st));
            OVS_CUDA_CHECK(cudaMemcpyAsync(hvalid + NQ * kTriK, L.valid + NQ * kTriK, 1, cudaMemcpyDeviceToHost, st));
            OVS_CUDA_CHECK(cudaMemcpyAsync(hrq, drq, 24, cudaMemcpyDeviceToHost, st));
            OVS_CUDA_CHECK(ovs::sync_stream(st));
            memcpy(fresh, hkeys + NQ * kTriK, kTriK * 4);
            rq_valid[k] = hvalid[NQ * kTriK];
            for (int c = 0; c < 3; ++c) rq_pos[3 * (size_t)k + c] = hrq[c];
            return OVS_OK;
        };
        angle_2.resize((size_t)K2.num_keypts);
        for (int i = 0; i < K2.num_keypts; ++i) angle_2[i] = K2.undist_keypts[i].angle;
        memset(taken + tbase[b], 0, rank2[b].size());
        std::fill(match.begin(), match.end(), -1);
        int nm = 0;
        if ((rc = tri_replay(Q, q1.data(), rank2[b].data(), hkeys + qoff * kTriK, taken + tbase[b], got.data(), angle_1.data(),
                             angle_2.data(), check_orientation, requery, match.data(), slot.data(), &nm)) != OVS_OK)
            return rc;
        // triangulate_with_two_keyframes: the pairs in idx_1 order
        for (int i1 = 0; i1 < n1; ++i1) {
            if (match[i1] < 0) continue;
            const int sl = slot[i1];
            if (!(sl >= 0 ? hvalid[qoff * kTriK + sl] : rq_valid[-1 - sl])) continue;
            ovs_new_landmark& r = out[num];
            r.neighbour = b; r.idx_1 = i1; r.idx_2 = match[i1]; r.reserved = 0;
            if (sl >= 0) {
                hchosen[list_rec.size()] = (int)(qoff * kTriK) + sl;
                list_rec.push_back(num);
            } else {
                for (int c = 0; c < 3; ++c) r.pos_w[c] = rq_pos[3 * (size_t)(-1 - sl) + c];
            }
            got[i1] = 1;
            ++num;
        }
    }
    const int nc = (int)list_rec.size();
    if (nc > 0) {
        OVS_CUDA_CHECK(cudaMemcpyAsync(dchosen, hchosen, 4 * (size_t)nc, cudaMemcpyHostToDevice, st));
        if ((rc = ovs::launch_gather_pos(nc, dchosen, L.pos, dgpos, st)) != OVS_OK) return rc;
        OVS_CUDA_CHECK(cudaMemcpyAsync(hgpos, dgpos, 24 * (size_t)nc, cudaMemcpyDeviceToHost, st));
        OVS_CUDA_CHECK(ovs::sync_stream(st));
        for (int j = 0; j < nc; ++j)
            for (int c = 0; c < 3; ++c) out[list_rec[j]].pos_w[c] = hgpos[3 * (size_t)j + c];
    }
    *num_out = num;
    return OVS_OK;
}

// ============================================================================ match::bow_tree
// match::bow_tree::{match_frame_and_keyframe, match_keyframes} (match/bow_tree.cc): the BoW feature vectors are inputs
// (per-keypoint vocabulary node ids, < 0 = none).  Nodes ascending, keypoints of a node in index order -- the lock-step walk
// over the two std::map<NodeId, std::vector<unsigned>> -- every query keypoint takes its nearest candidate of the same
// node that is still free, subject to HAMMING_DIST_THR_LOW and the ratio test against the second nearest free candidate.
// k_node_topk gives, per query, the 8 best (distance, visiting order) candidates of its node; the host replays the
// sequential first-taker rule on those lists and re-queries the GPU (claimed candidates excluded) only when a list cannot
// decide: the same scheme as robust::brute_force_match.
namespace {

constexpr int kNodeK = 8;

struct NodeArgs {
    int nq, q0, out_shift;
    const uint4* qdesc;            // [nq][2], visiting order
    const int2* qseg;              // [nq] candidate rank range [begin, end)
    const uint4* tdesc;            // rank order (node major, index minor)
    const unsigned char* taken;    // [R] or null
};

// one warp per query; keys = distance << 16 | rank: ascending order = the sequential loop's preference (strict '<': first wins)
__global__ void __launch_bounds__(128) k_node_topk(NodeArgs A, unsigned* __restrict__ keys_out) {
    const int q = A.q0 + blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= A.nq) return;
    const uint4 qa = A.qdesc[2 * (size_t)q], qb = A.qdesc[2 * (size_t)q + 1];
    const int2 seg = A.qseg[q];
    unsigned extra = 0xffffffffu;   // lane r < 8 carries entry r of the running top-8 from one chunk of candidates to the next
    for (int c0 = seg.x; c0 < seg.y; c0 += 32 * kNodeK) {
        unsigned mine[kNodeK];
#pragma unroll
        for (int k = 0; k < kNodeK; ++k) {
            mine[k] = 0xffffffffu;
            const int c = c0 + k * 32 + lane;
            if (c < seg.y && !(A.taken && A.taken[c])) {
                const uint4 ta = A.tdesc[2 * (size_t)c], tb = A.tdesc[2 * (size_t)c + 1];
                mine[k] = ((unsigned)hamming256(qa, qb, ta, tb) << 16) | (unsigned)c;
            }
        }
        extra = warp_merge_topk(extra, mine, lane);
    }
    if (lane < kNodeK) keys_out[(size_t)(q + A.out_shift) * kNodeK + lane] = extra;
}

// queries A (valid_a[i] != 0, node >= 0), candidates B (valid_b null or != 0, node >= 0): match_b_of_a[i] = index in B or -1
int bow_core(ovs_matcher* m, int na, const uint8_t* desc_a, const uint8_t* valid_a, const int32_t* node_a,
             int nb, const uint8_t* desc_b, const uint8_t* valid_b, const int32_t* node_b, float lowe_ratio,
             std::vector<int>& match_b_of_a, std::vector<int>& visit_order) {
    match_b_of_a.assign(std::max(na, 1), -1);
    visit_order.clear();
    if (na == 0 || nb == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    std::vector<int> rankb, qa;
    node_order(nb, node_b, [&](int i) { return !valid_b || valid_b[i]; }, rankb);
    node_order(na, node_a, [&](int i) { return !valid_a || valid_a[i]; }, qa);
    const int R = (int)rankb.size(), Q = (int)qa.size();
    if (R == 0 || Q == 0) return OVS_OK;
    OVS_REQUIRE(R < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 candidate keypoints");
    std::vector<int2> seg(Q);
    node_segments(qa, node_a, rankb, node_b, seg.data());
    NodeArgs A{};
    uint8_t *hqd, *htd, *taken, *dtaken; int2* hsg;
    ovs::Staging S;
    int rc = ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_q, m->d_q_cap, [&](ovs::Staging& S) {
        A.qdesc = (const uint4*)S.in(hqd, 32 * (size_t)Q); A.tdesc = (const uint4*)S.in(htd, 32 * (size_t)R); A.qseg = S.in(hsg, (size_t)Q);
        dtaken = S.out(taken, (size_t)R);   // uploaded a node's slice at a time by the re-queries
    });
    if (rc != OVS_OK) return rc;
    if ((rc = ovs::grow_dev(&m->d_keys, &m->d_keys_cap, (size_t)(Q + 1) * kNodeK)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&m->h_keys, &m->h_keys_cap, (size_t)(Q + 1) * kNodeK)) != OVS_OK) return rc;
    for (int k = 0; k < Q; ++k) {
        memcpy(hqd + 32 * (size_t)k, desc_a + 32 * (size_t)qa[k], 32);
        hsg[k] = seg[k];
    }
    for (int r = 0; r < R; ++r) memcpy(htd + 32 * (size_t)r, desc_b + 32 * (size_t)rankb[r], 32);
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    A.nq = Q;
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[0], st));
    k_node_topk<<<(Q + 3) / 4, 128, 0, st>>>(A, m->d_keys);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(m->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys, m->d_keys, (size_t)Q * kNodeK * 4, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    float ms = 0; cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]);
    m->last_kernel_us = ms * 1000.f;
    memset(taken, 0, (size_t)R);
    const auto decode = [](unsigned key) { return (int)(key & 0xffffu); };
    const auto not_taken = [&](int r, int) { return !taken[r]; };
    const auto ratio = [&](const ovs::ReplayList<kNodeK>& L, int second, ovs::Second) { return !(lowe_ratio * (float)(unsigned)second < (float)L.dist[0]); };
    const int complete_at = ovs::d_star(lowe_ratio);
    for (int k = 0; k < Q; ++k) {
        // the re-query's list goes to the spare row Q
        const auto requery = [&](unsigned* fresh) -> int {
            ++m->num_requeries;
            const size_t len = (size_t)(seg[k].y - seg[k].x);
            OVS_CUDA_CHECK(cudaMemcpyAsync(dtaken + seg[k].x, taken + seg[k].x, len, cudaMemcpyHostToDevice, st));
            NodeArgs B = A;
            B.q0 = k; B.nq = k + 1; B.out_shift = Q - k; B.taken = dtaken;
            k_node_topk<<<1, 128, 0, st>>>(B, m->d_keys);
            OVS_LAUNCH_CHECK();
            OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys + (size_t)Q * kNodeK, m->d_keys + (size_t)Q * kNodeK, kNodeK * 4, cudaMemcpyDeviceToHost, st));
            OVS_CUDA_CHECK(ovs::sync_stream(st));
            memcpy(fresh, m->h_keys + (size_t)Q * kNodeK, kNodeK * 4);
            return OVS_OK;
        };
        ovs::ReplayPick p;
        rc = ovs::replay_query<kNodeK>(m->h_keys + (size_t)k * kNodeK, OVS_HAMMING_DIST_THR_LOW, complete_at, decode, not_taken, ratio, requery, &p);
        if (rc != OVS_OK) return rc;
        if (p.id < 0) continue;
        taken[p.id] = 1;
        match_b_of_a[qa[k]] = rankb[p.id];
        visit_order.push_back(qa[k]);
    }
    return OVS_OK;
}

// Candidate segments [seg[2 k], seg[2 k + 1]) of the test hooks below, each inside [0, R - base[k / per_prob]).
int check_segments(int nq, const int32_t* seg, int R, const int32_t* base, int per_prob) {
    for (int k = 0; k < nq; ++k) {
        const int b = base ? base[k / per_prob] : 0;
        OVS_REQUIRE(0 <= seg[2 * k] && seg[2 * k] <= seg[2 * k + 1] && b + seg[2 * k + 1] <= R, OVS_ERR_INVALID_ARG,
                    "segment of query %d outside the %d candidates", k, R);
    }
    return OVS_OK;
}

}  // namespace

// Development aid / test hook: k_node_topk on host arrays, with bow_core's launch geometry and buffers.  q0 < 0: the list launch over
// all nq queries, taken (null: none) applied to every query, keys_out[nq * 8].  q0 >= 0: the list launch without taken, then
// bow_core's re-query of query q0 alone with taken, its list in the spare row nq, keys_out[(nq + 1) * 8].  Every key slot is filled
// with 0x5a5a5a5a first, so a slot the kernels leave unwritten shows.  tests/test_candidate_lists_gpu.py compares the keys with an
// exact numpy top-8.
extern "C" int ovs_debug_node_topk(ovs_matcher* m, int nq, const uint8_t* qdesc, const int32_t* qseg, int R, const uint8_t* tdesc,
                                   const uint8_t* taken, int q0, uint32_t* keys_out) {
    OVS_REQUIRE(m && qdesc && qseg && keys_out && nq >= 1 && R >= 0 && (R == 0 || tdesc) && q0 < nq, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(R < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 candidate keypoints");
    int rc = check_segments(nq, qseg, R, nullptr, 1);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    const size_t sQ = (size_t)nq, sR = (size_t)R, rows = sQ + (q0 >= 0 ? 1 : 0);
    NodeArgs A{};
    uint8_t *hqd, *htd, *htk, *dtk; int2* hsg;
    ovs::Staging S;
    rc = ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_q, m->d_q_cap, [&](ovs::Staging& S) {
        A.qdesc = (const uint4*)S.in(hqd, 32 * sQ); A.tdesc = (const uint4*)S.in(htd, 32 * sR); A.qseg = S.in(hsg, sQ);
        dtk = S.in(htk, sR);
    });
    if (rc != OVS_OK) return rc;
    if ((rc = ovs::grow_dev(&m->d_keys, &m->d_keys_cap, rows * kNodeK)) != OVS_OK) return rc;
    if ((rc = ovs::grow_host(&m->h_keys, &m->h_keys_cap, rows * kNodeK)) != OVS_OK) return rc;
    memcpy(hqd, qdesc, 32 * sQ);
    if (R) memcpy(htd, tdesc, 32 * sR);
    memcpy(hsg, qseg, 8 * sQ);
    if (taken) memcpy(htk, taken, sR);
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaMemsetAsync(m->d_keys, 0x5a, rows * kNodeK * 4, st));
    A.nq = nq; A.taken = taken && q0 < 0 ? dtk : nullptr;
    k_node_topk<<<(nq + 3) / 4, 128, 0, st>>>(A, m->d_keys);
    OVS_LAUNCH_CHECK();
    if (q0 >= 0) {
        NodeArgs B = A;
        B.q0 = q0; B.nq = q0 + 1; B.out_shift = nq - q0; B.taken = taken ? dtk : nullptr;
        k_node_topk<<<1, 128, 0, st>>>(B, m->d_keys);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaMemcpyAsync(m->h_keys, m->d_keys, rows * kNodeK * 4, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(keys_out, m->h_keys, rows * kNodeK * 4);
    return OVS_OK;
}

// Development aid / test hook: k_triangulation_topk on host arrays, with the launch geometry and buffers of
// ovs_robust_match_for_triangulation_host (batched == 0: one problem, nprob == 1, queries_per_prob == nq) or of
// ovs_create_new_landmarks_host (batched != 0: nq == nprob * queries_per_prob queries, query q of problem p = q / queries_per_prob
// reads keypoint entry q - p * queries_per_prob of qdesc / qbearing / qscale / qstereo, E_12 prob_E[9 p], epipole prob_epipole[3 p],
// and candidates (and taken flags) from prob_tbase[p] on).  qseg[2 nq] ranges are relative to the problem's base.  q0 and taken
// as ovs_debug_node_topk.
extern "C" int ovs_debug_triangulation_topk(ovs_matcher* m, int batched, int nq, int queries_per_prob, const uint8_t* qdesc,
                                            const double* qbearing, const float* qscale, const uint8_t* qstereo, const int32_t* qseg, int R,
                                            const uint8_t* tdesc, const double* tbearing, const uint8_t* tstereo, int nprob,
                                            const double* prob_E, const double* prob_epipole, const int32_t* prob_tbase, const uint8_t* taken,
                                            int q0, uint32_t* keys_out) {
    OVS_REQUIRE(m && qdesc && qbearing && qscale && qstereo && qseg && keys_out && prob_E && prob_epipole && nq >= 1 && R >= 0 &&
                (R == 0 || (tdesc && tbearing && tstereo)) && q0 < nq, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(R < 65536, OVS_ERR_UNSUPPORTED, "more than 65535 candidate keypoints");
    if (batched) OVS_REQUIRE(prob_tbase && nprob >= 1 && queries_per_prob >= 1 && (int64_t)nprob * queries_per_prob == nq, OVS_ERR_INVALID_ARG,
                             "batched: nq must be nprob * queries_per_prob");
    else OVS_REQUIRE(nprob == 1 && queries_per_prob == nq, OVS_ERR_INVALID_ARG, "one problem: nprob 1 and queries_per_prob == nq");
    int rc = check_segments(nq, qseg, R, batched ? prob_tbase : nullptr, queries_per_prob);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaSetDevice(m->device));
    const size_t sK = (size_t)queries_per_prob, sQ = (size_t)nq, sR = (size_t)R, NB = (size_t)nprob, rows = sQ + (q0 >= 0 ? 1 : 0);
    TriArgs A{};
    uint8_t *hqd, *htd, *hq8, *ht8, *htk, *dtk; double *hqb, *htb, *hE = nullptr, *hep = nullptr; int2* hsg; float* hqs; int* htb0 = nullptr;
    unsigned *hkeys, *dkeys;
    ovs::Staging S;
    const auto carve = [&](ovs::Staging& S) {
        A.qdesc = (const uint4*)S.in(hqd, 32 * sK); A.tdesc = (const uint4*)S.in(htd, 32 * sR);
        A.qbearing = S.in(hqb, 3 * sK); A.tbearing = S.in(htb, 3 * sR); A.qseg = S.in(hsg, sQ); A.qscale = S.in(hqs, sK);
        A.qstereo = S.in(hq8, sK); A.tstereo = S.in(ht8, sR);
        if (batched) { A.prob_E = S.in(hE, 9 * NB); A.prob_epipole = S.in(hep, 3 * NB); A.prob_tbase = S.in(htb0, NB); }
        dtk = S.in(htk, sR);
        if (batched) dkeys = S.out(hkeys, rows * kTriK);
    };
    rc = batched ? ovs::stage(S, m->h_tri, m->h_tri_cap, m->d_tri, m->d_tri_cap, carve) : ovs::stage(S, m->h_stage, m->h_stage_cap, m->d_q, m->d_q_cap, carve);
    if (rc != OVS_OK) return rc;
    if (!batched) {
        if ((rc = ovs::grow_dev(&m->d_keys, &m->d_keys_cap, rows * kTriK)) != OVS_OK) return rc;
        if ((rc = ovs::grow_host(&m->h_keys, &m->h_keys_cap, rows * kTriK)) != OVS_OK) return rc;
        dkeys = m->d_keys; hkeys = m->h_keys;
    }
    memcpy(hqd, qdesc, 32 * sK); memcpy(hqb, qbearing, 24 * sK); memcpy(hqs, qscale, 4 * sK); memcpy(hq8, qstereo, sK);
    memcpy(hsg, qseg, 8 * sQ);
    if (R) { memcpy(htd, tdesc, 32 * sR); memcpy(htb, tbearing, 24 * sR); memcpy(ht8, tstereo, sR); }
    if (taken) memcpy(htk, taken, sR);
    if (batched) { memcpy(hE, prob_E, 72 * NB); memcpy(hep, prob_epipole, 24 * NB); memcpy(htb0, prob_tbase, 4 * NB); }
    for (int k = 0; k < 9; ++k) A.E[k] = prob_E[k];
    for (int k = 0; k < 3; ++k) A.epipole[k] = prob_epipole[k];
    A.nq = nq; A.queries_per_prob = queries_per_prob; A.taken = taken && q0 < 0 ? dtk : nullptr;
    cudaStream_t st = m->stream;
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaMemsetAsync(dkeys, 0x5a, rows * kTriK * 4, st));
    const auto launch = [&](const TriArgs& a, int blocks) {
        if (batched) k_triangulation_topk<true><<<blocks, 128, 0, st>>>(a, dkeys);
        else k_triangulation_topk<false><<<blocks, 128, 0, st>>>(a, dkeys);
    };
    launch(A, (nq + 3) / 4);
    OVS_LAUNCH_CHECK();
    if (q0 >= 0) {
        TriArgs B = A;
        B.q0 = q0; B.nq = q0 + 1; B.out_shift = nq - q0; B.taken = taken ? dtk : nullptr;
        launch(B, 1);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaMemcpyAsync(hkeys, dkeys, rows * kTriK * 4, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(keys_out, hkeys, rows * kTriK * 4);
    return OVS_OK;
}

// bow_tree::match_frame_and_keyframe(keyfrm, frm, matched_lms_in_frm): matched_keyfrm_idx_of_frm[i] = the keyframe keypoint
// whose landmark frame keypoint i receives, or -1.  lm_valid_kf[k]: keyfrm landmark k non-null and not will_be_erased().
extern "C" int ovs_bow_tree_match_frame_and_keyframe_host(ovs_matcher* m, int n_kf, const uint8_t* desc_kf, const float* angle_kf, const uint8_t* lm_valid_kf,
                                                          const int32_t* bow_node_kf, int n_frm, const uint8_t* desc_frm, const float* angle_frm,
                                                          const int32_t* bow_node_frm, float lowe_ratio, int check_orientation,
                                                          int32_t* matched_keyfrm_idx_of_frm, int* num_matches) {
    OVS_REQUIRE(m && num_matches && n_kf >= 0 && n_frm >= 0 && (n_frm == 0 || matched_keyfrm_idx_of_frm), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n_kf == 0 || (desc_kf && angle_kf && lm_valid_kf && bow_node_kf), OVS_ERR_INVALID_ARG, "null keyframe array");
    OVS_REQUIRE(n_frm == 0 || (desc_frm && angle_frm && bow_node_frm), OVS_ERR_INVALID_ARG, "null frame array");
    *num_matches = 0;
    for (int i = 0; i < n_frm; ++i) matched_keyfrm_idx_of_frm[i] = -1;
    std::vector<int> match, order;
    const int rc = bow_core(m, n_kf, desc_kf, lm_valid_kf, bow_node_kf, n_frm, desc_frm, nullptr, bow_node_frm, lowe_ratio, match, order);
    if (rc != OVS_OK) return rc;
    int num = 0;
    ovs::OrientationCheck orientation;
    for (int k : order) {
        const int f = match[k];
        matched_keyfrm_idx_of_frm[f] = k; ++num;
        if (check_orientation) orientation.add(angle_kf[k] - angle_frm[f], f);
    }
    orientation.unset_invalid([&](int f) { matched_keyfrm_idx_of_frm[f] = -1; --num; });
    *num_matches = num;
    return OVS_OK;
}

// bow_tree::match_keyframes(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_1): both keypoints need a valid landmark, a keyframe-2
// keypoint is matched at most once.  matched_idx_2_of_1[i1] = keypoint of keyframe 2 or -1.
extern "C" int ovs_bow_tree_match_keyframes_host(ovs_matcher* m, int n1, const uint8_t* desc_1, const float* angle_1, const uint8_t* lm_valid_1,
                                                 const int32_t* bow_node_1, int n2, const uint8_t* desc_2, const float* angle_2, const uint8_t* lm_valid_2,
                                                 const int32_t* bow_node_2, float lowe_ratio, int check_orientation,
                                                 int32_t* matched_idx_2_of_1, int* num_matches) {
    OVS_REQUIRE(m && num_matches && n1 >= 0 && n2 >= 0 && (n1 == 0 || matched_idx_2_of_1), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n1 == 0 || (desc_1 && angle_1 && lm_valid_1 && bow_node_1), OVS_ERR_INVALID_ARG, "null keyframe-1 array");
    OVS_REQUIRE(n2 == 0 || (desc_2 && angle_2 && lm_valid_2 && bow_node_2), OVS_ERR_INVALID_ARG, "null keyframe-2 array");
    *num_matches = 0;
    for (int i = 0; i < n1; ++i) matched_idx_2_of_1[i] = -1;
    std::vector<int> match, order;
    const int rc = bow_core(m, n1, desc_1, lm_valid_1, bow_node_1, n2, desc_2, lm_valid_2, bow_node_2, lowe_ratio, match, order);
    if (rc != OVS_OK) return rc;
    int num = 0;
    ovs::OrientationCheck orientation;
    for (int i1 : order) {
        matched_idx_2_of_1[i1] = match[i1]; ++num;
        if (check_orientation) orientation.add(angle_1[i1] - angle_2[match[i1]], i1);
    }
    orientation.unset_invalid([&](int i1) { matched_idx_2_of_1[i1] = -1; --num; });
    *num_matches = num;
    return OVS_OK;
}
