// window_walk.cuh -- one query's walk over a grid-indexed frame (data::frame::get_keypoints_in_cell, then the per-candidate tests
// and the 256-bit Hamming distance of the projection, area and fuse searches), shared by k_window_topk (match_window.cu) and
// k_fuse_search (fuse.cu).  The frame's keypoints are in rank order: sorted by (cell_x, cell_y, index), the order
// get_keypoints_in_cell visits them, with a CSR of cell starts.
#pragma once
#include <cstdint>

namespace ovs {

__device__ __forceinline__ int cv_floor_f(float v) { return __float2int_rd(v); }
__device__ __forceinline__ int cv_ceil_f(float v) { return __float2int_ru(v); }

// match::compute_descriptor_distance_32 by eight population counts
__device__ __forceinline__ int hamming256(const uint4& qa, const uint4& qb, const uint4& ta, const uint4& tb) {
    return __popc(qa.x ^ ta.x) + __popc(qa.y ^ ta.y) + __popc(qa.z ^ ta.z) + __popc(qa.w ^ ta.w)
           + __popc(qb.x ^ tb.x) + __popc(qb.y ^ tb.y) + __popc(qb.z ^ tb.z) + __popc(qb.w ^ tb.w);
}

struct WindowFrame {
    float min_x, min_y, inv_w, inv_h;
    int cols, rows;
    const float* x; const float* y; const float* xr; const signed char* oct; const uint4* desc;
    const int* cell_start; const unsigned short* cap;
};

// One warp walks the cells of the window around `ref` (cell range in float arithmetic as in the reference), lane `lane` taking
// every 32nd keypoint of each cell column, and calls take((distance << 16) | rank) for every candidate that passes the box, the
// level range [min_level, max_level] (max_level < 0: unbounded) and either
//   - fuse_gate: match::fuse's chi-square bound on the reprojection error, weighted by inv_sigma_sq(candidate octave): 5.99, or
//     7.8 with the x_right term where the candidate has an x_right >= 0 and the query one (has_xr_q), or
//   - else, where the frame has x_right: |xr_q - x_right| <= margin for candidates with x_right > 0;
// and, with a per-keypoint cap, distance < cap.  A lane meets its candidates in visiting order, so a sorted insert keeps the
// reference's first-wins ties.  xr_q_of() returns the query's x_right (-1 without one: has_xr_q false), read only when the window
// holds a cell; qdesc points at the query's descriptor.
template <class XrQ, class InvSigmaSq, class Take>
__device__ __forceinline__ void window_walk(const WindowFrame& F, const float2 ref, const float margin, const int min_level, const int max_level,
                                            const bool has_xr_q, XrQ xr_q_of, const uint4* qdesc, const bool fuse_gate, InvSigmaSq inv_sigma_sq,
                                            const int lane, Take take) {
    const int min_cx = max(0, cv_floor_f(__fmul_rn(__fsub_rn(__fsub_rn(ref.x, F.min_x), margin), F.inv_w)));
    const int max_cx = min(F.cols - 1, cv_ceil_f(__fmul_rn(__fadd_rn(__fsub_rn(ref.x, F.min_x), margin), F.inv_w)));
    const int min_cy = max(0, cv_floor_f(__fmul_rn(__fsub_rn(__fsub_rn(ref.y, F.min_y), margin), F.inv_h)));
    const int max_cy = min(F.rows - 1, cv_ceil_f(__fmul_rn(__fadd_rn(__fsub_rn(ref.y, F.min_y), margin), F.inv_h)));
    if (F.cols > min_cx && max_cx >= 0 && F.rows > min_cy && max_cy >= 0) {
        const uint4 qa = __ldg(qdesc), qb = __ldg(qdesc + 1);
        const bool check_level = (0 < min_level) || (0 <= max_level);
        const float xr_q = xr_q_of();
        for (int cx = min_cx; cx <= max_cx; ++cx) {
            const int r0 = F.cell_start[cx * F.rows + min_cy], r1 = F.cell_start[cx * F.rows + max_cy + 1];
            for (int r = r0 + lane; r < r1; r += 32) {
                if (check_level) {
                    const int o = F.oct[r];
                    if (o < min_level) continue;
                    if (0 <= max_level && max_level < o) continue;
                }
                const float dist_x = __fsub_rn(F.x[r], ref.x), dist_y = __fsub_rn(F.y[r], ref.y);
                if (!(fabsf(dist_x) < margin && fabsf(dist_y) < margin)) continue;
                if (fuse_gate) {
                    const float ex = __fsub_rn(ref.x, F.x[r]), ey = __fsub_rn(ref.y, F.y[r]);
                    const float w = inv_sigma_sq(F.oct[r]);
                    const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                    const float kxr = F.xr ? F.xr[r] : -1.0f;
                    if (kxr >= 0 && has_xr_q) {
                        const float er = __fsub_rn(xr_q, kxr);
                        if (__fmul_rn(__fadd_rn(e2, __fmul_rn(er, er)), w) > 7.8f) continue;
                    } else {
                        if (__fmul_rn(e2, w) > 5.99f) continue;
                    }
                } else if (F.xr) {
                    const float kxr = F.xr[r];
                    if (0 < kxr) {
                        const float reproj_error = fabsf(__fsub_rn(xr_q, kxr));
                        if (margin < reproj_error) continue;
                    }
                }
                const uint4 ta = __ldg(F.desc + 2 * (size_t)r), tb = __ldg(F.desc + 2 * (size_t)r + 1);
                const int d = hamming256(qa, qb, ta, tb);
                if (F.cap && !(d < (int)F.cap[r])) continue;
                take(((unsigned)d << 16) | (unsigned)r);
            }
        }
    }
}

}  // namespace ovs
