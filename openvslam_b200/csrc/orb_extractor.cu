// orb_extractor.cu -- H100 (sm_90a) implementation of openvslam::feature::orb_extractor::extract
// (feature/orb_extractor.{h,cc}; names as recalled in SURVEY.md 8a -- /root/reference holds no
// source to cite line numbers from).
//
// Pipeline of one extract() (all kernels on the handle's stream):
//   upload            image -> pyramid level 0                        (cudaMemcpy2DAsync)
//   k_pyramid_group   cv::resize INTER_LINEAR fixed point, 3-4 levels per launch (a CTA
//                     owns a tile of the group's last level and recomputes the halo of
//                     the levels between in shared memory)                            x 2
//   k_fast_score      FAST-9 corner score S(p) for every pixel of every level         x 1
//   k_cell_nms        per 64x64 detection cell: 3x3 strict-max NMS, ini/min threshold
//                     fallback, row-major ordered emit                                x 1
//   k_tree_distribute cells -> ordered candidate list of the level, per-keypoint mask filter,
//                     distribute_keypoints_via_tree; one CTA per level (array passes, no
//                     host hop)                                                        x 1
//   k_orient_describe per selected keypoint: 43x43 patch -> IC angle, 7x7 Gaussian
//                     (bit-exact fixed point, computed on the patch only), rotated
//                     256-bit BRIEF, final cv::KeyPoint fields                        x 1
//   download          keypoints + descriptors
//
// HBM layout: the pyramid is one allocation, level l at byte offset off[l] (256 B aligned),
// row pitch a multiple of 128 B; the FAST score map uses the same geometry.  The blurred
// pyramid of the reference is never materialised: the blur is exact integer arithmetic, so the
// 37x37 blurred window each descriptor reads is recomputed from the raw patch in shared memory.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include <cuda.h>   // CUtensorMap (the encode function is fetched through cudaGetDriverEntryPoint; no -lcuda)

#include "orb_math.cuh"
#include "ovs_common.h"
#include "stereo_rectify.h"

namespace {

constexpr int kMaxLevels = 16;
constexpr int kBorder = 19;        // orb_patch_radius_
constexpr int kCell = 64;          // cell_size
constexpr int kOverlap = 6;        // overlap
constexpr int kCellCap = 1024;     // NMS survivors in a 64x64 cell are pairwise non-adjacent
constexpr int kTileW = 128, kTileH = 32;
constexpr int kStatTma = 64, kStatInts = 96;   // layout of the extractor's device status block (see ovs_extractor)

struct LevelTable {
    int num_levels;
    int w[kMaxLevels], h[kMaxLevels], pitch[kMaxLevels];
    unsigned off[kMaxLevels];
    int tile_begin[kMaxLevels + 1];
    int tiles_x[kMaxLevels];
    float scale[kMaxLevels];
    float kp_size[kMaxLevels];
};

struct CellInfo {
    short rx0, ry0;  // first examined pixel of the cell (ROI origin + 3)
    short rw, rh;    // examined extent (ROI size - 6), <= 64
    int level;
};

// FAST candidate as produced by the cell NMS kernel: x | y << 12 | score << 24, x and y relative to the 19 px level border
// (the reference's keypts_to_distribute coordinates).
struct SelKp {
    short lx, ly;
    unsigned char level, score;
    unsigned short pad;
};

struct UMax { signed char v[16]; };

// One TMA descriptor per pyramid level: u8 tensor {pitch, h}, box {kTmaBoxW, kTileH + 6}, zero fill outside.
// The box starts at a multiple of 16 bytes, 16 columns left of the tile: an unaligned innermost start coordinate was
// found to fault ("illegal instruction") when the kernels were first written, and the aligned start is kept.
constexpr int kTmaBoxW = 160;   // 16 (aligned left halo, 4 used) + 128 + 16 (right halo, 3 used)
constexpr int kTmaHaloX = 16;
struct TmapArray { CUtensorMap m[kMaxLevels]; };
// boxes of the two other TMA-staged kernels: the 66 x 66 score window of a detection cell (k_cell_nms) and the 43 x 43 patch of
// a keypoint (k_orient_describe).  A tiled TMA copy needs a 16-byte aligned innermost start coordinate, so the box starts at
// the window's x rounded down to 16 and is 15 bytes wider than the window needs.
constexpr int kNmsBoxW = 96, kNmsBoxH = 66;
constexpr int kPatchBoxW = 64, kPatchBoxH = 43;

// One TMA box copy (cp.async.bulk.tensor.2d, zero fill outside the tensor) into `dst` (128-byte aligned shared memory), issued by
// thread 0 and awaited by the whole block on the mbarrier `mbar`.  Returns false -- block-uniformly -- when the bytes did not
// arrive within the spin bound (a descriptor fault must not hang the device).
__device__ __forceinline__ bool tma_box_2d(void* dst, const CUtensorMap* map, int x, int y, unsigned bytes, unsigned long long* mbar) {
    const unsigned mbar_s = (unsigned)__cvta_generic_to_shared(mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" :: "r"(mbar_s));
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // make the init visible to the async (TMA) proxy
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
        const unsigned long long desc = reinterpret_cast<unsigned long long>(map);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(mbar_s), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
                     :: "r"(d), "l"(desc), "r"(x), "r"(y), "r"(mbar_s) : "memory");
    }
    unsigned done = 0;
    for (int spin = 0; spin < (1 << 22) && !done; ++spin)
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(mbar_s) : "memory");
    return !__syncthreads_or(!done);
}

__constant__ signed char c_pattern[256][4] = {
#include "orb_pattern.inc"
};

// ---------------------------------------------------------------------------- resize (compute_image_pyramid)
// xtab[dx] = {xofs, a0 | a1 << 16}, ytab[dy] = {yofs, b0 | b1 << 16}: cv::resize's INTER_LINEAR coefficient tables (11-bit fixed point).
// Several pyramid levels per launch.  The reference resizes level l into level l + 1 (cv::resize, INTER_LINEAR), level after
// level; each level is a function of the ROUNDED previous one, so the chain cannot be collapsed -- but a tile of level l + n needs only
// a slightly larger tile of level l + n - 1, and so on down.  One CTA owns a kPyrTW x kPyrTH tile of the group's LAST level: it works
// out, through the same coefficient tables, the intervals of every level of the group that its tile depends on, computes them level by
// level in shared memory (first level of the group from global memory) and writes to global memory the pixels it OWNS: its tile of
// the last level, and of every intermediate level the interval [first source column of its tile, first source column of the next
// tile) -- those intervals partition the level and lie inside what the CTA computes anyway (the recomputed halo is a few columns).
// Every pixel is computed with the reference's integer arithmetic from exact source pixels, so recomputation changes nothing.
constexpr int kPyrTW = 64, kPyrTH = 16, kPyrMaxGroup = 4;
struct PyrGroup {
    int src_level, nlev;                 // computes levels src_level + 1 .. src_level + nlev
    int tiles_x, tiles_y;
    int buf_w[kPyrMaxGroup], buf_h[kPyrMaxGroup];     // extent bound of the region of level src_level + k (k = 1 .. nlev - 1) held in shared memory
    int buf_off[kPyrMaxGroup];           // byte offset of that buffer in dynamic shared memory
    unsigned xtab_off[kPyrMaxGroup + 1], ytab_off[kPyrMaxGroup + 1];   // coefficient tables of level src_level + k (index k)
};
struct PyrSpan { int lo, hi, olo, ohi; };   // computed interval [lo, hi), owned interval [olo, ohi)

// Source interval of destination interval D through a coefficient table, united with the owned interval of the source level.
__device__ __host__ __forceinline__ PyrSpan pyr_source_span(const PyrSpan D, const int2* tab, int src_extent, bool first_tile, bool last_tile) {
    auto srcpos = [&](int d) { const int v = tab[d].x; return v < 0 ? 0 : (v > src_extent - 1 ? src_extent - 1 : v); };
    PyrSpan S;
    const int flo = srcpos(D.lo), fhi = min(src_extent - 1, srcpos(D.hi - 1) + 1) + 1;
    S.olo = first_tile ? 0 : srcpos(D.olo);
    S.ohi = last_tile ? src_extent : srcpos(D.ohi);
    S.lo = min(flo, S.olo);
    S.hi = max(fhi, S.ohi);
    return S;
}

__global__ void __launch_bounds__(256) k_pyramid_group(uint8_t* __restrict__ pyr, LevelTable T, const int2* __restrict__ tabs, PyrGroup G) {
    extern __shared__ __align__(16) uint8_t s_pyr[];
    const int tx = blockIdx.x % G.tiles_x, ty = blockIdx.x / G.tiles_x;
    const int last = G.src_level + G.nlev;
    PyrSpan X[kPyrMaxGroup + 1], Y[kPyrMaxGroup + 1];       // index k: level src_level + k
    X[G.nlev].lo = X[G.nlev].olo = tx * kPyrTW; X[G.nlev].hi = X[G.nlev].ohi = min(T.w[last], (tx + 1) * kPyrTW);
    Y[G.nlev].lo = Y[G.nlev].olo = ty * kPyrTH; Y[G.nlev].hi = Y[G.nlev].ohi = min(T.h[last], (ty + 1) * kPyrTH);
#pragma unroll
    for (int k = kPyrMaxGroup - 1; k >= 1; --k) {
        if (k < G.nlev) {
            const int l = G.src_level + k;
            X[k] = pyr_source_span(X[k + 1], tabs + G.xtab_off[k + 1], T.w[l], tx == 0, tx == G.tiles_x - 1);
            Y[k] = pyr_source_span(Y[k + 1], tabs + G.ytab_off[k + 1], T.h[l], ty == 0, ty == G.tiles_y - 1);
        }
    }
#pragma unroll
    for (int k = 1; k <= kPyrMaxGroup; ++k) {
        if (k <= G.nlev) {
            const int l = G.src_level + k;
            const int sw = T.w[l - 1], sh = T.h[l - 1];
            const int2* xtab = tabs + G.xtab_off[k];
            const int2* ytab = tabs + G.ytab_off[k];
            const uint8_t* gsrc = pyr + T.off[l - 1];
            const int gspitch = T.pitch[l - 1];
            const uint8_t* ssrc = k > 1 ? s_pyr + G.buf_off[k - 1] : nullptr;
            const int sbw = k > 1 ? G.buf_w[k - 1] : 0, sx0 = k > 1 ? X[k - 1].lo : 0, sy0 = k > 1 ? Y[k - 1].lo : 0;
            uint8_t* sdst = k < G.nlev ? s_pyr + G.buf_off[k] : nullptr;
            const int dbw = k < G.nlev ? G.buf_w[k] : 0;
            uint8_t* gdst = pyr + T.off[l];
            const int gdpitch = T.pitch[l];
            const PyrSpan RX = X[k], RY = Y[k];
            const int rw = RX.hi - RX.lo, rh = RY.hi - RY.lo;
            for (int i = threadIdx.x; i < rw * rh; i += 256) {
                const int ry = i / rw, rx = i - ry * rw;
                const int dx = RX.lo + rx, dy = RY.lo + ry;
                const int2 yt = ytab[dy], xt = xtab[dx];
                const int y0 = max(0, min(yt.x, sh - 1)), y1 = max(0, min(yt.x + 1, sh - 1));
                const int x0 = xt.x, x1 = min(xt.x + 1, sw - 1);
                const int a0 = (short)(xt.y & 0xffff), a1 = (short)(xt.y >> 16), b0 = (short)(yt.y & 0xffff), b1 = (short)(yt.y >> 16);
                uint8_t v;
                if (k == 1) {
                    const uint8_t* S0 = gsrc + (size_t)y0 * gspitch;
                    const uint8_t* S1 = gsrc + (size_t)y1 * gspitch;
                    v = ovs::resize_px(__ldg(S0 + x0), __ldg(S0 + x1), __ldg(S1 + x0), __ldg(S1 + x1), a0, a1, b0, b1);
                } else {
                    const uint8_t* S0 = ssrc + (y0 - sy0) * sbw - sx0;
                    const uint8_t* S1 = ssrc + (y1 - sy0) * sbw - sx0;
                    v = ovs::resize_px(S0[x0], S0[x1], S1[x0], S1[x1], a0, a1, b0, b1);
                }
                if (sdst) sdst[ry * dbw + rx] = v;
                if (dx >= RX.olo && dx < RX.ohi && dy >= RY.olo && dy < RY.ohi) gdst[(size_t)dy * gdpitch + dx] = v;
            }
            __syncthreads();
        }
    }
}

// ----------------------------------------------------------- undistortion + bearings
// data::frame's constructor, right after extract(): camera->undistort_keypoints(keypts_, undist_keypts_) and
// camera->convert_keypoints_to_bearings(undist_keypts_, bearings_).  Perspective: cv::undistortPoints with R = I, P = K and a
// fixed iteration count (OpenVSLAM: 20), in double precision, stored as float like the CV_32FC2 destination -- bit-exact
// with OpenCV because only + - x / are involved and this library is built with --fmad=false; equirectangular: identity.
struct UndistortArgs {
    int model, iters;
    double fx, fy, cx, cy, k1, k2, p1, p2, k3, cols, rows;
};

__global__ void __launch_bounds__(128) k_undistort_bearings(UndistortArgs A, int n, const ovs_keypoint* __restrict__ in, ovs_keypoint* __restrict__ out,
                                                             double* __restrict__ bearings) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    ovs_keypoint k = in[i];
    double bx, by, bz;
    if (A.model == OVS_CAMERA_EQUIRECTANGULAR) {
        const double lon = ((double)k.x / A.cols - 0.5) * (2.0 * 3.14159265358979323846);
        const double lat = -((double)k.y / A.rows - 0.5) * 3.14159265358979323846;
        bx = cos(lat) * sin(lon); by = -sin(lat); bz = cos(lat) * cos(lon);
    } else if (A.model == OVS_CAMERA_FISHEYE || A.model == OVS_CAMERA_RADIAL_DIVISION) {
        const double pwx = ((double)k.x - A.cx) / A.fx, pwy = ((double)k.y - A.cy) / A.fy;
        double ux, uy;
        if (A.model == OVS_CAMERA_FISHEYE) {
            // cv::fisheye::undistortPoints(pts, K, D = {k1, k2, k3, k4}, R = I, P = K), default criteria (<= iters Newton steps, 1e-8):
            // here k1, k2, p1, p2 hold the four fisheye coefficients
            const double kPi2 = 3.14159265358979323846 / 2.;
            double theta_d = sqrt(pwx * pwx + pwy * pwy);
            theta_d = fmin(fmax(-kPi2, theta_d), kPi2);
            bool converged = false;
            double theta = theta_d, scale = 0.0;
            if (fabs(theta_d) > 1e-8) {
                for (int j = 0; j < A.iters; ++j) {
                    const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
                    const double k0_theta2 = A.k1 * theta2, k1_theta4 = A.k2 * theta4, k2_theta6 = A.p1 * theta6, k3_theta8 = A.p2 * theta8;
                    const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                             (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
                    theta = theta - theta_fix;
                    if (fabs(theta_fix) < 1e-8) { converged = true; break; }
                }
                scale = tan(theta) / theta_d;
            } else {
                converged = true;
            }
            const bool flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
            if (converged && !flipped) { ux = A.fx * (pwx * scale) + A.cx; uy = A.fy * (pwy * scale) + A.cy; }
            else { ux = -1000000.0; uy = -1000000.0; }
        } else {
            // camera::radial_division: p_u = p_d / (1 + distortion |p_d|^2); k1 holds the distortion parameter
            const double r2 = pwx * pwx + pwy * pwy;
            const double sc = 1.0 / (1.0 + A.k1 * r2);
            ux = A.fx * (pwx * sc) + A.cx; uy = A.fy * (pwy * sc) + A.cy;
        }
        k.x = (float)ux; k.y = (float)uy;
        const double xn = ((double)k.x - A.cx) / A.fx, yn = ((double)k.y - A.cy) / A.fy;
        const double l2 = sqrt(xn * xn + yn * yn + 1.0);
        bx = xn / l2; by = yn / l2; bz = 1.0 / l2;
    } else {
        const double ifx = 1.0 / A.fx, ify = 1.0 / A.fy;
        double x = ((double)k.x - A.cx) * ifx, y = ((double)k.y - A.cy) * ify;
        const double x0 = x, y0 = y;
        for (int it = 0; it < A.iters; ++it) {
            const double r2 = x * x + y * y;
            const double icdist = 1.0 / (1.0 + ((A.k3 * r2 + A.k2) * r2 + A.k1) * r2);
            const double dx = 2.0 * A.p1 * x * y + A.p2 * (r2 + 2.0 * x * x);
            const double dy = A.p1 * (r2 + 2.0 * y * y) + 2.0 * A.p2 * x * y;
            x = (x0 - dx) * icdist;
            y = (y0 - dy) * icdist;
        }
        k.x = (float)(x * A.fx + A.cx);
        k.y = (float)(y * A.fy + A.cy);
        // bearing of the UNDISTORTED keypoint (the float the frame stores), as convert_keypoints_to_bearings does
        const double xn = ((double)k.x - A.cx) / A.fx, yn = ((double)k.y - A.cy) / A.fy;
        const double l2 = sqrt(xn * xn + yn * yn + 1.0);
        bx = xn / l2; by = yn / l2; bz = 1.0 / l2;
    }
    if (out) out[i] = k;
    if (bearings) { bearings[3 * (size_t)i] = bx; bearings[3 * (size_t)i + 1] = by; bearings[3 * (size_t)i + 2] = bz; }
}

// --------------------------------------------------------------------- colour -> gray
// util::convert_to_grayscale = cv::cvtColor(img, {BGR,RGB,BGRA,RGBA}2GRAY), CV_8U: 15-bit fixed point
// (B 3735, G 19235, R 9798, rounding 1 << 14), bit-exact with OpenCV 4.  One thread -> 4 pixels of level 0.
__global__ void __launch_bounds__(256) k_color_to_gray(const uint8_t* __restrict__ src, size_t spitch, int w, int h, int channels, int r_first,
                                                        uint8_t* __restrict__ dst, int dpitch) {
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x0 >= w || y >= h) return;
    const uint8_t* p = src + (size_t)y * spitch + (size_t)x0 * channels;
    unsigned packed = 0;
    const int cnt = min(4, w - x0);
    for (int i = 0; i < cnt; ++i, p += channels) {
        const int c0 = __ldg(p), c1 = __ldg(p + 1), c2 = __ldg(p + 2);
        const int b = r_first ? c2 : c0, r = r_first ? c0 : c2;
        packed |= (unsigned)((b * 3735 + c1 * 19235 + r * 9798 + 16384) >> 15) << (8 * i);
    }
    uint8_t* d = dst + (size_t)y * dpitch + x0;
    if (cnt == 4) *reinterpret_cast<unsigned*>(d) = packed;
    else for (int i = 0; i < cnt; ++i) d[i] = (uint8_t)(packed >> (8 * i));
}

// ------------------------------------------------------------------------- FAST score
__device__ __forceinline__ int byte_of(const unsigned (&w)[3], int b) {
    return (int)((w[b >> 2] >> (8 * (b & 3))) & 0xffu);
}

// Tile = 128 x 32 pixels, one thread -> 4 adjacent pixels of one row, 4 row groups.
// The tile plus its halo -- columns [x0-16, x0+144), rows [y0-3, y0+35) -- is staged into shared
// memory by ONE TMA bulk-tensor copy (cp.async.bulk.tensor.2d, zero fill outside the level) whose
// completion is signalled on an mbarrier; every thread then reads 32-bit words from the tile.
__global__ void __launch_bounds__(256) k_fast_score(const __grid_constant__ TmapArray maps, LevelTable T,
                                                     uint8_t* __restrict__ score, int min_thr, int* __restrict__ tma_timeout) {
    __shared__ __align__(128) unsigned tile[(kTileH + 6) * (kTmaBoxW / 4)];
    __shared__ __align__(8) unsigned long long mbar;
    constexpr int TW = kTmaBoxW / 4;   // tile pitch in 32-bit words
    int level = 0;
    while (level + 1 < T.num_levels && (int)blockIdx.x >= T.tile_begin[level + 1]) ++level;
    const int t = blockIdx.x - T.tile_begin[level];
    const int tx = t % T.tiles_x[level], ty = t / T.tiles_x[level];
    const int w = T.w[level], h = T.h[level], pitch = T.pitch[level];
    const int x0 = tx * kTileW, y0 = ty * kTileH;

    const unsigned mbar_s = (unsigned)__cvta_generic_to_shared(&mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" :: "r"(mbar_s));
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // make the init visible to the async (TMA) proxy
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned dst = (unsigned)__cvta_generic_to_shared(tile);
        const unsigned long long desc = reinterpret_cast<unsigned long long>(&maps.m[level]);
        constexpr unsigned bytes = (kTileH + 6) * kTmaBoxW;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(mbar_s), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
                     :: "r"(dst), "l"(desc), "r"(x0 - kTmaHaloX), "r"(y0 - 3), "r"(mbar_s) : "memory");
    }
    {
        // wait for the TMA bytes (phase 0); bounded so a descriptor fault cannot hang the device
        unsigned done = 0;
        for (int spin = 0; spin < (1 << 22) && !done; ++spin)
            asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(mbar_s) : "memory");
        // the whole block takes the same decision: either every thread saw the tile arrive or nobody writes a score
        if (__syncthreads_or(!done)) { if (threadIdx.x == 0) *tma_timeout = 1; return; }
    }

    const int q = threadIdx.x & 31;
    const int rr = threadIdx.x >> 5;
    constexpr int rdx[16] = OVS_FAST_RING_DX;
    constexpr int rdy[16] = OVS_FAST_RING_DY;
#pragma unroll 1
    for (int rg = 0; rg < 4; ++rg) {
        const int r = rg * 8 + rr;
        const int gy = y0 + r;
        const int gx0 = x0 + 4 * q;
        if (gy >= h || gx0 >= pitch) continue;
        unsigned rows[7][3];
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const unsigned* p = tile + (r + j) * TW + (kTmaHaloX / 4 - 1) + q;
            rows[j][0] = p[0]; rows[j][1] = p[1]; rows[j][2] = p[2];
        }
        unsigned packed = 0;
        const bool row_ok = gy >= 3 && gy < h - 3;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int gx = gx0 + i;
            int s = 0;
            if (row_ok && gx >= 3 && gx < w - 3) {
                const int v = byte_of(rows[3], 4 + i);
                const int d0 = v - byte_of(rows[3 + rdy[0]], 4 + i + rdx[0]);
                const int d4 = v - byte_of(rows[3 + rdy[4]], 4 + i + rdx[4]);
                const int d8 = v - byte_of(rows[3 + rdy[8]], 4 + i + rdx[8]);
                const int d12 = v - byte_of(rows[3 + rdy[12]], 4 + i + rdx[12]);
                if (ovs::fast9_maybe(d0, d4, d8, d12, min_thr)) {
                    int d[16];
#pragma unroll
                    for (int k = 0; k < 16; ++k) d[k] = v - byte_of(rows[3 + rdy[k]], 4 + i + rdx[k]);
                    s = ovs::fast9_score(d);
                    if (s < min_thr) s = 0;
                }
            }
            packed |= (unsigned)s << (8 * i);
        }
        *reinterpret_cast<unsigned*>(score + T.off[level] + (size_t)gy * pitch + gx0) = packed;
    }
}

// ---------------------------------------------------------------------------- cell NMS
// cv::FAST(nonmax=true) on the cell ROI, for threshold ini and (if that leaves nothing) min:
// a pixel survives iff its score is >= thr and strictly greater than the scores of its 8
// neighbours, pixels outside the cell's examined band counting as 0.  Because the score map
// holds S only where S >= min_thr, the survivors at ini are the survivors at min with S >= ini.
// Emits (x, y, score) in cv::FAST's row-major order into the cell's slot.
// The cell's 66 x 66 score window (examined band + 1 px) arrives as ONE TMA box; the ring outside the band is then cleared.
__global__ void __launch_bounds__(256) k_cell_nms(const __grid_constant__ TmapArray smaps, LevelTable T, const CellInfo* __restrict__ cells,
                                                   const uint8_t* __restrict__ cell_skip,
                                                   int ini_thr, uint32_t* __restrict__ cell_tmp, int* __restrict__ cell_count, int* __restrict__ tma_timeout) {
    __shared__ __align__(128) uint8_t win[kNmsBoxH][kNmsBoxW];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ int warp_sums[8];
    const int cell = blockIdx.x;
    if (cell_skip != nullptr && cell_skip[cell]) {
        if (threadIdx.x == 0) cell_count[cell] = 0;
        return;
    }
    const CellInfo ci = cells[cell];
    const int wx = ci.rx0 - 1, wy = ci.ry0 - 1;          // window origin; column `sh` of the box is column 0 of the window
    const int sh = wx & 15;
    if (!tma_box_2d(&win[0][0], &smaps.m[ci.level], wx - sh, wy, kNmsBoxH * kNmsBoxW, &mbar)) {
        if (threadIdx.x == 0) { *tma_timeout = 1; cell_count[cell] = 0; }
        return;
    }
    // pixels outside the examined band count as 0: rows 0 and rh + 1, columns 0 and rw + 1 of the window
    for (int i = threadIdx.x; i < 4 * 66; i += 256) {
        const int side = i / 66, j = i - side * 66;
        if (side == 0) win[0][sh + j] = 0;
        else if (side == 1) win[ci.rh + 1][sh + j] = 0;
        else if (side == 2) win[j][sh] = 0;
        else win[j][sh + ci.rw + 1] = 0;
    }
    __syncthreads();
    uint8_t (*sc)[kNmsBoxW] = reinterpret_cast<uint8_t (*)[kNmsBoxW]>(&win[0][sh]);    // sc[r][c]: window row r, column c

    const int r = threadIdx.x >> 2;
    const int c0 = (threadIdx.x & 3) * 16;
    unsigned keep = 0, keep_ini = 0;
    if (r < ci.rh) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int c = c0 + k;
            const int s = sc[r + 1][c + 1];
            if (c < ci.rw && s > 0) {
                const bool mx = s > sc[r][c] && s > sc[r][c + 1] && s > sc[r][c + 2] && s > sc[r + 1][c] && s > sc[r + 1][c + 2]
                                && s > sc[r + 2][c] && s > sc[r + 2][c + 1] && s > sc[r + 2][c + 2];
                if (mx) {
                    keep |= 1u << k;
                    if (s >= ini_thr) keep_ini |= 1u << k;
                }
            }
        }
    }
    const int any_ini = __syncthreads_or(keep_ini != 0);
    if (any_ini) keep = keep_ini;

    // block-wide exclusive scan of popcounts (thread order == row-major order)
    const int n = __popc(keep);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    int base = 0, total = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (k < wid) base += warp_sums[k];
        total += warp_sums[k];
    }
    int pos = base + incl - n;
    uint32_t* out = cell_tmp + (size_t)cell * kCellCap;
    if (keep) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (keep & (1u << k)) {
                const int c = c0 + k;
                const unsigned x = (unsigned)(ci.rx0 + c - kBorder), y = (unsigned)(ci.ry0 + r - kBorder);
                out[pos++] = x | (y << 12) | ((unsigned)sc[r + 1][c + 1] << 24);
            }
        }
    }
    if (threadIdx.x == 0) cell_count[cell] = total;
}

// ---------------------------------------------------------- tree distribution (orb_extractor::distribute_keypoints_via_tree)
// One CTA per pyramid level.  The reference keeps a std::list of nodes, splits every node holding more than one keypoint
// sweep after sweep (children are pushed to the list FRONT, the parent is erased) until one more sweep could overshoot the level's
// budget, then splits the remaining nodes largest-first (ties: latest created first) until the budget is reached, and keeps the
// best-response keypoint of every node in list order.  Restated without the list:
//   * every node carries the SERIAL of its creation (the reference's serial is implicit: heap order of `new`); children of the j-th
//     node processed in a pass whose first serial is sb get sb + 4 j + k, empty children included;
//   * a pass processes the nodes of the previous pass in list order = descending serial, so the next pass's node array is the
//     compaction of the children array read backwards;
//   * the final list order is "descending serial, then the surviving initial nodes in ascending order": the selected
//     (order key, candidate) pairs are sorted once at the end;
//   * largest-first phase: the children counts of ALL pool nodes are taken speculatively, a prefix sum over the sorted pool finds the
//     node at which the budget is reached; nodes behind it stay whole.
// Every step is a block-wide array pass (scan / histogram by integer atomics / bitonic sort), nothing depends on thread timing.
// tests/tree_device_model.py is the same sequence of passes in numpy, pinned against the oracle's list-based tree on the CPU.
constexpr int kTreeThreads = 1024;
constexpr int kTreeSortSmem = 8192;          // u64 keys sorted in shared memory up to this many (64 KB); beyond: in global scratch

struct TreeLevel {
    double delta_x, delta_y;    // initial node extent
    int target;                 // keypoints requested at this level
    int gx, nini;               // initial nodes: gx columns, nini in all
    int cap_nodes, cap_final;   // node slots of a pass, slots of the selection
    int node_off, final_off;    // first slot of the level in the node / selection scratch arrays (final_off in units of sort slots)
    int sel_off;                // first slot of the level's segment of the selection array read by k_orient_describe
    int cell_begin, cell_end;   // detection cells of the level (compute_fast_keypoints' visiting order)
    int cand_off, cand_cap;     // the level's slice of the per-candidate arrays
    int final_pow2;             // sort slots of the selection (power of two >= cap_final)
    int pool_pow2;              // sort slots of the pool (power of two >= cap_nodes)
    int pool_off;
};
struct TreeArgs {
    TreeLevel lv[kMaxLevels];
    float sf[kMaxLevels];
    int num_levels, total_nodes;
};
struct TreeBuffers {
    uint32_t* fc;                 // [cand_cap] candidates after the mask filter (per level at the level's candidate offset)
    int* node;                    // [cand_cap] node of a candidate in the current pass, -1 once it sits in a final single-keypoint node
    uint8_t* quad;                // [cand_cap] quadrant of the candidate in its node
    int4* box;                    // [2][total_nodes] node boxes (begin x, begin y, end x, end y), double buffered across passes
    int* cnt;                     // [2][total_nodes]
    int* ser;                     // [2][total_nodes]
    int* cc;                      // [4 total_nodes] keypoints per child
    int* nidx;                    // [4 total_nodes] child -> slot in the next pass
    unsigned* best;               // [5 total_nodes] best (score, first index) per final node
    unsigned long long* fin;      // selection sort slots
    unsigned long long* pool;     // pool sort slots (used when the pool does not fit in shared memory)
};

__device__ __forceinline__ int tcx(uint32_t c) { return (int)(c & 0xfffu); }
__device__ __forceinline__ int tcy(uint32_t c) { return (int)((c >> 12) & 0xfffu); }

__device__ __forceinline__ int tree_warp_scan(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
// exclusive prefix of one value per thread over the block; *total = sum.  Contains block barriers.
__device__ __forceinline__ int tree_block_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int inc = tree_warp_scan(v);
    __syncthreads();
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        const int x = s_warp[lane];
        const int xi = tree_warp_scan(x);
        s_warp[lane] = xi - x;
        if (lane == 31) s_warp[32] = xi;
    }
    __syncthreads();
    *total = s_warp[32];
    return s_warp[w] + inc - v;
}
__device__ __forceinline__ void tree_chunk(int len, int* b, int* e) {
    const int chunk = (len + kTreeThreads - 1) / kTreeThreads;
    *b = min(len, (int)threadIdx.x * chunk);
    *e = min(len, *b + chunk);
}
// ascending bitonic sort of P2 (power of two) keys
// Compare-exchange step j of the network touches (i, i | j) with i = ((t & ~(j - 1)) << 1) | (t & (j - 1)): for j <= 32 the 32
// consecutive t of a warp stay inside one aligned block of 64 keys, step after step, so between two such steps a warp barrier is
// enough; a block barrier is needed only around the steps with j >= 64 (51 of the 66 steps of a 2048-key sort are warp-local).
__device__ void tree_bitonic(unsigned long long* keys, int P2) {
    bool wide_before = true;                          // the keys were written by other warps
    for (int k = 2; k <= P2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            const bool wide = j >= 64;
            if (wide || wide_before) __syncthreads(); else __syncwarp();
            for (int t = threadIdx.x; t < (P2 >> 1); t += kTreeThreads) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), q = i | j;
                const bool up = (i & k) == 0;
                const unsigned long long a = keys[i], b = keys[q];
                if ((a > b) == up) { keys[i] = b; keys[q] = a; }
            }
            wide_before = wide;
        }
    __syncthreads();
}
__device__ __forceinline__ void tree_centre(const int4 b, int* cx, int* cy) {
    *cx = b.x + ((b.z - b.x + 1) >> 1);     // begin + ceil((end - begin) / 2.0)
    *cy = b.y + ((b.w - b.y + 1) >> 1);
}
// keypoints per child of the m nodes of this pass; remembers every candidate's quadrant
__device__ void tree_count_children(const uint32_t* __restrict__ fc, int n, const int* __restrict__ node, uint8_t* __restrict__ quad,
                                    const int4* __restrict__ box, int m, int* __restrict__ cc) {
    for (int c = threadIdx.x; c < 4 * m; c += kTreeThreads) cc[c] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kTreeThreads) {
        const int j = node[i];
        if (j < 0) continue;
        int cx, cy;
        tree_centre(box[j], &cx, &cy);
        const uint32_t c = fc[i];
        const int k = (cx <= tcx(c) ? 1 : 0) + (cy <= tcy(c) ? 2 : 0);
        quad[i] = (uint8_t)k;
        atomicAdd(&cc[4 * j + k], 1);
    }
    __syncthreads();
}
// The children holding more than one keypoint become the nodes of the next pass (slot order = descending child index = descending
// serial); candidates follow their child, those alone in theirs are final.  Returns the number of next-pass nodes, *ne = non-empty children.
__device__ int tree_build_next(int n, int* __restrict__ node, const uint8_t* __restrict__ quad, const int4* __restrict__ box, int m,
                               const int* __restrict__ cc, int* __restrict__ nidx, int4* __restrict__ nbox, int* __restrict__ ncnt, int* __restrict__ nser,
                               int sb, int* s_warp, int* ne, unsigned long long* fin, int cap_final, int* s_nfin) {
    int b, e;
    tree_chunk(4 * m, &b, &e);
    int big = 0, some = 0;
    for (int c = b; c < e; ++c) { const int v = cc[c]; big += v > 1; some += v > 0; }
    int tot_big, tot_some;
    const int ex = tree_block_scan(big, s_warp, &tot_big);
    tree_block_scan(some, s_warp, &tot_some);
    int run = ex;
    for (int c = b; c < e; ++c) {
        const int v = cc[c];
        if (v <= 1) continue;
        const int slot = tot_big - 1 - run;
        ++run;
        nidx[c] = slot;
        const int4 pb = box[c >> 2];
        int cx, cy;
        tree_centre(pb, &cx, &cy);
        const int k = c & 3;
        nbox[slot] = make_int4((k & 1) ? cx : pb.x, (k & 2) ? cy : pb.y, (k & 1) ? pb.z : cx, (k & 2) ? pb.w : cy);
        ncnt[slot] = v;
        nser[slot] = sb + c;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kTreeThreads) {
        const int j = node[i];
        if (j < 0) continue;
        const int c = 4 * j + quad[i];
        if (cc[c] == 1) {
            const int slot = atomicAdd(s_nfin, 1);
            if (slot < cap_final) fin[slot] = ((unsigned long long)(0x7FFFFFFFu - (unsigned)(sb + c)) << 32) | (unsigned)i;
            node[i] = -1;
        } else {
            node[i] = nidx[c];
        }
    }
    __syncthreads();
    *ne = tot_some;
    return tot_big;
}

// scratch for the cell offsets of a level: the child-slot array of the level (4 x cap_nodes ints, sized for the cells at configure)
__device__ __forceinline__ int* cc_scratch(const TreeBuffers& B, const TreeLevel& V) { return B.nidx + 4 * (size_t)V.node_off; }

// status: [0 .. L) selected keypoints per level, [L .. 2L) candidates per level after the mask filter, [2L] error flag
__global__ void __launch_bounds__(kTreeThreads, 1)
k_tree_distribute(const __grid_constant__ TreeArgs A, TreeBuffers B, const uint32_t* __restrict__ cell_tmp, const int* __restrict__ cell_count,
                  const uint8_t* __restrict__ mask, int mask_w, int mask_h, SelKp* __restrict__ sel, int* __restrict__ status) {
    extern __shared__ __align__(16) unsigned long long s_sort[];   // kTreeSortSmem keys
    __shared__ int s_warp[33];
    __shared__ int s_nfin;
    __shared__ unsigned long long s_hit;
    const int l = blockIdx.x, L = A.num_levels;
    const TreeLevel& V = A.lv[l];
    if (threadIdx.x == 0) s_nfin = 0;
    uint32_t* fcw = B.fc + V.cand_off;
    int* node = B.node + V.cand_off;
    uint8_t* quad = B.quad + V.cand_off;
    // ---- the level's candidates in the reference's order: cell after cell (compute_fast_keypoints), row-major inside a cell
    const int ncell = V.cell_end - V.cell_begin;
    int n_raw;
    {
        int* coff = cc_scratch(B, V);                       // exclusive prefix of the cell counts (ncell + 1 entries)
        int b, e;
        tree_chunk(ncell, &b, &e);
        int sum = 0;
        for (int c = b; c < e; ++c) sum += cell_count[V.cell_begin + c];
        int run = tree_block_scan(sum, s_warp, &n_raw);
        for (int c = b; c < e; ++c) { coff[c] = run; run += cell_count[V.cell_begin + c]; }
        if (threadIdx.x == 0) coff[ncell] = n_raw;
        __syncthreads();
        if (n_raw > V.cand_cap) {
            if (threadIdx.x == 0) { status[2 * L] = 2; status[l] = 0; status[L + l] = n_raw; }
            return;
        }
        uint32_t* raw = mask ? reinterpret_cast<uint32_t*>(node) : fcw;    // the node array is free until the first assignment
        for (int i = threadIdx.x; i < n_raw; i += kTreeThreads) {
            int lo = 0, hi = ncell;                         // last cell whose offset is <= i
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (coff[mid] <= i) lo = mid; else hi = mid; }
            raw[i] = cell_tmp[(size_t)(V.cell_begin + lo) * kCellCap + (i - coff[lo])];
        }
        __syncthreads();
    }
    int n = n_raw;
    // ---- per-keypoint mask filter (order preserving)
    const uint32_t* fc = fcw;
    if (mask) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(node);
        const float scale = A.sf[l];
        int b, e;
        tree_chunk(n_raw, &b, &e);
        auto keep = [&](uint32_t c) {
            const unsigned y = (unsigned)(float)((float)kBorder + (float)tcy(c));
            const unsigned x = (unsigned)(float)((float)kBorder + (float)tcx(c));
            int my = (int)(y * scale), mx = (int)(x * scale);
            if (my >= mask_h) my = mask_h - 1;
            if (mx >= mask_w) mx = mask_w - 1;
            return mask[(size_t)my * mask_w + mx] != 0;
        };
        int kept = 0;
        for (int i = b; i < e; ++i) kept += keep(src[i]) ? 1 : 0;
        int total;
        int pos = tree_block_scan(kept, s_warp, &total);
        for (int i = b; i < e; ++i) {
            const uint32_t c = src[i];
            if (keep(c)) fcw[pos++] = c;
        }
        __syncthreads();
        n = total;
    }
    if (threadIdx.x == 0) status[L + l] = n;
    const int N = V.target;
    unsigned long long* fin = B.fin + V.final_off;
    if (n == 0) {
        if (threadIdx.x == 0) status[l] = 0;
        return;
    }
    int4* box[2] = {B.box + V.node_off, B.box + A.total_nodes + V.node_off};
    int* cnt[2] = {B.cnt + V.node_off, B.cnt + A.total_nodes + V.node_off};
    int* ser[2] = {B.ser + V.node_off, B.ser + A.total_nodes + V.node_off};
    int* cc = B.cc + 4 * (size_t)V.node_off;
    int* nidx = B.nidx + 4 * (size_t)V.node_off;
    unsigned* best = B.best + 5 * (size_t)V.node_off;
    int cur = 0;

    // ---- initial nodes (orb_extractor::initialize_nodes + the first assignment)
    const int nini = V.nini, gx = V.gx;
    for (int k = threadIdx.x; k < nini; k += kTreeThreads) cc[k] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kTreeThreads) {
        const uint32_t c = fc[i];
        const unsigned ix = (unsigned)((double)(float)tcx(c) / V.delta_x);
        const unsigned iy = (unsigned)((double)(float)tcy(c) / V.delta_y) * (unsigned)gx;
        unsigned k = ix + iy;
        if (k >= (unsigned)nini) k = nini - 1;
        node[i] = (int)k;
        atomicAdd(&cc[k], 1);
    }
    __syncthreads();
    int m, Lsize, sb = nini;
    {
        int b, e;
        tree_chunk(nini, &b, &e);
        int big = 0, some = 0;
        for (int k = b; k < e; ++k) { const int v = cc[k]; big += v > 1; some += v > 0; }
        int tot_big, tot_some;
        int run = tree_block_scan(big, s_warp, &tot_big);
        tree_block_scan(some, s_warp, &tot_some);
        for (int k = b; k < e; ++k) {
            const int v = cc[k];
            if (v <= 1) continue;
            const int slot = run++;             // the first sweep walks the initial nodes front to back
            nidx[k] = slot;
            const int ix = k % gx, iy = k / gx;
            box[0][slot] = make_int4((int)(V.delta_x * ix), (int)(V.delta_y * iy), (int)(V.delta_x * (ix + 1)), (int)(V.delta_y * (iy + 1)));
            cnt[0][slot] = v;
            ser[0][slot] = k;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += kTreeThreads) {
            const int k = node[i];
            if (cc[k] == 1) {
                const int slot = atomicAdd(&s_nfin, 1);
                if (slot < V.cap_final) fin[slot] = ((unsigned long long)(0x80000000u + (unsigned)k) << 32) | (unsigned)i;
                node[i] = -1;
            } else {
                node[i] = nidx[k];
            }
        }
        __syncthreads();
        m = tot_big; Lsize = tot_some;
    }

    // ---- whole-list sweeps
    bool largest_first = false;
    for (int guard = 0; guard < 64 && m > 0; ++guard) {
        const int prev = Lsize;
        tree_count_children(fc, n, node, quad, box[cur], m, cc);
        int ne;
        const int pl = tree_build_next(n, node, quad, box[cur], m, cc, nidx, box[cur ^ 1], cnt[cur ^ 1], ser[cur ^ 1], sb, s_warp, &ne,
                                       fin, V.cap_final, &s_nfin);
        Lsize = Lsize - m + ne; sb += 4 * m; m = pl; cur ^= 1;
        if (N <= Lsize || Lsize == prev) break;
        if (N < Lsize + 3 * m) { largest_first = true; break; }
    }
    // ---- largest nodes first, until the budget is reached
    for (int guard = 0; largest_first && guard < 64 && m > 0; ++guard) {
        const int prev = Lsize;
        // (count desc, serial desc) = (count desc, slot asc): the node array is in descending serial order
        int p2 = 2;
        while (p2 < m) p2 <<= 1;
        unsigned long long* keys = p2 <= kTreeSortSmem ? s_sort : B.pool + V.pool_off;
        for (int r = threadIdx.x; r < p2; r += kTreeThreads)
            keys[r] = r < m ? (((unsigned long long)(~(unsigned)cnt[cur][r])) << 32) | (unsigned)r : ~0ull;
        __syncthreads();
        tree_bitonic(keys, p2);
        for (int r = threadIdx.x; r < m; r += kTreeThreads) {
            const int j = (int)(unsigned)keys[r];
            box[cur ^ 1][r] = box[cur][j]; cnt[cur ^ 1][r] = cnt[cur][j]; ser[cur ^ 1][r] = ser[cur][j];
            nidx[j] = r;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += kTreeThreads) {
            const int j = node[i];
            if (j >= 0) node[i] = nidx[j];
        }
        cur ^= 1;
        __syncthreads();
        tree_count_children(fc, n, node, quad, box[cur], m, cc);
        // prefix over the sorted pool of (non-empty children - 1): where does the list reach the budget?
        if (threadIdx.x == 0) s_hit = ~0ull;
        int b, e;
        tree_chunk(m, &b, &e);
        auto grow = [&](int r) { return (cc[4 * r] > 0) + (cc[4 * r + 1] > 0) + (cc[4 * r + 2] > 0) + (cc[4 * r + 3] > 0) - 1; };
        int local = 0;
        for (int r = b; r < e; ++r) local += grow(r);
        int total;
        int run = tree_block_scan(local, s_warp, &total);       // (its barriers also publish s_hit)
        for (int r = b; r < e; ++r) {
            run += grow(r);
            if (Lsize + run >= N) { atomicMin(&s_hit, ((unsigned long long)(unsigned)r << 32) | (unsigned)run); break; }
        }
        __syncthreads();
        const unsigned long long hit = s_hit;
        __syncthreads();
        if (hit != ~0ull) {
            const int p = (int)(hit >> 32);
            // nodes 0..p are split (every child is final), nodes behind p stay whole
            for (int f = threadIdx.x; f < 5 * m; f += kTreeThreads) best[f] = 0;
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += kTreeThreads) {
                const int r = node[i];
                if (r < 0) continue;
                const int f = r <= p ? 4 * r + quad[i] : 4 * m + r;
                atomicMax(&best[f], ((unsigned)(fc[i] >> 24) << 24) | (0xFFFFFFu - (unsigned)i));
            }
            __syncthreads();
            for (int f = threadIdx.x; f < 4 * (p + 1) + (m - p - 1); f += kTreeThreads) {
                unsigned key, bb;
                if (f < 4 * (p + 1)) {
                    if (cc[f] == 0) continue;
                    key = 0x7FFFFFFFu - (unsigned)(sb + f); bb = best[f];
                } else {
                    const int r = p + 1 + (f - 4 * (p + 1));
                    key = 0x7FFFFFFFu - (unsigned)ser[cur][r]; bb = best[4 * m + r];
                }
                const int slot = atomicAdd(&s_nfin, 1);
                if (slot < V.cap_final) fin[slot] = ((unsigned long long)key << 32) | (0xFFFFFFu - (bb & 0xFFFFFFu));
            }
            __syncthreads();
            Lsize += (int)(unsigned)hit;
            m = 0;
            break;
        }
        int ne;
        const int pl = tree_build_next(n, node, quad, box[cur], m, cc, nidx, box[cur ^ 1], cnt[cur ^ 1], ser[cur ^ 1], sb, s_warp, &ne,
                                       fin, V.cap_final, &s_nfin);
        Lsize += total; sb += 4 * m; m = pl; cur ^= 1;
        if (Lsize == prev) break;
    }
    // ---- nodes never split: find_keypoints_with_max_response (first strict maximum in candidate order)
    if (m > 0) {
        for (int f = threadIdx.x; f < m; f += kTreeThreads) best[f] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += kTreeThreads) {
            const int r = node[i];
            if (r >= 0) atomicMax(&best[r], ((unsigned)(fc[i] >> 24) << 24) | (0xFFFFFFu - (unsigned)i));
        }
        __syncthreads();
        for (int r = threadIdx.x; r < m; r += kTreeThreads) {
            const int s = ser[cur][r];
            const unsigned key = s >= nini ? 0x7FFFFFFFu - (unsigned)s : 0x80000000u + (unsigned)s;
            const int slot = atomicAdd(&s_nfin, 1);
            if (slot < V.cap_final) fin[slot] = ((unsigned long long)key << 32) | (0xFFFFFFu - (best[r] & 0xFFFFFFu));
        }
    }
    __syncthreads();
    // ---- list order, selection records
    const int nfin = s_nfin;
    if (nfin > V.cap_final) {
        if (threadIdx.x == 0) { status[2 * L] = 1; status[l] = 0; }
        return;
    }
    int p2 = 2;
    while (p2 < nfin) p2 <<= 1;
    unsigned long long* keys = p2 <= kTreeSortSmem ? s_sort : fin;
    if (keys != fin)
        for (int r = threadIdx.x; r < nfin; r += kTreeThreads) keys[r] = fin[r];
    for (int r = nfin + threadIdx.x; r < p2; r += kTreeThreads) keys[r] = ~0ull;
    __syncthreads();
    tree_bitonic(keys, p2);
    for (int r = threadIdx.x; r < nfin; r += kTreeThreads) {
        const uint32_t c = fc[(unsigned)keys[r]];
        SelKp s;
        s.lx = (short)(tcx(c) + kBorder); s.ly = (short)(tcy(c) + kBorder);
        s.level = (unsigned char)l; s.score = (unsigned char)(c >> 24); s.pad = 0;
        sel[V.sel_off + r] = s;
    }
    if (threadIdx.x == 0) status[l] = nfin;
}

// ---------------------------------------------------------- orientation + descriptor
// One block (4 warps) per selected keypoint.  raw: 43x43 window centred on the keypoint
// (BORDER_REFLECT_101 at the level border); hb: horizontal 8.8 pass; bl: blurred 37x37 window.
// The patch of a keypoint away from the level border arrives as ONE TMA box (64 x 43 bytes from the 16-byte aligned column left of it).
// The selection arrives in per-level segments (first slot seg.off[l], status[l] records used): block b of the grid
// is slot b; its keypoint goes to output position (records of the lower levels) + (slot - seg.off[l]).
struct SelSegments { int off[kMaxLevels + 1]; };
__global__ void __launch_bounds__(128) k_orient_describe(const __grid_constant__ TmapArray pmaps, LevelTable T, const uint8_t* __restrict__ pyr,
                                                          const SelKp* __restrict__ sel, SelSegments seg, const int* __restrict__ status, int capacity, UMax umax,
                                                          ovs_keypoint* __restrict__ kps, uint8_t* __restrict__ desc, int* __restrict__ tma_timeout) {
    __shared__ __align__(128) uint8_t raw[kPatchBoxH][kPatchBoxW];   // window columns start at byte `sh` (0..15) of each row
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ unsigned short hb[43][38];
    __shared__ uint8_t bl[37][40];
    __shared__ float s_sincos[2];
    int level = 0, kp = 0;
    for (int l = 0; l < T.num_levels; ++l) {
        if ((int)blockIdx.x >= seg.off[l + 1]) { kp += status[l]; level = l + 1; }
    }
    if (level >= T.num_levels) return;
    const int slot = (int)blockIdx.x - seg.off[level];
    if (slot >= status[level]) return;
    kp += slot;
    if (kp >= capacity) return;
    const SelKp sk = sel[blockIdx.x];
    const int w = T.w[level], h = T.h[level], pitch = T.pitch[level];
    const uint8_t* img = pyr + T.off[level];
    const int lx = sk.lx, ly = sk.ly;

    const int wx0 = lx - 21, wy0 = ly - 21;
    const bool inside = wx0 >= 0 && wy0 >= 0 && wx0 + 43 <= w && wy0 + 43 <= h;
    const int sh = inside ? (wx0 & 15) : 0;
    if (inside) {
        if (!tma_box_2d(&raw[0][0], &pmaps.m[level], wx0 - sh, wy0, kPatchBoxH * kPatchBoxW, &mbar)) {
            if (threadIdx.x == 0) *tma_timeout = 1;
            return;
        }
    } else {
        for (int i = threadIdx.x; i < 43 * 43; i += 128) {
            const int r = i / 43, c = i - r * 43;
            const int gy = ovs::reflect101(wy0 + r, h), gx = ovs::reflect101(wx0 + c, w);
            raw[r][c] = __ldg(img + (size_t)gy * pitch + gx);
        }
    }
    __syncthreads();

    constexpr int gk[7] = OVS_GAUSS7;
    for (int i = threadIdx.x; i < 43 * 37; i += 128) {
        const int r = i / 37, c = i - r * 37;
        int s = 0;
#pragma unroll
        for (int j = 0; j < 7; ++j) s += gk[j] * raw[r][sh + c + j];
        hb[r][c] = (unsigned short)s;
    }
    if (threadIdx.x < 32) {
        // orb_extractor::ic_angle: lane <-> patch row v = lane - 15
        const int lane = threadIdx.x;
        int rowsum = 0, rowu = 0;
        if (lane < 31) {
            const int v = lane - 15;
            const int d = umax.v[v < 0 ? -v : v];
            const uint8_t* p = &raw[21 + v][21 + sh];
            for (int u = -d; u <= d; ++u) {
                const int val = p[u];
                rowsum += val;
                rowu += u * val;
            }
            rowsum *= v;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            rowsum += __shfl_xor_sync(0xffffffffu, rowsum, o);
            rowu += __shfl_xor_sync(0xffffffffu, rowu, o);
        }
        if (lane == 0) {
            const float angle = ovs::fast_atan2_deg((float)rowsum, (float)rowu);
            float sn, cs;
            ovs::angle_sincos(angle, &sn, &cs);
            s_sincos[0] = sn; s_sincos[1] = cs;
            ovs_keypoint o;
            const float fx = (float)lx, fy = (float)ly;
            o.x = level == 0 ? fx : ovs::fmul(fx, T.scale[level]);
            o.y = level == 0 ? fy : ovs::fmul(fy, T.scale[level]);
            o.size = T.kp_size[level];
            o.angle = angle;
            o.response = (float)sk.score;
            o.octave = level;
            o.class_id = -1;
            kps[kp] = o;
        }
    }
    __syncthreads();

    for (int i = threadIdx.x; i < 37 * 37; i += 128) {
        const int r = i / 37, c = i - r * 37;
        unsigned s = 0;
#pragma unroll
        for (int j = 0; j < 7; ++j) s += (unsigned)gk[j] * hb[r + j][c];
        bl[r][c] = (uint8_t)((s + 32768u) >> 16);
    }
    __syncthreads();

    const float sn = s_sincos[0], cs = s_sincos[1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int round = 0; round < 2; ++round) {
        const int b = round * 128 + threadIdx.x;
        const signed char* p = c_pattern[b];
        int r0, c0, r1, c1;
        ovs::brief_offset(p[0], p[1], sn, cs, &r0, &c0);
        ovs::brief_offset(p[2], p[3], sn, cs, &r1, &c1);
        const int t0 = bl[18 + r0][18 + c0], t1 = bl[18 + r1][18 + c1];
        const unsigned word = __ballot_sync(0xffffffffu, t0 < t1);
        if (lane == 0) *reinterpret_cast<unsigned*>(desc + (size_t)kp * 32 + (round * 4 + wid) * 4) = word;
    }
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

// ================================================================================ handle
struct ovs_extractor {
    ovs_orb_params P{};
    int device = 0;
    cudaStream_t stream = nullptr;
    std::vector<float> mask_rects;
    std::vector<uint8_t> rect_mask;
    float sf[kMaxLevels]{}, inv_sf[kMaxLevels]{}, sigma_sq[kMaxLevels]{}, inv_sigma_sq[kMaxLevels]{};
    unsigned per_level[kMaxLevels]{};
    UMax umax{};
    int max_out = 0;

    // geometry-dependent state
    int img_w = 0, img_h = 0;
    LevelTable T{};
    TmapArray tmaps{}, tmaps_score{}, tmaps_patch{};   // FAST tiles (pyramid), NMS windows (score map), descriptor patches (pyramid)
    int* d_tma_timeout = nullptr;
    size_t pyr_bytes = 0;
    uint8_t* d_pyr = nullptr;
    uint8_t* d_score = nullptr;
    int2* d_tabs = nullptr;
    std::vector<PyrGroup> pyr_groups;           // pyramid launch groups (levels per launch) and their dynamic shared memory
    std::vector<size_t> pyr_smem;
    size_t xtab_off[kMaxLevels]{}, ytab_off[kMaxLevels]{};
    std::vector<CellInfo> h_cells;
    std::vector<int> cell_roi;  // per cell: min_x, min_y, max_x, max_y (ROI, for the mask test)
    int level_cell_begin[kMaxLevels + 1]{};
    CellInfo* d_cells = nullptr;
    uint32_t* d_cell_tmp = nullptr;
    int* d_cell_count = nullptr;
    uint8_t* d_cell_skip = nullptr;
    uint8_t* h_cell_skip = nullptr;   // pinned
    int cand_cap = 0;
    // device status block, copied to h_status at the end of every call: [0, 2L] tree status (selected per level, candidates per
    // level after the mask filter, error flag: 1 selection overflow, 2 candidate overflow), [kStatTma] TMA time-out
    int* d_status = nullptr;
    int* h_status = nullptr;          // pinned
    TreeArgs targs{};
    TreeBuffers tbuf{};
    void* d_tree = nullptr;           // one allocation behind tbuf
    SelSegments seg{};
    SelKp* d_sel = nullptr;           // selection segments, seg.off[L] records
    uint8_t* d_mask_rect = nullptr;   // the handle's rectangle mask (level-0 geometry)
    uint8_t* d_mask_call = nullptr;   // a caller's mask of the current call
    bool last_masked = false;
    uint8_t* h_img = nullptr;         // pinned staging for pageable input
    ovs::HostUpload color;            // colour / raw stereo input staging (extract_host_color, extract_host_rectified)
    uint8_t* d_und = nullptr; size_t und_bytes = 0;                                   // scratch of ovs_undistort_keypoints_host
    size_t h_img_bytes = 0;

    // size-independent buffers
    ovs_keypoint* d_kps = nullptr;
    uint8_t* d_desc = nullptr;
    ovs_keypoint* h_kps = nullptr;    // pinned
    uint8_t* h_desc = nullptr;        // pinned

    cudaEvent_t ev[8]{};
    float timings[8]{};
};

namespace {

void free_geometry(ovs_extractor* h) {
    cudaFree(h->d_pyr); cudaFree(h->d_score); cudaFree(h->d_tabs); cudaFree(h->d_cells);
    cudaFree(h->d_cell_tmp); cudaFree(h->d_cell_count); cudaFree(h->d_cell_skip);
    cudaFreeHost(h->h_cell_skip); cudaFreeHost(h->h_img);
    cudaFree(h->d_tree); cudaFree(h->d_sel); cudaFree(h->d_mask_rect); cudaFree(h->d_mask_call);
    h->d_pyr = h->d_score = nullptr; h->d_tabs = nullptr; h->d_cells = nullptr; h->d_cell_tmp = nullptr;
    h->d_cell_count = nullptr; h->d_cell_skip = nullptr; h->h_cell_skip = nullptr;
    h->d_tree = nullptr; h->d_sel = nullptr; h->d_mask_rect = h->d_mask_call = nullptr;
    h->h_img = nullptr; h->h_img_bytes = 0;
}

// cv::resize coefficient tables for src extent `ssize` -> dst extent `dsize`.
void make_resize_table(int ssize, int dsize, bool clamp_hi, std::vector<int2>& tab) {
    tab.resize(dsize);
    const double inv_scale = (double)dsize / ssize;
    const double scale = 1. / inv_scale;
    for (int d = 0; d < dsize; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        f -= s;
        if (clamp_hi) {  // x direction: cv::resize folds the clamp into the table
            if (s < 0) { f = 0; s = 0; }
            if (s >= ssize - 1) { f = 0; s = ssize - 1; }
        }
        const int a0 = (int)lrintf((1.f - f) * 2048.f), a1 = (int)lrintf(f * 2048.f);
        tab[d] = make_int2(s, (a0 & 0xffff) | (a1 << 16));
    }
}

int configure(ovs_extractor* h, int w, int hgt) {
    if (h->img_w == w && h->img_h == hgt) return OVS_OK;
    OVS_REQUIRE(w >= 2 * kBorder + 8 && hgt >= 2 * kBorder + 8, OVS_ERR_INVALID_ARG, "image %dx%d too small", w, hgt);
    OVS_REQUIRE(w - 2 * kBorder < 4096 && hgt - 2 * kBorder < 4096, OVS_ERR_UNSUPPORTED,
                "image %dx%d exceeds the 4096 px candidate coordinate range", w, hgt);
    free_geometry(h);
    h->img_w = h->img_h = 0;
    const int L = (int)h->P.num_levels;
    LevelTable& T = h->T;
    T.num_levels = L;
    size_t off = 0;
    int tiles = 0;
    for (int l = 0; l < L; ++l) {
        if (l == 0) { T.w[l] = w; T.h[l] = hgt; }
        else {
            const double s = (double)h->sf[l];
            T.w[l] = (int)std::round(w * 1.0 / s);
            T.h[l] = (int)std::round(hgt * 1.0 / s);
        }
        OVS_REQUIRE(T.w[l] >= 8 && T.h[l] >= 8, OVS_ERR_INVALID_ARG, "pyramid level %d degenerates (%dx%d)", l, T.w[l], T.h[l]);
        T.pitch[l] = (int)align_up((size_t)T.w[l], 128);
        T.off[l] = (unsigned)off;
        off += align_up((size_t)T.pitch[l] * T.h[l], 256);
        T.tiles_x[l] = (T.w[l] + kTileW - 1) / kTileW;
        T.tile_begin[l] = tiles;
        tiles += T.tiles_x[l] * ((T.h[l] + kTileH - 1) / kTileH);
        T.scale[l] = h->sf[l];
        T.kp_size[l] = (float)(unsigned)(31 * h->sf[l]);
    }
    T.tile_begin[L] = tiles;
    {
        // distribute_keypoints_via_tree returns at most the level's budget plus 3 (the last split) -- but never fewer leaves than its
        // first pass creates: every initial node (round(aspect) of them) is split unconditionally.  A very wide or very tall image
        // with a small budget can therefore return more keypoints than max_num_keypts + slack: the handle's buffers follow.
        long worst = 0;
        for (int l = 0; l < L; ++l) {
            const double rw = T.w[l] - 2 * kBorder, rh = T.h[l] - 2 * kBorder;
            long nini = 1;
            if (rw > 0 && rh > 0) nini = std::max(1L, (long)std::lround(rw > rh ? rw / rh : rh / rw));
            worst += std::max((long)h->per_level[l], 4 * nini) + 3;
        }
        if (worst > (long)h->max_out) {
            // grow the keypoint buffers of the handle for this geometry (the caller's own capacity still bounds what one call returns)
            OVS_REQUIRE(worst < (1L << 24), OVS_ERR_UNSUPPORTED, "image %dx%d: degenerate aspect ratio", w, hgt);
            OVS_CUDA_CHECK(ovs::sync_stream(h->stream));
            cudaFree(h->d_kps); cudaFree(h->d_desc); cudaFreeHost(h->h_kps); cudaFreeHost(h->h_desc);
            h->d_kps = nullptr; h->d_desc = nullptr; h->h_kps = nullptr; h->h_desc = nullptr;
            h->max_out = (int)worst;
            OVS_CUDA_CHECK(cudaMalloc(&h->d_kps, (size_t)h->max_out * sizeof(ovs_keypoint)));
            OVS_CUDA_CHECK(cudaMalloc(&h->d_desc, (size_t)h->max_out * 32));
            OVS_CUDA_CHECK(cudaHostAlloc(&h->h_kps, (size_t)h->max_out * sizeof(ovs_keypoint), cudaHostAllocDefault));
            OVS_CUDA_CHECK(cudaHostAlloc(&h->h_desc, (size_t)h->max_out * 32, cudaHostAllocDefault));
        }
    }
    h->pyr_bytes = off;
    OVS_CUDA_CHECK(cudaMalloc(&h->d_pyr, off));
    OVS_CUDA_CHECK(cudaMalloc(&h->d_score, off));
    OVS_CUDA_CHECK(cudaMemsetAsync(h->d_pyr, 0, off, h->stream));
    OVS_CUDA_CHECK(cudaMemsetAsync(h->d_score, 0, off, h->stream));

    // TMA descriptors of the pyramid levels (k_fast_score stages its tiles with them)
    {
        typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                      const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        OVS_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        OVS_REQUIRE(fn && qres == cudaDriverEntryPointSuccess, OVS_ERR_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
        for (int l = 0; l < L; ++l) {
            const cuuint64_t gdim[2] = {(cuuint64_t)T.pitch[l], (cuuint64_t)T.h[l]};
            const cuuint64_t gstride[1] = {(cuuint64_t)T.pitch[l]};
            const cuuint32_t box[2] = {(cuuint32_t)kTmaBoxW, (cuuint32_t)(kTileH + 6)};
            const cuuint32_t estride[2] = {1, 1};
            const CUresult r = reinterpret_cast<encode_fn>(fn)(&h->tmaps.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, h->d_pyr + T.off[l], gdim, gstride, box, estride,
                                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            OVS_REQUIRE(r == CUDA_SUCCESS, OVS_ERR_CUDA, "cuTensorMapEncodeTiled failed for level %d (CUresult %d)", l, (int)r);
            const cuuint32_t box_s[2] = {(cuuint32_t)kNmsBoxW, (cuuint32_t)kNmsBoxH}, box_p[2] = {(cuuint32_t)kPatchBoxW, (cuuint32_t)kPatchBoxH};
            const CUresult rs = reinterpret_cast<encode_fn>(fn)(&h->tmaps_score.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, h->d_score + T.off[l], gdim, gstride, box_s,
                                                                estride, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                                CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            const CUresult rp = reinterpret_cast<encode_fn>(fn)(&h->tmaps_patch.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, h->d_pyr + T.off[l], gdim, gstride, box_p,
                                                                estride, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                                CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            OVS_REQUIRE(rs == CUDA_SUCCESS && rp == CUDA_SUCCESS, OVS_ERR_CUDA, "cuTensorMapEncodeTiled (window / patch boxes) failed for level %d (%d, %d)", l, (int)rs, (int)rp);
        }
    }

    // resize tables
    std::vector<int2> all, tab;
    for (int l = 1; l < L; ++l) {
        make_resize_table(T.w[l - 1], T.w[l], true, tab);
        h->xtab_off[l] = all.size(); all.insert(all.end(), tab.begin(), tab.end());
        make_resize_table(T.h[l - 1], T.h[l], false, tab);
        h->ytab_off[l] = all.size(); all.insert(all.end(), tab.begin(), tab.end());
    }
    if (!all.empty()) {
        OVS_CUDA_CHECK(cudaMalloc(&h->d_tabs, all.size() * sizeof(int2)));
        OVS_CUDA_CHECK(cudaMemcpy(h->d_tabs, all.data(), all.size() * sizeof(int2), cudaMemcpyHostToDevice));
    }
    // pyramid launch groups: up to 3 levels from the full-size image, then up to 4 per launch; a group shrinks until the regions its
    // CTAs keep in shared memory fit in 40 KB (they grow with the scale factor)
    h->pyr_groups.clear(); h->pyr_smem.clear();
    for (int src = 0; src < L - 1;) {
        int nlev = std::min(L - 1 - src, src == 0 ? 3 : kPyrMaxGroup);
        for (;; --nlev) {
            PyrGroup G{};
            G.src_level = src; G.nlev = nlev;
            const int last = src + nlev;
            G.tiles_x = (T.w[last] + kPyrTW - 1) / kPyrTW; G.tiles_y = (T.h[last] + kPyrTH - 1) / kPyrTH;
            for (int k = 1; k <= nlev; ++k) { G.xtab_off[k] = (unsigned)h->xtab_off[src + k]; G.ytab_off[k] = (unsigned)h->ytab_off[src + k]; }
            // extent bounds of the intermediate regions: the same interval recurrences as the kernel, over every tile column / row
            int bw[kPyrMaxGroup + 1] = {0}, bh[kPyrMaxGroup + 1] = {0};
            for (int dim = 0; dim < 2; ++dim) {
                const int ntile = dim ? G.tiles_y : G.tiles_x, tsize = dim ? kPyrTH : kPyrTW;
                for (int t = 0; t < ntile; ++t) {
                    PyrSpan D;
                    const int ext_last = dim ? T.h[last] : T.w[last];
                    D.lo = D.olo = t * tsize; D.hi = D.ohi = std::min(ext_last, (t + 1) * tsize);
                    for (int k = nlev - 1; k >= 1; --k) {
                        const int l = src + k;
                        const int2* tab = all.data() + (dim ? h->ytab_off[l + 1] : h->xtab_off[l + 1]);
                        D = pyr_source_span(D, tab, dim ? T.h[l] : T.w[l], t == 0, t == ntile - 1);
                        int& m = dim ? bh[k] : bw[k];
                        m = std::max(m, D.hi - D.lo);
                    }
                }
            }
            size_t smem = 0;
            for (int k = 1; k < nlev; ++k) { G.buf_w[k] = bw[k]; G.buf_h[k] = bh[k]; G.buf_off[k] = (int)smem; smem += align_up((size_t)bw[k] * bh[k], 16); }
            if (smem <= 40 * 1024 || nlev == 1) { h->pyr_groups.push_back(G); h->pyr_smem.push_back(smem); break; }
        }
        src += h->pyr_groups.back().nlev;
    }

    // detection cells, in the order compute_fast_keypoints visits them.  A level's candidate slice holds what its cells can emit at
    // most: the survivors of one cell's strict-max NMS are pairwise non-adjacent, so an rw x rh band yields at most
    // ceil(rw / 2) * ceil(rh / 2) of them (kCellCap for a full cell).  The bands of neighbouring cells abut and pixels outside a band
    // count as 0, so survivors on either side of a seam can be adjacent: the per-cell bounds add up.  A dense image comes close to a
    // quarter of the level's pixels (a lattice of bright pixels at (x + 2 y) % 4 == 0 does).
    h->h_cells.clear(); h->cell_roi.clear();
    size_t cand_cap = 0;
    size_t level_cand_cap[kMaxLevels] = {};
    for (int l = 0; l < L; ++l) {
        h->level_cell_begin[l] = (int)h->h_cells.size();
        if (T.w[l] <= 2 * kBorder || T.h[l] <= 2 * kBorder) continue;
        const unsigned min_bx = kBorder, min_by = kBorder;
        const unsigned max_bx = T.w[l] - kBorder, max_by = T.h[l] - kBorder;
        const unsigned width = max_bx - min_bx, height = max_by - min_by;
        const unsigned num_cols = (unsigned)std::ceil((double)(width / kCell)) + 1;
        const unsigned num_rows = (unsigned)std::ceil((double)(height / kCell)) + 1;
        for (unsigned i = 0; i < num_rows; ++i) {
            const unsigned min_y = min_by + i * kCell;
            if (max_by <= min_y + kOverlap) continue;  // max_border_y - overlap <= min_y (unsigned-safe)
            unsigned max_y = min_y + kCell + kOverlap;
            if (max_by < max_y) max_y = max_by;
            for (unsigned j = 0; j < num_cols; ++j) {
                const unsigned min_x = min_bx + j * kCell;
                if (max_bx <= min_x + kOverlap) continue;
                unsigned max_x = min_x + kCell + kOverlap;
                if (max_bx < max_x) max_x = max_bx;
                CellInfo ci;
                ci.rx0 = (short)(min_x + 3); ci.ry0 = (short)(min_y + 3);
                ci.rw = (short)(max_x - min_x - 6); ci.rh = (short)(max_y - min_y - 6);
                ci.level = l;
                h->h_cells.push_back(ci);
                h->cell_roi.push_back((int)min_x); h->cell_roi.push_back((int)min_y);
                h->cell_roi.push_back((int)max_x); h->cell_roi.push_back((int)max_y);
                level_cand_cap[l] += (size_t)((ci.rw + 1) / 2) * ((ci.rh + 1) / 2);
            }
        }
        // the tree kernel keeps a candidate's index within its level in 24 bits (the low bits of its best-response keys)
        OVS_REQUIRE(level_cand_cap[l] < (1u << 24), OVS_ERR_UNSUPPORTED, "image %dx%d: more than 2^24 candidate slots at level %d", w, hgt, l);
        cand_cap += level_cand_cap[l];
    }
    h->level_cell_begin[L] = (int)h->h_cells.size();
    const size_t nc = h->h_cells.size();
    if (nc) {
        OVS_CUDA_CHECK(cudaMalloc(&h->d_cells, nc * sizeof(CellInfo)));
        OVS_CUDA_CHECK(cudaMemcpy(h->d_cells, h->h_cells.data(), nc * sizeof(CellInfo), cudaMemcpyHostToDevice));
        OVS_CUDA_CHECK(cudaMalloc(&h->d_cell_tmp, nc * kCellCap * sizeof(uint32_t)));
        OVS_CUDA_CHECK(cudaMalloc(&h->d_cell_count, nc * sizeof(int)));
        OVS_CUDA_CHECK(cudaMalloc(&h->d_cell_skip, nc));
        OVS_CUDA_CHECK(cudaHostAlloc(&h->h_cell_skip, nc, cudaHostAllocDefault));
    }
    h->cand_cap = (int)cand_cap;

    // tree distribution: initial nodes per level (orb_extractor::initialize_nodes), scratch, selection segments
    {
        TreeArgs& A = h->targs;
        A = TreeArgs{};
        A.num_levels = L;
        size_t nodes = 0, fins = 0, pools = 0, cands = 0;
        int sel = 0;
        auto pow2_at_least = [](int v) { int p = 2; while (p < v) p <<= 1; return p; };
        for (int l = 0; l < L; ++l) {
            TreeLevel& V = A.lv[l];
            A.sf[l] = h->sf[l];
            V.target = (int)h->per_level[l];
            V.cell_begin = h->level_cell_begin[l]; V.cell_end = h->level_cell_begin[l + 1];
            V.cand_off = (int)cands; V.cand_cap = (int)level_cand_cap[l];
            cands += V.cand_cap;
            const int min_x = kBorder, max_x = T.w[l] - kBorder, min_y = kBorder, max_y = T.h[l] - kBorder;
            V.gx = 1; V.nini = 1; V.delta_x = 1; V.delta_y = 1;
            if (max_x > min_x && max_y > min_y) {
                const double ratio = (double)(max_x - min_x) / (max_y - min_y);
                unsigned gx, gy;
                if (ratio > 1) {
                    gx = (unsigned)std::round(ratio); gy = 1;
                    V.delta_x = (double)(max_x - min_x) / gx; V.delta_y = max_y - min_y;
                } else {
                    gx = 1; gy = (unsigned)std::round(1 / ratio);
                    V.delta_x = max_x - min_x; V.delta_y = (double)(max_y - min_y) / gy;
                }
                V.gx = (int)gx; V.nini = (int)(gx * gy);
            }
            // a sweep is only started while the list can still take three more nodes per pool node, so neither the nodes of a pass nor
            // the final list exceed max(budget, 4 x initial nodes) (+3 for the last split)
            const int bound = std::max(V.target, 4 * V.nini);
            // (the child-slot array, 4 x cap_nodes ints, doubles as the scratch of the level's cell offsets)
            V.cap_nodes = std::max(bound + 8, (V.cell_end - V.cell_begin + 8) / 4); V.cap_final = bound + 4;
            V.final_pow2 = pow2_at_least(V.cap_final); V.pool_pow2 = pow2_at_least(V.cap_nodes);
            V.node_off = (int)nodes; V.final_off = (int)fins; V.pool_off = (int)pools; V.sel_off = sel;
            h->seg.off[l] = sel;
            nodes += V.cap_nodes; fins += V.final_pow2; pools += V.pool_pow2; sel += V.cap_final;
        }
        for (int l = L; l <= kMaxLevels; ++l) h->seg.off[l] = sel;
        A.total_nodes = (int)nodes;
        const size_t b_box = 2 * nodes * sizeof(int4), b_fin = fins * 8, b_pool = pools * 8, b_i = nodes * sizeof(int);
        const size_t total = b_box + b_fin + b_pool + (2 + 2 + 4 + 4 + 5) * b_i + cand_cap * (4 + 4 + 1) + 64;
        OVS_CUDA_CHECK(cudaMalloc(&h->d_tree, total));
        char* q = static_cast<char*>(h->d_tree);
        TreeBuffers& B = h->tbuf;
        B.box = reinterpret_cast<int4*>(q); q += b_box;
        B.fin = reinterpret_cast<unsigned long long*>(q); q += b_fin;
        B.pool = reinterpret_cast<unsigned long long*>(q); q += b_pool;
        B.cnt = reinterpret_cast<int*>(q); q += 2 * b_i;
        B.ser = reinterpret_cast<int*>(q); q += 2 * b_i;
        B.cc = reinterpret_cast<int*>(q); q += 4 * b_i;
        B.nidx = reinterpret_cast<int*>(q); q += 4 * b_i;
        B.best = reinterpret_cast<unsigned*>(q); q += 5 * b_i;
        B.fc = reinterpret_cast<uint32_t*>(q); q += cand_cap * 4;
        B.node = reinterpret_cast<int*>(q); q += cand_cap * 4;
        B.quad = reinterpret_cast<uint8_t*>(q);
        OVS_CUDA_CHECK(cudaMalloc(&h->d_sel, (size_t)std::max(sel, 1) * sizeof(SelKp)));
        OVS_CUDA_CHECK(cudaFuncSetAttribute(k_tree_distribute, cudaFuncAttributeMaxDynamicSharedMemorySize, kTreeSortSmem * 8));
    }
    h->h_img_bytes = (size_t)w * hgt;
    OVS_CUDA_CHECK(cudaHostAlloc(&h->h_img, h->h_img_bytes, cudaHostAllocDefault));

    // orb_extractor::create_rectangle_mask (once per image size)
    h->rect_mask.clear();
    if (!h->mask_rects.empty()) {
        h->rect_mask.assign((size_t)w * hgt, 255);
        for (size_t r = 0; r + 3 < h->mask_rects.size(); r += 4) {
            const float* q = &h->mask_rects[r];
            const unsigned x0 = (unsigned)(w * q[0]), x1 = (unsigned)(w * q[1]);
            const unsigned y0 = (unsigned)(hgt * q[2]), y1 = (unsigned)(hgt * q[3]);
            for (unsigned y = y0; y < y1 && y < (unsigned)hgt; ++y)
                for (unsigned x = x0; x < x1 && x < (unsigned)w; ++x) h->rect_mask[(size_t)y * w + x] = 0;
        }
        OVS_CUDA_CHECK(cudaMalloc(&h->d_mask_rect, (size_t)w * hgt));
        OVS_CUDA_CHECK(cudaMemcpy(h->d_mask_rect, h->rect_mask.data(), (size_t)w * hgt, cudaMemcpyHostToDevice));
    }
    OVS_CUDA_CHECK(ovs::sync_stream(h->stream));
    h->img_w = w; h->img_h = hgt;
    return OVS_OK;
}

inline bool mask_is_zero(const uint8_t* mask, int mw, int mh, size_t mpitch, unsigned y, unsigned x, float scale) {
    int my = (int)(y * scale), mx = (int)(x * scale);
    if (my >= mh) my = mh - 1;
    if (mx >= mw) mx = mw - 1;
    return mask[(size_t)my * mpitch + mx] == 0;
}

// Everything between "level 0 is in d_pyr" and "keypoints + descriptors are in d_kps_out / d_desc_out (device)" is ENQUEUED
// here; nothing waits for the device.  The caller synchronises once and reads the outcome with finish_pipeline().
int run_pipeline(ovs_extractor* h, const uint8_t* mask, size_t mask_pitch,
                 ovs_keypoint* d_kps_out, uint8_t* d_desc_out, int capacity) {
    const LevelTable& T = h->T;
    const int L = T.num_levels;
    cudaStream_t st = h->stream;
    const int ncells = (int)h->h_cells.size();

    // --- pyramid
    for (size_t g = 0; g < h->pyr_groups.size(); ++g) {
        const PyrGroup& G = h->pyr_groups[g];
        k_pyramid_group<<<G.tiles_x * G.tiles_y, 256, h->pyr_smem[g], st>>>(h->d_pyr, T, h->d_tabs, G);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[2], st));

    // --- FAST score over all levels (status block cleared: flags of a previous call must not stick to the handle)
    OVS_CUDA_CHECK(cudaMemsetAsync(h->d_status, 0, kStatInts * sizeof(int), st));
    k_fast_score<<<T.tile_begin[L], 256, 0, st>>>(h->tmaps, T, h->d_score, (int)h->P.min_fast_thr, h->d_tma_timeout);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[3], st));

    // --- cells: mask test on the four ROI corners (host, on the caller's mask), NMS
    const uint8_t* eff_mask = mask;
    size_t eff_pitch = mask_pitch;
    const uint8_t* d_mask = nullptr;
    if (eff_mask) {
        if (!h->d_mask_call) OVS_CUDA_CHECK(cudaMalloc(&h->d_mask_call, (size_t)h->img_w * h->img_h));
        OVS_CUDA_CHECK(cudaMemcpy2DAsync(h->d_mask_call, h->img_w, mask, mask_pitch, h->img_w, h->img_h, cudaMemcpyHostToDevice, st));
        d_mask = h->d_mask_call;
    } else if (!h->rect_mask.empty()) {
        eff_mask = h->rect_mask.data(); eff_pitch = (size_t)h->img_w;
        d_mask = h->d_mask_rect;
    }
    h->last_masked = d_mask != nullptr;
    if (ncells) {
        const uint8_t* d_skip = nullptr;
        if (eff_mask) {
            for (int c = 0; c < ncells; ++c) {
                const int* roi = &h->cell_roi[4 * c];
                const float s = h->sf[h->h_cells[c].level];
                h->h_cell_skip[c] = mask_is_zero(eff_mask, h->img_w, h->img_h, eff_pitch, roi[1], roi[0], s)
                                    || mask_is_zero(eff_mask, h->img_w, h->img_h, eff_pitch, roi[3], roi[0], s)
                                    || mask_is_zero(eff_mask, h->img_w, h->img_h, eff_pitch, roi[1], roi[2], s)
                                    || mask_is_zero(eff_mask, h->img_w, h->img_h, eff_pitch, roi[3], roi[2], s);
            }
            OVS_CUDA_CHECK(cudaMemcpyAsync(h->d_cell_skip, h->h_cell_skip, ncells, cudaMemcpyHostToDevice, st));
            d_skip = h->d_cell_skip;
        }
        k_cell_nms<<<ncells, 256, 0, st>>>(h->tmaps_score, T, h->d_cells, d_skip, (int)h->P.ini_fast_thr, h->d_cell_tmp, h->d_cell_count, h->d_tma_timeout);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[4], st));

    // --- ordered candidate list of each level, per-keypoint mask filter, tree distribution: one CTA per level
    if (ncells) {
        k_tree_distribute<<<L, kTreeThreads, kTreeSortSmem * 8, st>>>(h->targs, h->tbuf, h->d_cell_tmp, h->d_cell_count, d_mask, h->img_w, h->img_h,
                                                                       h->d_sel, h->d_status);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[5], st));

    // --- orientation + descriptors: one block per selection slot, the unused slots of a level's segment leave at once
    if (ncells && h->seg.off[L] > 0 && capacity > 0) {
        k_orient_describe<<<h->seg.off[L], 128, 0, st>>>(h->tmaps_patch, T, h->d_pyr, h->d_sel, h->seg, h->d_status, capacity, h->umax,
                                                         d_kps_out, d_desc_out, h->d_tma_timeout);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[6], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_status, h->d_status, kStatInts * sizeof(int), cudaMemcpyDeviceToHost, st));
    return OVS_OK;
}

// After the caller's synchronisation: the verdict of the device-side pipeline.
int finish_pipeline(ovs_extractor* h, int capacity, int* num_out) {
    const int L = h->T.num_levels;
    const int* S = h->h_status;
    OVS_REQUIRE(S[kStatTma] == 0, OVS_ERR_CUDA, "TMA tile load timed out (k_fast_score / k_cell_nms / k_orient_describe)");
    OVS_REQUIRE(S[2 * L] != 2, OVS_ERR_OVERFLOW, "FAST candidate buffer overflow");
    OVS_REQUIRE(S[2 * L] == 0, OVS_ERR_OVERFLOW, "tree distribution returned more keypoints than its level segment holds");
    int nsel = 0;
    for (int l = 0; l < L; ++l) nsel += S[l];
    *num_out = nsel;
    OVS_REQUIRE(nsel <= capacity, OVS_ERR_CAPACITY, "output capacity %d < %d keypoints", capacity, nsel);
    return OVS_OK;
}

int collect_timings(ovs_extractor* h, std::chrono::steady_clock::time_point t_begin) {
    float ms = 0;
    auto el = [&](int a, int b) { ms = 0; cudaEventElapsedTime(&ms, h->ev[a], h->ev[b]); return ms * 1000.f; };
    h->timings[0] = el(0, 1);
    h->timings[1] = el(1, 2);
    h->timings[2] = el(2, 3);
    h->timings[3] = el(3, 4);
    h->timings[4] = el(4, 5);
    h->timings[5] = el(5, 6);
    h->timings[6] = el(6, 7);
    h->timings[7] = std::chrono::duration<float, std::micro>(std::chrono::steady_clock::now() - t_begin).count();
    return OVS_OK;
}

// The host entries once level 0 has been queued on the handle's stream: the pipeline, the copies of what the caller can take,
// one host wait, the verdict and the outputs.
int extract_to_host(ovs_extractor* h, const uint8_t* mask, size_t mask_pitch, ovs_keypoint* keypts_out, uint8_t* descriptors_out,
                    int capacity, int* num_out, std::chrono::steady_clock::time_point t_begin) {
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    // the number of keypoints is known to the device only: the copies cover what the caller can take
    const int bound = std::min(capacity, h->max_out);
    int rc = run_pipeline(h, mask, mask_pitch, h->d_kps, h->d_desc, bound);
    if (rc != OVS_OK) return rc;
    if (bound) {
        OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_kps, h->d_kps, (size_t)bound * sizeof(ovs_keypoint), cudaMemcpyDeviceToHost, st));
        OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_desc, h->d_desc, (size_t)bound * 32, cudaMemcpyDeviceToHost, st));
    }
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[7], st));
    OVS_CUDA_CHECK(ovs::sync_event(h->ev[7]));
    rc = finish_pipeline(h, bound, num_out);
    if (rc != OVS_OK) return rc;
    const int n = *num_out;
    if (n) {
        memcpy(keypts_out, h->h_kps, (size_t)n * sizeof(ovs_keypoint));
        memcpy(descriptors_out, h->h_desc, (size_t)n * 32);
    }
    return collect_timings(h, t_begin);
}

}  // namespace

// ================================================================================ C ABI
extern "C" int ovs_extractor_create(const ovs_orb_params* params, const float* mask_rects, int num_mask_rects,
                                    int device, ovs_extractor** out) {
    OVS_REQUIRE(params && out, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(params->num_levels >= 1 && params->num_levels <= kMaxLevels, OVS_ERR_INVALID_ARG, "num_levels must be 1..16");
    OVS_REQUIRE(params->scale_factor > 1.0f || params->num_levels == 1, OVS_ERR_INVALID_ARG, "scale_factor must be > 1");
    OVS_REQUIRE(params->min_fast_thr >= 1 && params->min_fast_thr <= params->ini_fast_thr && params->ini_fast_thr <= 255,
                OVS_ERR_INVALID_ARG, "need 1 <= min_fast_thr <= ini_fast_thr <= 255");
    OVS_REQUIRE(num_mask_rects >= 0 && (num_mask_rects == 0 || mask_rects), OVS_ERR_INVALID_ARG, "bad mask rects");
    int rc = ovs::select_device(device);
    if (rc != OVS_OK) return rc;
    ovs_extractor* h = new (std::nothrow) ovs_extractor();
    OVS_REQUIRE(h, OVS_ERR_CUDA, "out of host memory");
    h->P = *params;
    h->device = device;
    if (num_mask_rects) h->mask_rects.assign(mask_rects, mask_rects + 4 * num_mask_rects);
    const int L = (int)params->num_levels;
    // orb_params::calc_scale_factors / calc_level_sigma_sq
    h->sf[0] = 1.0f; h->sigma_sq[0] = 1.0f;
    for (int l = 1; l < L; ++l) { h->sf[l] = params->scale_factor * h->sf[l - 1]; h->sigma_sq[l] = h->sf[l] * h->sf[l]; }
    for (int l = 0; l < L; ++l) { h->inv_sf[l] = 1.0f / h->sf[l]; h->inv_sigma_sq[l] = 1.0f / h->sigma_sq[l]; }
    // orb_extractor::initialize(): keypoints per level
    {
        double desired = params->max_num_keypts * (1.0 - 1.0 / params->scale_factor)
                         / (1.0 - std::pow(1.0 / params->scale_factor, (double)L));
        unsigned total = 0;
        for (int l = 0; l < L - 1; ++l) {
            h->per_level[l] = (unsigned)std::round(desired);
            total += h->per_level[l];
            desired *= 1.0 / params->scale_factor;
        }
        h->per_level[L - 1] = (unsigned)std::max((int)params->max_num_keypts - (int)total, 0);
        if (L == 1) h->per_level[0] = params->max_num_keypts;
    }
    // u_max_ of the circular patch (half size 15)
    {
        const int hp = 15;
        int um[16] = {0};
        const int vmax = (int)std::floor(hp * std::sqrt(2.0) / 2 + 1);
        const int vmin = (int)std::ceil(hp * std::sqrt(2.0) / 2);
        for (int v = 0; v <= vmax; ++v) um[v] = (int)std::round(std::sqrt((double)hp * hp - (double)v * v));
        for (int v = hp, v0 = 0; v >= vmin; --v) {
            while (um[v0] == um[v0 + 1]) ++v0;
            um[v] = v0;
            ++v0;
        }
        for (int v = 0; v < 16; ++v) h->umax.v[v] = (signed char)um[v];
    }
    h->max_out = (int)params->max_num_keypts + L * (3 + 64);

    auto fail = [&](int code) { ovs_extractor_destroy(h); return code; };
#define OVS_TRY(expr)                                                                                  \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess) {                                                                       \
            ovs::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));      \
            return fail(OVS_ERR_CUDA);                                                                 \
        }                                                                                              \
    } while (0)
    OVS_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& e : h->ev) OVS_TRY(cudaEventCreateWithFlags(&e, ovs::event_flags()));
    OVS_TRY(cudaMalloc(&h->d_status, kStatInts * sizeof(int)));
    OVS_TRY(cudaMemset(h->d_status, 0, kStatInts * sizeof(int)));
    OVS_TRY(cudaHostAlloc(&h->h_status, kStatInts * sizeof(int), cudaHostAllocDefault));
    memset(h->h_status, 0, kStatInts * sizeof(int));
    h->d_tma_timeout = h->d_status + kStatTma;
    OVS_TRY(cudaMalloc(&h->d_kps, (size_t)h->max_out * sizeof(ovs_keypoint)));
    OVS_TRY(cudaMalloc(&h->d_desc, (size_t)h->max_out * 32));
    OVS_TRY(cudaHostAlloc(&h->h_kps, (size_t)h->max_out * sizeof(ovs_keypoint), cudaHostAllocDefault));
    OVS_TRY(cudaHostAlloc(&h->h_desc, (size_t)h->max_out * 32, cudaHostAllocDefault));
#undef OVS_TRY
    *out = h;
    return OVS_OK;
}

extern "C" void ovs_extractor_destroy(ovs_extractor* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) ovs::sync_stream(h->stream);
    free_geometry(h);
    cudaFree(h->d_status); cudaFreeHost(h->h_status);
    ovs::free_upload(h->color); cudaFree(h->d_und);
    cudaFree(h->d_kps); cudaFree(h->d_desc);
    cudaFreeHost(h->h_kps); cudaFreeHost(h->h_desc);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" int ovs_extractor_max_keypoints(const ovs_extractor* h) { return h ? h->max_out : 0; }

extern "C" int ovs_extract_host(ovs_extractor* h, const uint8_t* image, int width, int height, size_t pitch,
                                const uint8_t* mask, size_t mask_pitch,
                                ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out) {
    OVS_REQUIRE(h && image && num_out && (capacity == 0 || (keypts_out && descriptors_out)), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(width > 0 && height > 0 && pitch >= (size_t)width, OVS_ERR_INVALID_ARG, "bad image geometry");
    OVS_REQUIRE(!mask || mask_pitch >= (size_t)width, OVS_ERR_INVALID_ARG, "bad mask pitch");
    const auto t_begin = std::chrono::steady_clock::now();
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = configure(h, width, height);
    if (rc != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    // pageable input goes through the handle's pinned staging buffer; pinned input is copied directly
    cudaPointerAttributes attr;
    const bool pinned = cudaPointerGetAttributes(&attr, image) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (pinned) {
        OVS_CUDA_CHECK(cudaMemcpy2DAsync(h->d_pyr, h->T.pitch[0], image, pitch, width, height, cudaMemcpyHostToDevice, st));
    } else {
        for (int y = 0; y < height; ++y) memcpy(h->h_img + (size_t)y * width, image + (size_t)y * pitch, width);
        OVS_CUDA_CHECK(cudaMemcpy2DAsync(h->d_pyr, h->T.pitch[0], h->h_img, width, width, height, cudaMemcpyHostToDevice, st));
    }
    return extract_to_host(h, mask, mask_pitch, keypts_out, descriptors_out, capacity, num_out, t_begin);
}

// camera->undistort_keypoints + camera->convert_keypoints_to_bearings on DEVICE arrays (the extractor's device output);
// d_undist_out may alias d_keypts_in, either output may be NULL.
extern "C" int ovs_undistort_keypoints_device(ovs_extractor* h, const ovs_camera* cam, const double* dist_k1k2p1p2k3, int num_iterations, int n,
                                              const ovs_keypoint* d_keypts_in, ovs_keypoint* d_undist_out, double* d_bearings_out) {
    OVS_REQUIRE(h && cam && n >= 0 && (n == 0 || d_keypts_in), OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(cam->model == OVS_CAMERA_PERSPECTIVE || cam->model == OVS_CAMERA_EQUIRECTANGULAR || cam->model == OVS_CAMERA_FISHEYE
                || cam->model == OVS_CAMERA_RADIAL_DIVISION, OVS_ERR_INVALID_ARG, "unknown camera model");
    OVS_REQUIRE(num_iterations >= 0 && num_iterations <= 1000, OVS_ERR_INVALID_ARG, "bad iteration count");
    if (n == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    UndistortArgs A{};
    A.model = cam->model; A.iters = num_iterations;
    A.fx = cam->fx; A.fy = cam->fy; A.cx = cam->cx; A.cy = cam->cy; A.cols = cam->cols; A.rows = cam->rows;
    const double* d = dist_k1k2p1p2k3;
    if (cam->model == OVS_CAMERA_FISHEYE) {
        if (d) { A.k1 = d[0]; A.k2 = d[1]; A.p1 = d[2]; A.p2 = d[3]; }      // k1..k4 of the fisheye model
    } else if (cam->model == OVS_CAMERA_RADIAL_DIVISION) {
        if (d) A.k1 = d[0];                                                 // the single distortion parameter
    } else if (d) { A.k1 = d[0]; A.k2 = d[1]; A.p1 = d[2]; A.p2 = d[3]; A.k3 = d[4]; }
    else A.iters = 0;
    if (cam->model == OVS_CAMERA_EQUIRECTANGULAR) OVS_REQUIRE(cam->cols > 0.0 && cam->rows > 0.0, OVS_ERR_INVALID_ARG, "equirectangular camera needs cols / rows");
    else OVS_REQUIRE(cam->fx != 0.0 && cam->fy != 0.0, OVS_ERR_INVALID_ARG, "zero focal length");
    k_undistort_bearings<<<(n + 127) / 128, 128, 0, h->stream>>>(A, n, d_keypts_in, d_undist_out, d_bearings_out);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(ovs::sync_stream(h->stream));
    return OVS_OK;
}

// the same on HOST arrays (keypts_ -> undist_keypts_, bearings_)
extern "C" int ovs_undistort_keypoints_host(ovs_extractor* h, const ovs_camera* cam, const double* dist_k1k2p1p2k3, int num_iterations, int n,
                                            const ovs_keypoint* keypts_in, ovs_keypoint* undist_out, double* bearings_out) {
    OVS_REQUIRE(h && cam && n >= 0 && (n == 0 || keypts_in), OVS_ERR_INVALID_ARG, "bad argument");
    if (n == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // grow-only scratch owned by the handle (no cudaMalloc / cudaFree per frame)
    const size_t need = (size_t)n * (sizeof(ovs_keypoint) + 24) + 256;
    if (need > h->und_bytes) {
        cudaFree(h->d_und); h->d_und = nullptr; h->und_bytes = 0;
        OVS_CUDA_CHECK(cudaMalloc(&h->d_und, need + need / 2));
        h->und_bytes = need + need / 2;
    }
    double* db = reinterpret_cast<double*>(h->d_und);
    ovs_keypoint* dk = reinterpret_cast<ovs_keypoint*>(h->d_und + ((size_t)n * 24 + 255) / 256 * 256);
    cudaError_t e = cudaMemcpyAsync(dk, keypts_in, (size_t)n * sizeof(ovs_keypoint), cudaMemcpyHostToDevice, h->stream);
    int rc = OVS_OK;
    if (e == cudaSuccess) rc = ovs_undistort_keypoints_device(h, cam, dist_k1k2p1p2k3, num_iterations, n, dk, dk, db);
    if (e == cudaSuccess && rc == OVS_OK && undist_out) e = cudaMemcpyAsync(undist_out, dk, (size_t)n * sizeof(ovs_keypoint), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess && rc == OVS_OK && bearings_out) e = cudaMemcpyAsync(bearings_out, db, (size_t)n * 24, cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess && rc == OVS_OK) e = ovs::sync_stream(h->stream);
    if (rc != OVS_OK) return rc;
    if (e != cudaSuccess) { ovs::set_error("undistort_keypoints: %s", cudaGetErrorString(e)); return OVS_ERR_CUDA; }
    return OVS_OK;
}

// tracking_module::track_*: util::convert_to_grayscale(img, camera->color_order_) followed by extract().  The colour
// image is uploaded as it is and reduced to gray on the device, straight into level 0 of the pyramid.
extern "C" int ovs_extract_host_color(ovs_extractor* h, const uint8_t* image, int width, int height, size_t pitch, int channels, int color_order,
                                      const uint8_t* mask, size_t mask_pitch,
                                      ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out) {
    OVS_REQUIRE(h && image && num_out && (capacity == 0 || (keypts_out && descriptors_out)), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(channels == 3 || channels == 4, OVS_ERR_INVALID_ARG, "colour images have 3 or 4 channels (got %d)", channels);
    OVS_REQUIRE(color_order == OVS_COLOR_ORDER_BGR || color_order == OVS_COLOR_ORDER_RGB, OVS_ERR_INVALID_ARG, "bad colour order");
    OVS_REQUIRE(width > 0 && height > 0 && pitch >= (size_t)width * channels, OVS_ERR_INVALID_ARG, "bad image geometry");
    OVS_REQUIRE(!mask || mask_pitch >= (size_t)width, OVS_ERR_INVALID_ARG, "bad mask pitch");
    const auto t_begin = std::chrono::steady_clock::now();
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = configure(h, width, height);
    if (rc != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    const size_t row = (size_t)width * channels;
    rc = ovs::reserve_upload(h->color, row * height);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    rc = ovs::upload_image(h->color, image, pitch, row, height, st);
    if (rc != OVS_OK) return rc;
    k_color_to_gray<<<dim3((width + 1023) / 1024, height), 256, 0, st>>>(h->color.d, row, width, height, channels, color_order == OVS_COLOR_ORDER_RGB,
                                                                       h->d_pyr, h->T.pitch[0]);
    OVS_LAUNCH_CHECK();
    return extract_to_host(h, mask, mask_pitch, keypts_out, descriptors_out, capacity, num_out, t_begin);
}

// util::stereo_rectifier::rectify of one side, util::convert_to_grayscale and extract(): the raw image is uploaded as it is
// and remapped (and reduced to gray) on the device, straight into level 0 of the pyramid.  The rectifier is only read.
extern "C" int ovs_extract_host_rectified(ovs_extractor* h, const ovs_stereo_rectifier* rectifier, int side, const uint8_t* image, int width,
                                          int height, size_t pitch, int channels, int color_order, const uint8_t* mask, size_t mask_pitch,
                                          ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out) {
    OVS_REQUIRE(h && rectifier && image && num_out && (capacity == 0 || (keypts_out && descriptors_out)), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(side == 0 || side == 1, OVS_ERR_INVALID_ARG, "side must be 0 (left) or 1 (right), got %d", side);
    OVS_REQUIRE(channels == 1 || channels == 3 || channels == 4, OVS_ERR_INVALID_ARG, "images have 1, 3 or 4 channels (got %d)", channels);
    OVS_REQUIRE(color_order == OVS_COLOR_ORDER_BGR || color_order == OVS_COLOR_ORDER_RGB, OVS_ERR_INVALID_ARG, "bad colour order");
    OVS_REQUIRE(rectifier->device == h->device, OVS_ERR_INVALID_ARG, "rectifier on device %d, extractor on device %d", rectifier->device,
                h->device);
    OVS_REQUIRE(width == rectifier->cols && height == rectifier->rows, OVS_ERR_INVALID_ARG, "image %dx%d differs from the rectifier's %dx%d",
                width, height, rectifier->cols, rectifier->rows);
    OVS_REQUIRE(pitch >= (size_t)width * channels, OVS_ERR_INVALID_ARG, "bad image geometry");
    OVS_REQUIRE(!mask || mask_pitch >= (size_t)width, OVS_ERR_INVALID_ARG, "bad mask pitch");
    const auto t_begin = std::chrono::steady_clock::now();
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = configure(h, width, height);
    if (rc != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    const size_t row = (size_t)width * channels;
    rc = ovs::reserve_upload(h->color, row * height);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    rc = ovs::upload_image(h->color, image, pitch, row, height, st);
    if (rc == OVS_OK)
        rc = ovs::launch_stereo_remap(rectifier, side, h->color.d, row, channels, 1, color_order == OVS_COLOR_ORDER_RGB, h->d_pyr,
                                      h->T.pitch[0], st);
    if (rc != OVS_OK) return rc;
    return extract_to_host(h, mask, mask_pitch, keypts_out, descriptors_out, capacity, num_out, t_begin);
}

extern "C" int ovs_extract_device(ovs_extractor* h, const uint8_t* d_image, int width, int height, size_t pitch,
                                  const uint8_t* mask, size_t mask_pitch,
                                  ovs_keypoint* d_keypts_out, uint8_t* d_descriptors_out, int capacity, int* num_out) {
    OVS_REQUIRE(h && d_image && num_out && d_keypts_out && d_descriptors_out, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(width > 0 && height > 0 && pitch >= (size_t)width, OVS_ERR_INVALID_ARG, "bad image geometry");
    const auto t_begin = std::chrono::steady_clock::now();
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = configure(h, width, height);
    if (rc != OVS_OK) return rc;
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    OVS_CUDA_CHECK(cudaMemcpy2DAsync(h->d_pyr, h->T.pitch[0], d_image, pitch, width, height, cudaMemcpyDeviceToDevice, st));
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    rc = run_pipeline(h, mask, mask_pitch, d_keypts_out, d_descriptors_out, capacity);
    if (rc != OVS_OK) return rc;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[7], st));
    OVS_CUDA_CHECK(ovs::sync_event(h->ev[7]));
    rc = finish_pipeline(h, capacity, num_out);
    if (rc != OVS_OK) return rc;
    return collect_timings(h, t_begin);
}

extern "C" int ovs_extractor_pyramid_level(const ovs_extractor* h, int level, const uint8_t** d_ptr, size_t* pitch,
                                           int* width, int* height) {
    OVS_REQUIRE(h && h->img_w > 0, OVS_ERR_INVALID_ARG, "no image extracted yet");
    OVS_REQUIRE(level >= 0 && level < h->T.num_levels, OVS_ERR_INVALID_ARG, "level out of range");
    if (d_ptr) *d_ptr = h->d_pyr + h->T.off[level];
    if (pitch) *pitch = (size_t)h->T.pitch[level];
    if (width) *width = h->T.w[level];
    if (height) *height = h->T.h[level];
    return OVS_OK;
}

extern "C" int ovs_extractor_copy_pyramid_level(ovs_extractor* h, int level, uint8_t* out, size_t out_pitch) {
    OVS_REQUIRE(h && out && h->img_w > 0, OVS_ERR_INVALID_ARG, "no image extracted yet");
    OVS_REQUIRE(level >= 0 && level < h->T.num_levels && out_pitch >= (size_t)h->T.w[level], OVS_ERR_INVALID_ARG, "bad level / pitch");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    OVS_CUDA_CHECK(cudaMemcpy2D(out, out_pitch, h->d_pyr + h->T.off[level], h->T.pitch[level], h->T.w[level], h->T.h[level],
                                cudaMemcpyDeviceToHost));
    return OVS_OK;
}

extern "C" int ovs_extractor_scale_factors(const ovs_extractor* h, float* scale_factors, float* inv_scale_factors,
                                           float* level_sigma_sq, float* inv_level_sigma_sq) {
    OVS_REQUIRE(h, OVS_ERR_INVALID_ARG, "null handle");
    const int L = (int)h->P.num_levels;
    for (int l = 0; l < L; ++l) {
        if (scale_factors) scale_factors[l] = h->sf[l];
        if (inv_scale_factors) inv_scale_factors[l] = h->inv_sf[l];
        if (level_sigma_sq) level_sigma_sq[l] = h->sigma_sq[l];
        if (inv_level_sigma_sq) inv_level_sigma_sq[l] = h->inv_sigma_sq[l];
    }
    return OVS_OK;
}

extern "C" int ovs_extractor_debug_score_map(ovs_extractor* h, int level, uint8_t* out, size_t out_pitch) {
    OVS_REQUIRE(h && out && h->img_w > 0, OVS_ERR_INVALID_ARG, "no image extracted yet");
    OVS_REQUIRE(level >= 0 && level < h->T.num_levels && out_pitch >= (size_t)h->T.w[level], OVS_ERR_INVALID_ARG, "bad level / pitch");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    OVS_CUDA_CHECK(cudaMemcpy2D(out, out_pitch, h->d_score + h->T.off[level], h->T.pitch[level], h->T.w[level], h->T.h[level],
                                cudaMemcpyDeviceToHost));
    return OVS_OK;
}

extern "C" int ovs_extractor_debug_candidates(ovs_extractor* h, int level, int32_t* xys_out, int cap, int* n_out) {
    OVS_REQUIRE(h && n_out && h->img_w > 0, OVS_ERR_INVALID_ARG, "no image extracted yet");
    const int L = h->T.num_levels;
    OVS_REQUIRE(level >= 0 && level < L, OVS_ERR_INVALID_ARG, "level out of range");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // the level's candidates (after the mask filter) as k_tree_distribute left them in its scratch
    const int* S = h->h_status;
    const int o = h->targs.lv[level].cand_off;
    const int n = S[L + level];
    *n_out = n;
    const int m = std::min(n, cap);
    if (m > 0) {
        std::vector<uint32_t> c(m);
        OVS_CUDA_CHECK(cudaMemcpy(c.data(), h->tbuf.fc + o, (size_t)m * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        for (int i = 0; i < m; ++i) {
            xys_out[3 * i] = (int)(c[i] & 0xfffu); xys_out[3 * i + 1] = (int)((c[i] >> 12) & 0xfffu); xys_out[3 * i + 2] = (int)(c[i] >> 24);
        }
    }
    return OVS_OK;
}

extern "C" int ovs_extractor_last_timings(const ovs_extractor* h, float* out_us) {
    OVS_REQUIRE(h && out_us, OVS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < 8; ++i) out_us[i] = h->timings[i];
    return OVS_OK;
}
