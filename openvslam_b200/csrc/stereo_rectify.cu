// stereo_rectify.cu -- util::stereo_rectifier on the device (DESIGN section 1 row f15).
//
// create: cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap (CV_32FC1 maps) for both cameras, one thread per
// map entry, evaluated in float64 exactly as OpenCV 4 writes it (see oracle/rectify_oracle.c): no contraction into FMAs, the
// perspective row walked in OpenCV's blocks of 8 columns, the fisheye row one column at a time.  The same kernel stores
// remap's fixed-point form of each entry, so the per-frame remap reads one int2 per output pixel.
// rectify: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) on u8, with the 15-bit weights OpenCV's bilinear table holds, and a
// variant that converts to gray (util::convert_to_grayscale) in the same pass, straight into the extractor's pyramid.
#include "ovs_common.h"
#include "stereo_rectify.h"

#include <limits.h>
#include <math.h>
#include <string.h>

#include <new>

namespace {

struct RectifySide {
    double fx, fy, cx, cy;
    double d[5];    // k1 k2 p1 p2 k3 (perspective) | k1 k2 k3 k4 (fisheye)
    double ir[9];   // (K_rect R)^-1, row-major
};

struct RectifyMapArgs {
    int model, cols, rows;
    RectifySide side[2];
};

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }

// remap's map conversion: cvRound(m * 32), and x86's INT_MIN where the product is NaN or outside int (CUDA's conversion
// would give 0 for NaN and saturate the rest)
__device__ __forceinline__ int remap_fixed(float m) {
    const float t = __fmul_rn(m, 32.f);
    return (t >= -2147483648.f && t < 2147483648.f) ? __float2int_rn(t) : INT_MIN;
}

// grid (ceil(cols / 128), rows, 2 sides), one thread per map entry
__global__ void __launch_bounds__(128) k_rectify_map(const RectifyMapArgs A, float* __restrict__ maps, int2* __restrict__ fixed) {
    const int j = blockIdx.x * 128 + threadIdx.x, i = blockIdx.y, s = blockIdx.z;
    if (j >= A.cols) return;
    const RectifySide& S = A.side[s];
    const double* ir = S.ir;
    double X = da(dm((double)i, ir[1]), ir[2]), Y = da(dm((double)i, ir[4]), ir[5]), W = da(dm((double)i, ir[7]), ir[8]);
    double u, v;
    if (A.model == OVS_CAMERA_PERSPECTIVE) {
        // OpenCV's loop: blocks of 8 columns at base + jj ir_0 (the base advancing by 8 ir_0), then one ir_0 per column
        const int nb = A.cols / 8 * 8;
        const int blocks = (j < nb ? j : nb) / 8;
        const double sx = dm(8.0, ir[0]), sy = dm(8.0, ir[3]), sw = dm(8.0, ir[6]);
        for (int b = 0; b < blocks; ++b) { X = da(X, sx); Y = da(Y, sy); W = da(W, sw); }
        if (j < nb) {
            const double jj = (double)(j & 7);
            X = da(X, dm(ir[0], jj)); Y = da(Y, dm(ir[3], jj)); W = da(W, dm(ir[6], jj));
        } else {
            for (int t = nb; t < j; ++t) { X = da(X, ir[0]); Y = da(Y, ir[3]); W = da(W, ir[6]); }
        }
        const double w = __ddiv_rn(1.0, W), x = dm(X, w), y = dm(Y, w);
        const double x2 = dm(x, x), y2 = dm(y, y), r2 = da(x2, y2), xy2 = dm(dm(2.0, x), y);
        const double* d = S.d;
        const double kr = da(1.0, dm(da(dm(da(dm(d[4], r2), d[1]), r2), d[0]), r2));
        const double xd = da(da(dm(x, kr), dm(d[2], xy2)), dm(d[3], da(r2, dm(2.0, x2))));
        const double yd = da(da(dm(y, kr), dm(d[2], da(r2, dm(2.0, y2)))), dm(d[3], xy2));
        u = da(dm(S.fx, xd), S.cx);
        v = da(dm(S.fy, yd), S.cy);
    } else {
        for (int t = 0; t < j; ++t) { X = da(X, ir[0]); Y = da(Y, ir[3]); W = da(W, ir[6]); }
        if (W <= 0) {
            u = X > 0 ? -INFINITY : INFINITY;
            v = Y > 0 ? -INFINITY : INFINITY;
        } else {
            const double x = __ddiv_rn(X, W), y = __ddiv_rn(Y, W);
            const double r = __dsqrt_rn(da(dm(x, x), dm(y, y)));
            const double th = atan(r);
            const double t2 = dm(th, th), t4 = dm(t2, t2), t6 = dm(t4, t2), t8 = dm(t4, t4);
            const double* k = S.d;
            const double td = dm(th, da(da(da(da(1.0, dm(k[0], t2)), dm(k[1], t4)), dm(k[2], t6)), dm(k[3], t8)));
            const double scale = r == 0 ? 1.0 : __ddiv_rn(td, r);
            u = da(dm(dm(S.fx, x), scale), S.cx);
            v = da(dm(dm(S.fy, y), scale), S.cy);
        }
    }
    const size_t n = (size_t)A.cols * A.rows, e = (size_t)i * A.cols + j;
    const float uf = __double2float_rn(u), vf = __double2float_rn(v);
    maps[(2 * s) * n + e] = uf;
    maps[(2 * s + 1) * n + e] = vf;
    fixed[s * n + e] = make_int2(remap_fixed(uf), remap_fixed(vf));
}

// One thread -> 4 output pixels of one row.  Each pixel's fixed-point map entry is read once; its four source samples are
// gathered per channel through the read-only path, a sample outside the image counting 0.  GRAY: the remapped channels are
// reduced with cvtColor's 15-bit weights (B 3735, G 19235, R 9798) and 4 gray pixels are stored as one word.
template <int C, bool GRAY>
__global__ void __launch_bounds__(256) k_stereo_remap(const int2* __restrict__ fixed, const uint8_t* __restrict__ src, size_t spitch, int w,
                                                      int h, int r_first, uint8_t* __restrict__ dst, size_t dpitch) {
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x0 >= w) return;
    const int cnt = min(4, w - x0);
    const int2* q = fixed + (size_t)y * w + x0;
    uint8_t* d = dst + (size_t)y * dpitch;
    unsigned packed = 0;
    for (int p = 0; p < cnt; ++p) {
        const int2 X = __ldg(q + p);
        const int sx = X.x >> 5, sy = X.y >> 5, ax = X.x & 31, ay = X.y & 31;
        const int wt[4] = {(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32};
        int acc[C];
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int xs = sx + (k & 1), ys = sy + (k >> 1);
            if ((unsigned)xs < (unsigned)w && (unsigned)ys < (unsigned)h) {
                const uint8_t* s = src + (size_t)ys * spitch + (size_t)xs * C;
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] += wt[k] * (int)__ldg(s + c);
            }
        }
        int o[C];
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = (acc[c] + (1 << 14)) >> 15;
        if (GRAY) {
            int g = o[0];
            if (C >= 3) {
                const int b = r_first ? o[2] : o[0], r = r_first ? o[0] : o[2];
                g = (b * 3735 + o[1] * 19235 + r * 9798 + 16384) >> 15;
            }
            packed |= (unsigned)g << (8 * p);
        } else {
#pragma unroll
            for (int c = 0; c < C; ++c) d[(size_t)(x0 + p) * C + c] = (uint8_t)o[c];
        }
    }
    if (GRAY) {
        if (cnt == 4 && ((reinterpret_cast<uintptr_t>(d + x0) & 3) == 0)) *reinterpret_cast<unsigned*>(d + x0) = packed;
        else for (int p = 0; p < cnt; ++p) d[x0 + p] = (uint8_t)(packed >> (8 * p));
    }
}

// cv::invert's closed form for 3 x 3 (DECOMP_LU) of the product K_rect R; false if singular
bool rectify_inverse(const double* P, const double* R, double* iR) {
    double m[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[3 * i + j] = P[3 * i] * R[j] + P[3 * i + 1] * R[3 + j] + P[3 * i + 2] * R[6 + j];
    double d = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
    if (d == 0. || !std::isfinite(d)) return false;
    d = 1. / d;
    iR[0] = (m[4] * m[8] - m[5] * m[7]) * d;
    iR[1] = (m[2] * m[7] - m[1] * m[8]) * d;
    iR[2] = (m[1] * m[5] - m[2] * m[4]) * d;
    iR[3] = (m[5] * m[6] - m[3] * m[8]) * d;
    iR[4] = (m[0] * m[8] - m[2] * m[6]) * d;
    iR[5] = (m[2] * m[3] - m[0] * m[5]) * d;
    iR[6] = (m[3] * m[7] - m[4] * m[6]) * d;
    iR[7] = (m[1] * m[6] - m[0] * m[7]) * d;
    iR[8] = (m[0] * m[4] - m[1] * m[3]) * d;
    return true;
}

}  // namespace

namespace ovs {

int reserve_upload(HostUpload& u, size_t bytes) {
    if (bytes <= u.bytes) return OVS_OK;
    free_upload(u);
    OVS_CUDA_CHECK(cudaHostAlloc(&u.h, bytes, cudaHostAllocDefault));
    OVS_CUDA_CHECK(cudaMalloc(&u.d, bytes));
    u.bytes = bytes;
    return OVS_OK;
}

int upload_image(HostUpload& u, const uint8_t* image, size_t pitch, size_t row, int height, cudaStream_t st) {
    cudaPointerAttributes attr;
    const bool pinned = cudaPointerGetAttributes(&attr, image) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (pinned) {
        OVS_CUDA_CHECK(cudaMemcpy2DAsync(u.d, row, image, pitch, row, height, cudaMemcpyHostToDevice, st));
    } else {
        for (int y = 0; y < height; ++y) memcpy(u.h + (size_t)y * row, image + (size_t)y * pitch, row);
        OVS_CUDA_CHECK(cudaMemcpyAsync(u.d, u.h, row * height, cudaMemcpyHostToDevice, st));
    }
    return OVS_OK;
}

void free_upload(HostUpload& u) {
    cudaFreeHost(u.h); cudaFree(u.d);
    u.h = nullptr; u.d = nullptr; u.bytes = 0;
}

int launch_stereo_remap(const ovs_stereo_rectifier* r, int side, const uint8_t* d_src, size_t spitch, int channels, int gray, int r_first,
                        uint8_t* d_dst, size_t dpitch, cudaStream_t st) {
    const int w = r->cols, h = r->rows;
    const int2* q = r->d_fixed + (size_t)side * w * h;
    const dim3 grid((w + 1023) / 1024, h);
#define OVS_REMAP(C, G) k_stereo_remap<C, G><<<grid, 256, 0, st>>>(q, d_src, spitch, w, h, r_first, d_dst, dpitch)
    if (gray) {
        if (channels == 1) OVS_REMAP(1, true); else if (channels == 3) OVS_REMAP(3, true); else OVS_REMAP(4, true);
    } else {
        if (channels == 1) OVS_REMAP(1, false); else if (channels == 3) OVS_REMAP(3, false); else OVS_REMAP(4, false);
    }
#undef OVS_REMAP
    OVS_LAUNCH_CHECK();
    return OVS_OK;
}

}  // namespace ovs

// ================================================================================ C ABI
extern "C" int ovs_stereo_rectifier_create(int device, int model, int cols, int rows, const double* K_l, const double* D_l, const double* R_l,
                                           const double* K_r, const double* D_r, const double* R_r, const double* K_rect,
                                           ovs_stereo_rectifier** out) {
    OVS_REQUIRE(out && K_l && D_l && R_l && K_r && D_r && R_r && K_rect, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(model == OVS_CAMERA_PERSPECTIVE || model == OVS_CAMERA_FISHEYE, OVS_ERR_INVALID_ARG,
                "stereo rectification supports the perspective and fisheye models (got %d)", model);
    OVS_REQUIRE(cols >= 1 && rows >= 1 && cols <= 32767 && rows <= 32767, OVS_ERR_INVALID_ARG, "bad image size %dx%d", cols, rows);
    RectifyMapArgs A{};
    A.model = model; A.cols = cols; A.rows = rows;
    const double* K[2] = {K_l, K_r};
    const double* D[2] = {D_l, D_r};
    const double* R[2] = {R_l, R_r};
    for (int s = 0; s < 2; ++s) {
        RectifySide& S = A.side[s];
        S.fx = K[s][0]; S.fy = K[s][4]; S.cx = K[s][2]; S.cy = K[s][5];
        for (int k = 0; k < (model == OVS_CAMERA_FISHEYE ? 4 : 5); ++k) S.d[k] = D[s][k];
        OVS_REQUIRE(rectify_inverse(K_rect, R[s], S.ir), OVS_ERR_INVALID_ARG, "K_rect R of side %d is singular", s);
    }
    int rc = ovs::select_device(device);
    if (rc != OVS_OK) return rc;
    ovs_stereo_rectifier* h = new (std::nothrow) ovs_stereo_rectifier();
    OVS_REQUIRE(h, OVS_ERR_CUDA, "out of host memory");
    h->device = device; h->model = model; h->cols = cols; h->rows = rows;
    const size_t n = (size_t)cols * rows;
    cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&h->d_maps, 4 * n * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&h->d_fixed, 2 * n * sizeof(int2));
    if (e == cudaSuccess) {
        k_rectify_map<<<dim3((cols + 127) / 128, rows, 2), 128, 0, h->stream>>>(A, h->d_maps, h->d_fixed);
        ovs::count_launch();
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = ovs::sync_stream(h->stream);
    if (e != cudaSuccess) {
        ovs::set_error("stereo_rectifier_create: %s", cudaGetErrorString(e));
        ovs_stereo_rectifier_destroy(h);
        return OVS_ERR_CUDA;
    }
    *out = h;
    return OVS_OK;
}

extern "C" void ovs_stereo_rectifier_destroy(ovs_stereo_rectifier* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) ovs::sync_stream(h->stream);
    cudaFree(h->d_maps); cudaFree(h->d_fixed);
    for (auto& u : h->in) ovs::free_upload(u);
    cudaFree(h->d_out); cudaFreeHost(h->h_out);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" int ovs_stereo_rectifier_maps(const ovs_stereo_rectifier* h, int side, float* map_x, float* map_y) {
    OVS_REQUIRE(h && map_x && map_y, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(side == 0 || side == 1, OVS_ERR_INVALID_ARG, "side must be 0 (left) or 1 (right), got %d", side);
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    const size_t n = (size_t)h->cols * h->rows;
    OVS_CUDA_CHECK(cudaMemcpy(map_x, h->d_maps + (2 * side) * n, n * sizeof(float), cudaMemcpyDeviceToHost));
    OVS_CUDA_CHECK(cudaMemcpy(map_y, h->d_maps + (2 * side + 1) * n, n * sizeof(float), cudaMemcpyDeviceToHost));
    return OVS_OK;
}

extern "C" int ovs_stereo_rectify_host(ovs_stereo_rectifier* h, const uint8_t* left, const uint8_t* right, int width, int height, size_t pitch,
                                       int channels, uint8_t* out_left, uint8_t* out_right, size_t out_pitch) {
    OVS_REQUIRE(h && left && right && out_left && out_right, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(channels == 1 || channels == 3 || channels == 4, OVS_ERR_INVALID_ARG, "images have 1, 3 or 4 channels (got %d)", channels);
    OVS_REQUIRE(width == h->cols && height == h->rows, OVS_ERR_INVALID_ARG, "image %dx%d differs from the rectifier's %dx%d", width, height,
                h->cols, h->rows);
    const size_t row = (size_t)width * channels, bytes = row * height;
    OVS_REQUIRE(pitch >= row && out_pitch >= row, OVS_ERR_INVALID_ARG, "bad image pitch");
    std::lock_guard<std::mutex> lock(h->host_mutex);
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    int rc = ovs::reserve_upload(h->in[0], bytes);
    if (rc == OVS_OK) rc = ovs::reserve_upload(h->in[1], bytes);
    if (rc != OVS_OK) return rc;
    if (2 * bytes > h->out_bytes) {
        cudaFree(h->d_out); cudaFreeHost(h->h_out); h->d_out = nullptr; h->h_out = nullptr; h->out_bytes = 0;
        OVS_CUDA_CHECK(cudaMalloc(&h->d_out, 2 * bytes));
        OVS_CUDA_CHECK(cudaHostAlloc(&h->h_out, 2 * bytes, cudaHostAllocDefault));
        h->out_bytes = 2 * bytes;
    }
    cudaStream_t st = h->stream;
    const uint8_t* img[2] = {left, right};
    for (int s = 0; s < 2; ++s) {
        rc = ovs::upload_image(h->in[s], img[s], pitch, row, height, st);
        if (rc == OVS_OK) rc = ovs::launch_stereo_remap(h, s, h->in[s].d, row, channels, 0, 0, h->d_out + s * bytes, row, st);
        if (rc != OVS_OK) return rc;
    }
    OVS_CUDA_CHECK(cudaMemcpyAsync(h->h_out, h->d_out, 2 * bytes, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    uint8_t* out[2] = {out_left, out_right};
    for (int s = 0; s < 2; ++s)
        for (int y = 0; y < height; ++y) memcpy(out[s] + (size_t)y * out_pitch, h->h_out + s * bytes + (size_t)y * row, row);
    return OVS_OK;
}
