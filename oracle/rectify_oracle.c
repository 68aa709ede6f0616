/* rectify_oracle.c -- util::stereo_rectifier restated in C: the two rectification map builders and bilinear remap.
 * TEST INFRASTRUCTURE ONLY.  Pinned against cv2 4.13.0 by tests/test_rectify_oracle.py.
 *
 * initUndistortRectifyMap (perspective): iR = (K_rect R)^-1 by cv::invert's 3 x 3 closed form (DECOMP_LU).  Per row i the
 * homogeneous ray starts at (i iR01 + iR02, i iR11 + iR12, i iR21 + iR22); OpenCV's vector loop walks the row in blocks of 8
 * columns, each block's base advanced by 8 iR_0 and column b + jj at base + jj iR_0, and the last W mod 8 columns advance one
 * iR_0 at a time.  x = _x (1 / _w), then the radtan polynomial with kr = 1 + ((k3 r2 + k2) r2 + k1) r2,
 * u = fx (x kr + p1 2xy + p2 (r2 + 2x^2)) + u0, v = fy (y kr + p1 (r2 + 2y^2) + p2 2xy) + v0, rounded to float.
 *
 * fisheye::initUndistortRectifyMap: the ray advances one iR_0 per column; _w <= 0 maps to -+inf; otherwise x = _x / _w,
 * theta = atan(r), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8), scale = theta_d / r (1 at r = 0),
 * u = fx x scale + u0.
 *
 * remap INTER_LINEAR / BORDER_CONSTANT 0 on u8: X = cvRound(m * 32) (INT_MIN, as x86's conversion gives, for NaN or a
 * product outside int), sx = saturate_cast<short>(X >> 5), ax = X & 31; the same for y.  Weights (32-ax)(32-ay) 32,
 * ax (32-ay) 32, (32-ax) ay 32, ax ay 32 sum to 2^15; a sample outside the image contributes 0; out = (sum + 2^14) >> 15.
 * All float64 arithmetic is evaluated as written (-ffp-contract=off). */
#include "rectify_oracle.h"

#include <limits.h>
#include <math.h>
#include <stddef.h>

int orc_rectify_inverse(const double P[9], const double R[9], double iR[9]) {
    double m[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[3 * i + j] = P[3 * i] * R[j] + P[3 * i + 1] * R[3 + j] + P[3 * i + 2] * R[6 + j];
    double d = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
    if (d == 0.) return 0;
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
    return 1;
}

static void perspective_pixel(const double* K, const double* D, double X, double Y, double W, float* u_out, float* v_out) {
    const double w = 1. / W, x = X * w, y = Y * w;
    const double x2 = x * x, y2 = y * y, r2 = x2 + y2, _2xy = 2 * x * y;
    const double kr = 1 + ((D[4] * r2 + D[1]) * r2 + D[0]) * r2;
    const double xd = x * kr + D[2] * _2xy + D[3] * (r2 + 2 * x2);
    const double yd = y * kr + D[2] * (r2 + 2 * y2) + D[3] * _2xy;
    *u_out = (float)(K[0] * xd + K[2]);
    *v_out = (float)(K[4] * yd + K[5]);
}

static void fisheye_pixel(const double* K, const double* D, double X, double Y, double W, float* u_out, float* v_out) {
    if (W <= 0) {
        *u_out = (float)(X > 0 ? -INFINITY : INFINITY);
        *v_out = (float)(Y > 0 ? -INFINITY : INFINITY);
        return;
    }
    const double x = X / W, y = Y / W;
    const double r = sqrt(x * x + y * y);
    const double th = atan(r);
    const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    const double td = th * (1 + D[0] * t2 + D[1] * t4 + D[2] * t6 + D[3] * t8);
    const double scale = r == 0 ? 1.0 : td / r;
    *u_out = (float)(K[0] * x * scale + K[2]);
    *v_out = (float)(K[4] * y * scale + K[5]);
}

int orc_init_rectify_map(int model, int cols, int rows, const double K[9], const double* D, const double R[9], const double K_rect[9],
                         float* map_x, float* map_y) {
    double ir[9];
    if (!orc_rectify_inverse(K_rect, R, ir)) return 0;
    for (int i = 0; i < rows; ++i) {
        float* mx = map_x + (size_t)i * cols;
        float* my = map_y + (size_t)i * cols;
        double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
        int j = 0;
        if (model == 0) {
            for (; j <= cols - 8; j += 8, _x += 8 * ir[0], _y += 8 * ir[3], _w += 8 * ir[6])
                for (int jj = 0; jj < 8; ++jj)
                    perspective_pixel(K, D, _x + ir[0] * jj, _y + ir[3] * jj, _w + ir[6] * jj, mx + j + jj, my + j + jj);
            for (; j < cols; ++j, _x += ir[0], _y += ir[3], _w += ir[6]) perspective_pixel(K, D, _x, _y, _w, mx + j, my + j);
        } else {
            for (; j < cols; ++j, _x += ir[0], _y += ir[3], _w += ir[6]) fisheye_pixel(K, D, _x, _y, _w, mx + j, my + j);
        }
    }
    return 1;
}

int orc_remap_quantise(float m) {
    const float t = m * 32.f;
    if (!(t >= -2147483648.f && t < 2147483648.f)) return INT_MIN;
    return (int)nearbyintf(t);
}

static int sat_short(int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; }

void orc_remap_linear(const uint8_t* src, int w, int h, int src_pitch, int channels, const float* map_x, const float* map_y,
                      int map_w, int map_h, uint8_t* dst, int dst_pitch) {
    for (int i = 0; i < map_h; ++i) {
        uint8_t* d = dst + (size_t)i * dst_pitch;
        for (int j = 0; j < map_w; ++j) {
            const int X = orc_remap_quantise(map_x[(size_t)i * map_w + j]), Y = orc_remap_quantise(map_y[(size_t)i * map_w + j]);
            const int sx = sat_short(X >> 5), sy = sat_short(Y >> 5), ax = X & 31, ay = Y & 31;
            const int wt[4] = {(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32};
            for (int c = 0; c < channels; ++c) {
                int acc = 0;
                for (int k = 0; k < 4; ++k) {
                    const int x = sx + (k & 1), y = sy + (k >> 1);
                    if (x >= 0 && x < w && y >= 0 && y < h) acc += wt[k] * src[(size_t)y * src_pitch + (size_t)x * channels + c];
                }
                d[(size_t)j * channels + c] = (uint8_t)((acc + (1 << 14)) >> 15);
            }
        }
    }
}
