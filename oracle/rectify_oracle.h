/* rectify_oracle.h -- see rectify_oracle.c.  TEST INFRASTRUCTURE ONLY. */
#ifndef RECTIFY_ORACLE_H
#define RECTIFY_ORACLE_H
#include <stdint.h>

/* iR = (K_rect * R)^-1 as initUndistortRectifyMap forms it (3 x 3 product, cv::invert DECOMP_LU); row-major. Returns 0 if singular. */
int orc_rectify_inverse(const double K_rect[9], const double R[9], double iR[9]);
/* cv::initUndistortRectifyMap (model 0, dist = k1 k2 p1 p2 k3) / cv::fisheye::initUndistortRectifyMap (model 2, dist = k1..k4),
 * CV_32FC1 maps of cols x rows.  Returns 0 if K_rect * R is singular. */
int orc_init_rectify_map(int model, int cols, int rows, const double K[9], const double* dist, const double R[9], const double K_rect[9],
                         float* map_x, float* map_y);
/* cv::remap(src, dst, map_x, map_y, INTER_LINEAR, BORDER_CONSTANT, 0) on u8 with 1..4 channels; dst is map_w x map_h. */
void orc_remap_linear(const uint8_t* src, int w, int h, int src_pitch, int channels, const float* map_x, const float* map_y,
                      int map_w, int map_h, uint8_t* dst, int dst_pitch);
/* The fixed-point form remap uses per map entry: X = cvRound(m * 32) with x86's INT_MIN for NaN and out-of-range products. */
int orc_remap_quantise(float m);
#endif
