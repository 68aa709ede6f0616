// stereo_rectify.h -- what the extractor uses of util::stereo_rectifier (stereo_rectify.cu), and the staged host-image upload
// that ovs_extract_host_color, ovs_extract_host_rectified and ovs_stereo_rectify_host share.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <mutex>

#include "ovs_common.h"

namespace ovs {

// A u8 host image on its way to the device: a grow-only pinned staging buffer for pageable input and a grow-only device
// buffer that holds the image densely (rows of `row` bytes).
struct HostUpload {
    uint8_t* h = nullptr;
    uint8_t* d = nullptr;
    size_t bytes = 0;
};
int reserve_upload(HostUpload& u, size_t bytes);
// Queues the copy of `height` rows of `row` bytes, `pitch` apart, into u.d: pinned input is copied directly, pageable input
// through u.h.  reserve_upload(u, row * height) must have succeeded.
int upload_image(HostUpload& u, const uint8_t* image, size_t pitch, size_t row, int height, cudaStream_t st);
void free_upload(HostUpload& u);

}  // namespace ovs

struct ovs_stereo_rectifier {
    int device = 0, model = 0, cols = 0, rows = 0;
    float* d_maps = nullptr;   // [side][x / y][rows * cols]: the float maps, kept for export
    int2* d_fixed = nullptr;   // [side][rows * cols]: remap's fixed-point form of each entry, cvRound(m * 32) (INT_MIN: outside)
    // ovs_stereo_rectify_host's stream and scratch; the maps above never change after create
    std::mutex host_mutex;
    cudaStream_t stream = nullptr;
    ovs::HostUpload in[2];
    uint8_t* d_out = nullptr;
    uint8_t* h_out = nullptr;
    size_t out_bytes = 0;
};

namespace ovs {

// Queues the remap of one side: d_src is the raw cols x rows image with `channels` interleaved u8 channels, `spitch` bytes per
// row.  gray = 0 writes the remapped image with the same channels; gray = 1 writes cvtColor(remapped, *2GRAY) (r_first: RGB
// order), or the remapped image itself for 1 channel.  One launch.
int launch_stereo_remap(const ovs_stereo_rectifier* r, int side, const uint8_t* d_src, size_t spitch, int channels, int gray, int r_first,
                        uint8_t* d_dst, size_t dpitch, cudaStream_t st);

}  // namespace ovs
