// staging.h -- host-side buffer layout of every library call: grow-only arenas, buffers carved from them, and the staging of a
// call's inputs and outputs through a pinned host arena and a device arena.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>

#include "ovs_common.h"

namespace ovs {

// Grow-only buffers of n >= need elements of T.  A quarter of slack: the sizes creep from call to call (keypoints per frame,
// a map's local window), and every cudaFree / cudaMalloc stalls all streams of the device.
template <typename T>
int grow_dev(T** p, size_t* cap, size_t need) {
    if (need <= *cap) return OVS_OK;
    cudaFree(*p); *p = nullptr; *cap = 0;
    const size_t n = std::max(need + need / 4, (size_t)4096);
    OVS_CUDA_CHECK(cudaMalloc(p, n * sizeof(T)));
    *cap = n;
    return OVS_OK;
}
template <typename T>
int grow_host(T** p, size_t* cap, size_t need) {
    if (need <= *cap) return OVS_OK;
    cudaFreeHost(*p); *p = nullptr; *cap = 0;
    const size_t n = std::max(need + need / 4, (size_t)4096);
    OVS_CUDA_CHECK(cudaHostAlloc(p, n * sizeof(T), cudaHostAllocDefault));
    *cap = n;
    return OVS_OK;
}

// Buffers carved one after another from a byte arena, each aligned to 256 bytes.  With a null base the carve only counts:
// `off` is then the size the arena needs.
struct Arena {
    uint8_t* base; size_t off;
    template <typename T> T* take(size_t n) {
        off = (off + 255) / 256 * 256;
        T* p = reinterpret_cast<T*>(base + off);
        off += n * sizeof(T);
        return p;
    }
};

// The buffers of one call, carved from a pinned host arena and a device arena together.  Each input, in/out buffer and output
// is named once and gets the same offset in both arenas, so the inputs and in/out buffers go up in one copy and the in/out
// buffers and outputs come back in another.  Carve the inputs first, then the in/out buffers, then the outputs, then the
// device-only scratch: `ordered` turns false when a take breaks that order (an input after an output would move the end of the
// upload past outputs, and the copy back would miss them).
struct Staging {
    Arena h{nullptr, 0}, d{nullptr, 0};
    size_t in_end = 0;                               // bytes of the inputs
    size_t io_end = 0;                               // bytes of the inputs and the in/out buffers: the upload
    int phase = 0;                                   // 0 inputs, 1 in/out, 2 outputs, 3 device scratch
    bool ordered = true;
    template <typename T> T* in(T*& host, size_t n) {
        ordered = ordered && phase == 0;
        host = h.take<T>(n);
        in_end = io_end = h.off;
        return d.take<T>(n);
    }
    template <typename T> T* io(T*& host, size_t n) {
        ordered = ordered && phase <= 1;
        phase = 1;
        host = h.take<T>(n);
        io_end = h.off;
        return d.take<T>(n);
    }
    template <typename T> T* out(T*& host, size_t n) {
        ordered = ordered && phase <= 2;
        phase = 2;
        host = h.take<T>(n);
        return d.take<T>(n);
    }
    template <typename T> T* dev(size_t n) {
        phase = 3;
        return d.take<T>(n);
    }
    size_t down_begin() const { return (in_end + 255) / 256 * 256; }
    cudaError_t upload(cudaStream_t st) const { return cudaMemcpyAsync(d.base, h.base, io_end, cudaMemcpyHostToDevice, st); }
    cudaError_t download(cudaStream_t st) const {
        const size_t b = down_begin();
        return cudaMemcpyAsync(h.base + b, d.base + b, h.off - b, cudaMemcpyDeviceToHost, st);
    }
};

// Sizes the arenas by running carve(S) on null bases, grows the device arena and then the host arena (either may move), then
// carves them for real into S.  A carve out of order is refused before anything is allocated.
template <class Carve>
int stage(Staging& S, uint8_t*& h_base, size_t& h_cap, uint8_t*& d_base, size_t& d_cap, Carve carve) {
    S = Staging{};
    carve(S);
    OVS_REQUIRE(S.ordered, OVS_ERR_UNSUPPORTED, "staging carved out of order (inputs, then in/out, then outputs, then device scratch)");
    int rc = grow_dev(&d_base, &d_cap, S.d.off);
    if (rc == OVS_OK) rc = grow_host(&h_base, &h_cap, S.h.off);
    if (rc != OVS_OK) return rc;
    S = Staging{{h_base, 0}, {d_base, 0}};
    carve(S);
    return OVS_OK;
}

}  // namespace ovs
