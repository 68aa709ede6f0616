// ovs_common.h -- shared host-side helpers of libovs_b200 (error reporting, launch counting).
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ovs_b200.h"

namespace ovs {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Checks that `device` exists and is a Hopper sm_90 part (H100); selects it.  No CPU fallback.
int select_device(int device);

// Host waits.  Default: spin (cudaStreamSynchronize), the lowest latency for one camera stream per GPU.  With
// ovs_set_wait_mode(1) the calling thread sleeps on a blocking event instead, so that many streams (host
// threads) per GPU do not each burn a core while the device works.
bool blocking_waits();
cudaError_t sync_stream(cudaStream_t st);
cudaError_t sync_event(cudaEvent_t ev);
unsigned event_flags();   // flags for events a handle will cudaEventSynchronize() on

}  // namespace ovs

#define OVS_CUDA_CHECK(expr)                                                                      \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            ovs::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return OVS_ERR_CUDA;                                                                  \
        }                                                                                         \
    } while (0)

#define OVS_LAUNCH_CHECK()                                                                        \
    do {                                                                                          \
        ovs::count_launch();                                                                      \
        cudaError_t _e = cudaGetLastError();                                                      \
        if (_e != cudaSuccess) {                                                                  \
            ovs::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
            return OVS_ERR_CUDA;                                                                  \
        }                                                                                         \
    } while (0)

#define OVS_REQUIRE(cond, code, ...)      \
    do {                                  \
        if (!(cond)) {                    \
            ovs::set_error(__VA_ARGS__);  \
            return (code);                \
        }                                 \
    } while (0)
