// match_common.h -- the matcher handle shared by match_bruteforce.cu, match_window.cu, two_view_ransac.cu,
// two_view_triangulate.cu, initializer.cu, tracking_search.cu and fuse.cu.  Its arenas
// grow and are carved through staging.h.
#pragma once
#include <algorithm>
#include <vector>
#include "ovs_common.h"
#include "staging.h"

// device buffer of a released frame index, kept for the next ovs_frame_index_create* (one per frame in a tracking loop:
// cudaMalloc / cudaFree per frame would serialise every stream of the device)
struct ovs_index_buf { uint8_t* base = nullptr; size_t cap = 0; };

struct ovs_matcher {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 132;
    // grow-only device / pinned scratch
    uint8_t* d_q = nullptr; size_t d_q_cap = 0;
    uint8_t* d_t = nullptr; size_t d_t_cap = 0;
    unsigned* d_part = nullptr; size_t d_part_cap = 0;
    unsigned* d_keys = nullptr; size_t d_keys_cap = 0;
    unsigned* d_mask = nullptr; size_t d_mask_cap = 0;
    unsigned* h_keys = nullptr; size_t h_keys_cap = 0;  // pinned
    uint8_t* h_stage = nullptr; size_t h_stage_cap = 0; // pinned
    // the essential solver's own arenas (two_view_ransac.cu): a solve leaves the brute-force buffers above untouched
    uint8_t* d_ess = nullptr; size_t d_ess_cap = 0;
    uint8_t* h_ess = nullptr; size_t h_ess_cap = 0;     // pinned
    // the homography / fundamental-matrix solvers' own arenas (two_view_ransac.cu)
    uint8_t* d_tv = nullptr; size_t d_tv_cap = 0;
    uint8_t* h_tv = nullptr; size_t h_tv_cap = 0;       // pinned
    // the two-view triangulator's and create_new_landmarks' own arenas (two_view_triangulate.cu, match_window.cu)
    uint8_t* d_tri = nullptr; size_t d_tri_cap = 0;
    uint8_t* h_tri = nullptr; size_t h_tri_cap = 0;     // pinned
    // map initialisation's own arenas (initializer.cu): its solves and kernels leave the solver entry points' buffers untouched
    uint8_t* d_init = nullptr; size_t d_init_cap = 0;
    uint8_t* h_init = nullptr; size_t h_init_cap = 0;   // pinned
    // the tracker's per-landmark geometry (tracking_search.cu): its kernel leaves the matchers' buffers untouched
    uint8_t* d_trk = nullptr; size_t d_trk_cap = 0;
    uint8_t* h_trk = nullptr; size_t h_trk_cap = 0;     // pinned
    // match::fuse::replace_duplication's batched search (fuse.cu): every target's index and the queries, staged per call
    uint8_t* d_fuse = nullptr; size_t d_fuse_cap = 0;
    uint8_t* h_fuse = nullptr; size_t h_fuse_cap = 0;   // pinned
    cudaEvent_t ev[2]{};
    float last_kernel_us = 0.f;
    int num_requeries = 0;   // GPU re-queries issued by the greedy replays so far (diagnostic)
    std::vector<ovs_index_buf> index_pool;
};

namespace ovs {
// the matcher a frame index was built on (match_window.cu): the composed tracking calls (tracking_search.cu) run on its stream
ovs_matcher* frame_index_matcher(const ovs_frame_index* f);
// data::assign_keypoints_to_grid (match_window.cu): the rank order of n keypoints -- sorted by (cell_x, cell_y, index), the order
// frame::get_keypoints_in_cell visits them; keypoints outside the grid get no rank -- and the CSR of cell starts (cols * rows + 1)
std::vector<int> rank_keypoints(const ovs_grid& grid, int n, const float* x, const float* y, std::vector<int>& rank_to_idx,
                                std::vector<int>& idx_to_rank, int* nranked);
// the checks every call taking an ovs_frame_geometry makes (tracking_search.cu)
int check_geometry(const ovs_frame_geometry* g);
}  // namespace ovs
