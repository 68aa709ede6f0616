// optimize.cu -- H100 (sm_90a) implementation of openvslam::optimize::pose_optimizer::optimize and
// openvslam::optimize::local_bundle_adjuster::optimize (optimize/pose_optimizer.cc,
// optimize/local_bundle_adjuster.cc), replacing the g2o call they make: Levenberg-Marquardt with
// g2o's damping schedule, Huber kernel, landmarks marginalised by the Schur complement, dense
// Cholesky on the reduced camera system.  All arithmetic FP64 (g2o computes in double; the
// north-star tolerance is 1e-4 relative on the final reprojection error).
//
// Local BA, per LM iteration (state on the device, one host sync per batch of LM trials):
//   k_ba_linearize         per observation: residual, Jacobians, robust weight -> one edge record {Jp, Jl, ww, e};
//                          per landmark: Hll, bl           (observations are grouped by landmark)
//   k_ba_pose_accum_chunk  per free keyframe: Hpp, bp      (two-stage deterministic reduction over its edge
//   / _final               list)
//  per batch of up to 4 speculative LM trials (damping values lambda, 2 lambda, 8 lambda, 64 lambda):
//   k_ba_schur_chunk       per keyframe pair (a <= b): S_ab = Hpp - sum_l Y_al Hpl_bl'  over the landmarks both
//                          keyframes observe (co-observation lists sorted on the device once per call),
//                          b_S = bp - sum Y bl, on the FP64 tensor cores (DMMA)          -- no atomics
//   k_ba_cholesky_solve    one 8-CTA cluster per trial: blocked (32) look-ahead Cholesky of the dense reduced
//                          system (DMMA trailing update / panel GEMM) + both triangular solves
//   k_ba_update            landmarks: back-substitution + update; keyframes: exp-map update;
//                          LM scale term  x'(lambda x + b)
//   k_ba_errors            per observation: residuals at the trial state, robust chi2
//   k_ba_reduce            deterministic final sums -> pinned mapped host memory
//
// Pose optimiser: the whole optimize() (num_trials rounds x num_each_iter LM iterations, outlier
// re-classification between rounds) is ONE kernel on an 8-CTA cluster (edges sliced over the CTAs, 6x6 normal equations
// reduced through distributed shared memory in a fixed order); the system is 6x6.
//
// Transform optimiser (loop closure, optimize::transform_optimizer): the same shape with one Sim3 vertex and a 7x7
// system -- both rounds, the outlier cut, the early exit and the write-back are ONE kernel, k_sim3_optimize.
// The two kernels share the cluster reduction (ClusterSum), the Levenberg round (cluster_lm_round) and the packed SPD
// solve (ovs::solve_spd, ba_math.cuh); each keeps its own edge pass, update and round structure.
//
// Pose graph (loop closure, optimize::graph_optimizer): one Sim3 vertex per keyframe, a dense 7 n_free system assembled per trial
// batch (k_pg_*) and factorised by the local BA's solver, under the same device-side Levenberg controller (LmCtl, k_ba_reduce,
// lm_round); see the section at the end of this file.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <sched.h>
#include <time.h>
#include <vector>


#include "ba_math.cuh"
#include "block_sum.cuh"
#include "ovs_common.h"
#include "pnp_math.cuh"
#include "ransac.cuh"
#include "sim3_math.cuh"
#include "staging.h"

namespace {

using ovs::Arena;
using ovs::CameraD;

constexpr int kMaxReducedDimBig = 6000;  // 1000 free keyframes: beyond this the dense (n + 1) x n x 4 systems alone are > 1 GB
// (the cluster Cholesky takes n <= 684, i.e. 114 free keyframes: its (n + 4) x 36 panel must fit in shared memory)
constexpr int kCholMaxDynSmem = 226 * 1024;  // 227 KB opt-in limit minus the kernel's static shared memory
constexpr int kNB = 32;
constexpr int kCholThreads = 512;   // 16 warps: 128 registers per thread for the unrolled panel solve
constexpr int kCholCluster = 8;     // CTAs sharing the trailing update of the reduced system
constexpr int kPoseThreads = 256;
constexpr int kPoseCluster = 8;     // portable cluster size

// ------------------------------------------------------------------------------ reductions
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum of v over the block (blockDim.x multiple of 32, <= 1024); result valid in every thread.
__device__ double block_sum(double v, double* smem /* >= 33 */) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    double t = 0;
    for (int k = 0; k < nw; ++k) t += smem[k];
    return t;
}

__device__ __forceinline__ void atomic_max_pos(double* addr, double v) {
    // non-negative doubles order like their bit patterns
    atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

// ---- thread-block cluster primitives (barrier, rank, distributed shared memory load)
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::);
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::);
}
__device__ __forceinline__ unsigned cluster_size() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;\n" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned cluster_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r)); return r; }
__device__ __forceinline__ double ld_dsmem(const double* local_ptr, unsigned rank) {
    const unsigned addr = (unsigned)__cvta_generic_to_shared(local_ptr);
    unsigned remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(addr), "r"(rank));
    double v;
    asm volatile("ld.shared::cluster.f64 %0, [%1];\n" : "=d"(v) : "r"(remote));
    return v;
}
__device__ __forceinline__ void st_dsmem(double* local_ptr, unsigned rank, double v) {
    const unsigned addr = (unsigned)__cvta_generic_to_shared(local_ptr);
    unsigned remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(addr), "r"(rank));
    asm volatile("st.shared::cluster.f64 [%0], %1;\n" :: "r"(remote), "d"(v) : "memory");
}
// cluster barrier that also orders ordinary / distributed shared-memory accesses for the compiler
__device__ __forceinline__ void cluster_sync_mem() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// Sum of up to NS per-thread values over a cluster of CLUSTER CTAs of THREADS threads each, the same bits in every CTA: each
// value is summed over the warp, then over the warps in index order, then over the ranks in rank order.  Every CTA pushes its
// block sums into slot [its rank] of EVERY CTA's shared memory (st.shared::cluster), one cluster barrier (release / acquire)
// makes them visible, every CTA adds the slots in rank order.  The slots are double-buffered by the parity of the reduction,
// so one barrier per reduction is enough: a CTA that is already pushing reduction q + 1 writes the other buffer, and it can
// only push reduction q + 2 after every CTA has arrived at barrier q + 1, i.e. has finished reading buffer q.
// Every thread of the cluster calls it; the result stays valid until the next call.
template <int NS, int CLUSTER, int THREADS>
struct ClusterSum {
    int parity = 0;
    __device__ __forceinline__ const double* operator()(const double* acc, int count) {
        constexpr int NW = THREADS / 32;
        __shared__ double sm_red[NS][NW];
        __shared__ double s_slots[2][CLUSTER][NS];
        __shared__ double s_sys[NS];
        const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
        const unsigned rank = cluster_rank();
        __syncthreads();
        for (int k = 0; k < count; ++k) {
            const double v = warp_sum(acc[k]);
            if (lane == 0) sm_red[k][wid] = v;
        }
        __syncthreads();
        if (tid < count) {
            double t = 0;
#pragma unroll
            for (int k = 0; k < NW; ++k) t += sm_red[tid][k];
#pragma unroll
            for (unsigned r = 0; r < (unsigned)CLUSTER; ++r) st_dsmem(&s_slots[parity][rank][tid], r, t);
        }
        cluster_sync_mem();
        if (tid < count) {
            double v = 0;
#pragma unroll
            for (int r = 0; r < CLUSTER; ++r) v += s_slots[parity][r][tid];
            s_sys[tid] = v;
        }
        parity ^= 1;
        __syncthreads();
        return s_sys;
    }
};

// Speculative Levenberg trials: g2o rejects a step by multiplying lambda by ni (2, 4, 8, ...), so the
// damping values of the next trials are known in advance.  kSpec of them are evaluated in one batch
// (blockIdx.y / cluster index = trial) and then walked in order, exactly as the sequential loop would.
//
// The whole Levenberg state lives in DEVICE memory (LmCtl): the accept / reject walk, the damping schedule, the
// ring slot of the current estimate and the termination flags are updated by the one-thread tail of k_ba_reduce
// (and by k_ba_pose_final_plan at the start of an iteration), every other kernel reads its damping values / ring slots /
// "is there anything to do" from it.
// The host enqueues, per round, a static launch sequence (per iteration: linearisation, plan, ONE trial batch of 4) and
// waits once at the end of the round.  In the rare case that all four trials of an iteration are rejected (in practice: the
// last iteration of a converged round, which g2o ends after 10 rejected trials) the device halts itself (need_more; the
// launches already enqueued exit at their first instruction), and the host enqueues the remaining trials of that iteration
// (4 + 2) and, if the round goes on, the remaining iterations.
constexpr int kSpec = 4;
constexpr int kMaxTrials = 10;    // g2o: _maxTrialsAfterFailure
struct LmCtl {
    // g2o OptimizationAlgorithmLevenberg state
    double lambda, ni, currentChi, rho;
    // next trial batch: damping values, the ni each trial would be followed by if rejected, ring slots of the candidates
    double lam[kSpec], ni_after[kSpec];
    int buf[kSpec];
    int nbatch;        // trials in the next batch; 0 = nothing to do (the batch's kernels return at once)
    int cur;           // ring index of the current estimate
    int err_slot;      // slot of derr holding edge->_error as of the last trial the sequential loop evaluated
    int it;            // iterations of this round completed
    int qmax;          // trials of the current iteration so far
    int active;        // the round's `for (it < iterations && ok)` loop is still running
    int iterations;    // iteration budget of this round
    int use_huber;
    int stopped;       // force_stop_flag was seen
    int spec_width;    // width of the first batch of an iteration
    int round_live;    // this optimize() call was entered (the reference skips its second call when stopped)
    int need_more;     // the enqueued trial batch was rejected entirely: the device halted, the host must enqueue the rest
    int pending_nbatch;
    // statistics (ovs_ba_stats)
    int num_rounds, num_iterations, num_trials, batches, solver_trials;
    int round_iterations[8];
    double lambda_init[8];
    double last_chi2, last_lambda;
};

struct BaDev {
    CameraD cam;
    int K, L, M, nfree, n;
    const double* poses; const double* points;   // state being linearised / evaluated (set from the ring inside the kernels)
    const double* poses_ring; const double* points_ring;   // kSpec + 1 slots each
    const int* obs_kf; const int* obs_lm; const float2* obs_xy; const float* obs_xr; const float* inv_sigma_sq;
    const unsigned char* level;
    const int* free_idx;      // K
    const int* lm_first;      // L + 1
    int use_huber; double delta;
};

// --------------------------------------------------------------------------- linearisation
// Edge record: what the normal equations of an edge are made of, {Jp (R x 6), Jl (R x 3), ww, e (R)}, padded to an even
// number of doubles (16-byte aligned records).  R = 2 for a problem without stereo edges, 3 otherwise (chosen in prepare).
// The per-edge blocks Jp'WJl, Jl'WJl, Jp'WJp and the gradients are formed from it where they are read (ba_math.cuh,
// edge_*): storing the products costs far more memory traffic than forming them again.  Jp, Jl and ww come first, so the
// gathers that only need Jp'WJl read a prefix of the record.
template <int R> struct EdgeRec {
    static constexpr int kJl = 6 * R, kWw = 9 * R, kE = 9 * R + 1;
    static constexpr int kSize = (10 * R + 2) / 2 * 2;     // doubles per record: 22 (R = 2), 32 (R = 3)
    static constexpr int kHpl2 = (9 * R + 2) / 2;          // double2 loads covering Jp, Jl, ww
    static constexpr int kTail0 = 9 * R / 2, kTail1 = (10 * R + 2) / 2;   // double2 loads [kTail0, kTail1) cover ww and e
};
// landmark block table of k_ba_linearize (k_ba_landmark_blocks): segments of kLbSegEdges edges, up to kLbSegCap blocks each
constexpr int kLbSegEdges = 2048, kLbSegCap = 2 * (kLbSegEdges / 128) + 2, kLbThreads = 256;
// rows of edge i: 3 for a stereo observation of a 3-row problem
template <int R> __device__ __forceinline__ int edge_dim(const BaDev& P, size_t i) { return R == 3 && P.obs_xr[i] >= 0.0f ? 3 : 2; }

// One block per entry of the landmark block table ({first landmark, end landmark, first edge, end edge}: consecutive
// landmarks with at most 128 edges in all, k_ba_landmark_blocks; grid = segments x kLbSegCap), one thread per edge.  A thread evaluates its edge and
// stores the record; the records are staged in shared memory and leave the block as contiguous 16-byte stores.  Edges
// outside the graph (outliers of the first round) store zeros, edges on fixed keyframes a zero Jp; no consumer reads them.
// The landmark blocks Hll, bl are summed here too, one thread per landmark, sequentially in edge order from 0.0 over the
// per-edge Jl'WJl / bl parked in shared memory.  A landmark with more than 128 edges has a block of its own and walks its
// edges in passes of 128, its thread carrying the sums.
template <int R>
__global__ void __launch_bounds__(128) k_ba_linearize(BaDev P, const LmCtl* __restrict__ ctl, const int* __restrict__ nblocks,
                                                       const int4* __restrict__ lblocks, double* __restrict__ rec,
                                                       double* __restrict__ Hll, double* __restrict__ bl, double* __restrict__ maxdiag) {
    using ER = EdgeRec<R>;
    constexpr int RS = ER::kSize;
    __shared__ __align__(16) double s_rec[128 * RS];
    __shared__ double s_hll[128 * 6], s_bl[128 * 3];
    __shared__ unsigned char s_live[128];
    if (!ctl->active || (int)(blockIdx.x % kLbSegCap) >= nblocks[blockIdx.x / kLbSegCap]) return;
    P.poses = P.poses_ring + (size_t)ctl->cur * 12 * P.K; P.points = P.points_ring + (size_t)ctl->cur * 3 * P.L;
    P.use_huber = ctl->use_huber;
    const int4 blk = lblocks[blockIdx.x];
    const int t = threadIdx.x;
    double H[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0}, md = 0;
    for (int base = blk.z; base < blk.w; base += 128) {
        const int i = base + t;
        const int nedge = min(128, blk.w - base);
        const bool live = i < blk.w && !P.level[i];
        int dim = 0, fi = -1;
        double e[3] = {0, 0, 0}, Jp[18], Jl[9], ww = 0;
#pragma unroll
        for (int k = 0; k < 18; ++k) Jp[k] = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) Jl[k] = 0;
        if (live) {
            const int kf = P.obs_kf[i], lm = P.obs_lm[i];
            fi = P.free_idx[kf];
            const float xr = P.obs_xr ? P.obs_xr[i] : -1.0f;
            const bool stereo = xr >= 0.0f;
            const float2 xy = P.obs_xy[i];
            const double obs[3] = {(double)xy.x, (double)xy.y, (double)xr};
            double pose[12], pw[3];
#pragma unroll
            for (int k = 0; k < 12; ++k) pose[k] = P.poses[12 * (size_t)kf + k];
#pragma unroll
            for (int k = 0; k < 3; ++k) pw[k] = P.points[3 * (size_t)lm + k];
            dim = ovs::edge_eval(P.cam, pose, pw, obs, stereo, e, Jp, Jl);
            const double w = (double)P.inv_sigma_sq[i];
            double chi = 0;
            for (int d = 0; d < dim; ++d) chi += w * e[d] * e[d];
            double rho0 = chi, rho1 = 1.0;
            if (P.use_huber) ovs::huber(chi, P.delta, &rho0, &rho1);
            ww = rho1 * w;
        }
        {
            double* r = s_rec + RS * t;
            const bool fr = fi >= 0;
#pragma unroll
            for (int k = 0; k < 6 * R; ++k) r[k] = fr ? Jp[k] : 0.0;
#pragma unroll
            for (int k = 0; k < 3 * R; ++k) r[ER::kJl + k] = Jl[k];
            r[ER::kWw] = ww;
#pragma unroll
            for (int k = 0; k < R; ++k) r[ER::kE + k] = e[k];
#pragma unroll
            for (int k = ER::kE + R; k < RS; ++k) r[k] = 0.0;
            ovs::edge_hll<R>(Jl, ww, dim, s_hll + 6 * t);
            ovs::edge_bl<R>(Jl, ww, e, dim, s_bl + 3 * t);
            s_live[t] = live ? 1 : 0;
        }
        __syncthreads();
        {
            const double2* s2 = reinterpret_cast<const double2*>(s_rec); double2* g2 = reinterpret_cast<double2*>(rec + RS * (size_t)base);
            for (int q = t; q < (RS / 2) * nedge; q += 128) g2[q] = s2[q];
        }
        for (int l = blk.x + t; l < blk.y; l += 128) {     // several passes only for a block of one landmark (thread 0)
            const int p0 = max(P.lm_first[l], base), p1 = min(P.lm_first[l + 1], base + nedge);
            if (blk.y - blk.x > 1) {
#pragma unroll
                for (int k = 0; k < 6; ++k) H[k] = 0;
#pragma unroll
                for (int k = 0; k < 3; ++k) b[k] = 0;
            }
            for (int p = p0; p < p1; ++p) {
                if (!s_live[p - base]) continue;
#pragma unroll
                for (int k = 0; k < 6; ++k) H[k] += s_hll[6 * (p - base) + k];
#pragma unroll
                for (int k = 0; k < 3; ++k) b[k] += s_bl[3 * (p - base) + k];
            }
            if (base + 128 >= blk.w) {                   // the landmark's last pass
#pragma unroll
                for (int k = 0; k < 6; ++k) Hll[6 * (size_t)l + k] = H[k];
#pragma unroll
                for (int k = 0; k < 3; ++k) bl[3 * (size_t)l + k] = b[k];
                md = fmax(md, fmax(fabs(H[0]), fmax(fabs(H[3]), fabs(H[5]))));
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, o));
    if ((threadIdx.x & 31) == 0 && md > 0) atomic_max_pos(maxdiag, md);
}

// Hpp / bp of the free keyframes: two-stage deterministic reduction over the (a, a) co-observation
// segment of each keyframe (its edge list), cut into chunks of 128 edges (one edge per thread) so the
// dependent-load latency of a chunk overlaps with that of many others.  Each thread forms its edge's
// Jp'WJp and -Jp'We from the record (Jp, ww, e).
// chunk = {keyframe a, begin, end, unused}; ppart[chunk][27] = {Hpp packed 21, bp 6}.
template <int R>
__global__ void __launch_bounds__(128) k_ba_pose_accum_chunk(BaDev P, const LmCtl* __restrict__ ctl, const int* __restrict__ nchunks,
                                                              const int4* __restrict__ pair_rec, const int4* __restrict__ chunks,
                                                              const double* __restrict__ rec, double* __restrict__ ppart) {
    using ER = EdgeRec<R>;
    __shared__ double red[27][4];
    if (!ctl->active || (int)blockIdx.x >= *nchunks) return;
    const int4 ch = chunks[blockIdx.x];
    const int e = ch.y + threadIdx.x;
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) acc[k] = 0;
    if (e < ch.z) {
        const int4 pr = pair_rec[e];           // diagonal pair: both edges are this keyframe's edge
        const int o = pr.x;
        if (!pr.w) {
            const double2* r2 = reinterpret_cast<const double2*>(rec + ER::kSize * (size_t)o);
            double r[2 * ER::kTail1];
#pragma unroll
            for (int k = 0; k < 3 * R; ++k) { const double2 v = r2[k]; r[2 * k] = v.x; r[2 * k + 1] = v.y; }
#pragma unroll
            for (int k = ER::kTail0; k < ER::kTail1; ++k) { const double2 v = r2[k]; r[2 * k] = v.x; r[2 * k + 1] = v.y; }
            const int dim = edge_dim<R>(P, o);
            ovs::edge_hpp<R>(r, r[ER::kWw], dim, acc);
            ovs::edge_bp<R>(r, r[ER::kWw], r + ER::kE, dim, acc + 21);
        }
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 27; ++k) {
        const double v = warp_sum(acc[k]);
        if (lane == 0) red[k][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x < 27)
        ppart[27 * (size_t)blockIdx.x + threadIdx.x] = red[threadIdx.x][0] + red[threadIdx.x][1] + red[threadIdx.x][2] + red[threadIdx.x][3];
}

// Second stage of the Hpp / bp reduction AND the plan of the iteration, in one single-block kernel: the final
// sums are a few thousand short ordered additions, and the thread that plans the trial batch needs their largest diagonal
// entry anyway (computeLambdaInit).  Declared here, defined after the control-block helpers.
__global__ void k_ba_pose_final_plan(LmCtl* ctl, int nfree, const int* __restrict__ kf_chunk_begin, const double* __restrict__ ppart,
                                     double* __restrict__ Hpp, double* __restrict__ bp, double* maxdiag, int* fail,
                                     const volatile int* stop_word, volatile int* mirror);

// ------------------------------------------------------------------------------ per trial
// (Hll + lambda I)^-1 of a landmark is not stored: the kernels that need it (Schur complement, back-substitution) form it from
// the 3 x 3 block Hll and the damping value -- ~30 flops against a dependent 48-byte gather per damping value.
// FP64 tensor-core MMA (DMMA), D(8x8) += A(8x4) * B(4x8).  Fragment layout (PTX ISA, m8n8k4 .f64):
// a = A[lane >> 2][lane & 3], b = B[lane & 3][lane >> 2], d0/d1 = D[lane >> 2][2 * (lane & 3) + {0, 1}].
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// Schur complement, two-stage and deterministic.  Stage 1: one block (4 warps) per chunk of <= 128
// co-observations of a keyframe pair (a <= b).  Each lane loads the blocks of ONE co-observation
// (Hpl_a, Hpl_b, the shared landmark's (Hll + lambda I)^-1), forms Y_a = Hpl_a Hll^-1 and parks Y_a and
// Hpl_b in shared memory; the warp then accumulates  sum_e Y_a,e (6x3) Hpl_b,e' (3x6)  as ONE GEMM on the
// FP64 tensor cores: A = [Y_1 Y_2 ...] (6 x 3E), B = [W_1 W_2 ...]' (3E x 6), K = 3E walked four at a time,
// i.e. three m8n8k4 DMMAs per four co-observations, no K padding and no cross-lane reduction.
// On diagonal pairs the rhs contribution  sum_e Hpl_e z_e = sum_e Hpl_e (Hll + lambda I)^-1 bl = sum_e Y_e bl
// rides along as column 6 of B (B[3e + k][6] = bl_e[k]) -- same A operand, no extra MMA.
// chunk = {pair id, begin, end, unused}; spart[chunk][42] = {S_ab partial 36, b_S partial 6}.
// The kernel is bound by dependent L2 round trips at low occupancy, so the chain is kept short: one 16-byte record per
// co-observation carries both edge indices, the landmark and the "either edge excluded" flag (no index chasing); the
// (Hll + lambda I)^-1 of the NEXT damping value is in flight while the current one is multiplied; four independent DMMA
// accumulator chains; the partial blocks of all damping values stay in registers and meet in ONE cross-warp reduction.
// 4 blocks per SM on purpose (registers): the solver's clusters need several SMs of one GPC with their whole shared memory
// free at the same time, and denser Schur blocks starve them when several camera streams share the GPU.
// Shared-memory layout of the DMMA operands: FRAGMENT ORDER.  A warp's 32 co-observations form 8 groups of four; the K = 12 slots
// of a group are walked by three DMMAs; element (row r, K slot 4 t + k) of group g sits at g * pitch + t * rows * 4 + r * 4 + k
// (rows = 6 for Y, 7 for W: Hpl_b and the bl column), so the lanes of a DMMA read consecutive doubles (2 wavefronts, the minimum
// for 64-bit accesses).  The pitches are = 4 or 12 mod 16, which makes the producer side conflict free as well (lane = co-observation
// 4 g + en writes element (r, kc) to K slot 3 en + kc: the sixteen lanes of a half warp hit banks 4 g' + k, all different).
// A record-per-lane layout costs 3-4 wavefronts per fragment load.  41 KB per block: the solver's clusters need SMs with free
// shared memory while eight streams share the GPU, a larger footprint here costs more there than it saves.
constexpr int kSGY = 76, kSGW = 84;
template <int R>
__global__ void __launch_bounds__(128, 4) k_ba_schur_chunk(BaDev P, const LmCtl* __restrict__ ctl, const int* __restrict__ nchunks,
                                                         const int4* __restrict__ pair_rec, const int4* __restrict__ chunks,
                                                         const int2* __restrict__ pair_ab, const double* __restrict__ Hll,
                                                         const double* __restrict__ rec, const double* __restrict__ bl,
                                                         double* __restrict__ spart, size_t spart_stride) {
    using ER = EdgeRec<R>;
    // The Jacobian blocks Hpl_a, Hpl_b of a co-observation do not depend on lambda: they are loaded once
    // and all `nbatch` speculative damping values are processed by the same block (only (Hll + lambda I)^-1
    // differs).  per warp: 32 co-observations x {Y (6x3), W = Hpl_b (6x3) + bl (3)}
    __shared__ double s_y[4 * 8 * kSGY];      // after the last damping value: the cross-warp reduction buffer [kSpec][4][64]
    __shared__ double s_w[4 * 8 * kSGW];
    double* sYw = s_y + (threadIdx.x >> 5) * 8 * kSGY;
    double* sWw = s_w + (threadIdx.x >> 5) * 8 * kSGW;
    static_assert(4 * 8 * kSGY >= kSpec * 4 * 64, "reduction buffer must fit in the Y region");
    const int nbatch = ctl->nbatch;
    if (nbatch == 0 || (int)blockIdx.x >= *nchunks) return;
    const int4 ch = chunks[blockIdx.x];
    const int2 ab = pair_ab[ch.x];
    const bool diag = ab.x == ab.y;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int e = ch.y + threadIdx.x;
    double wa[18], hl[6] = {0, 0, 0, 0, 0, 0};
    int lm = -1;
    {
        // Hpl_a, Hpl_b are formed from the prefix {Jp, Jl, ww} of the two edge records; Hpl_b goes to shared memory element by
        // element as it is formed, Hpl_a stays in registers.  Two-row records: all loads are issued first.  Three-row records
        // do not fit in registers together with the rest: record b is loaded into the registers of record a, which is loaded
        // once Hpl_b is parked.
        constexpr bool kLoadAFirst = R == 2;
        double gl[3] = {0, 0, 0}, ra[2 * ER::kHpl2], rb2[2 * ER::kHpl2];
        double (&rb)[2 * ER::kHpl2] = kLoadAFirst ? rb2 : ra;
        const double2* pa = nullptr;
        bool live = false, same = true;
        int da = 2, db = 2;
        auto load_rec = [](const double2* p, double (&r)[2 * ER::kHpl2]) {
#pragma unroll
            for (int k = 0; k < ER::kHpl2; ++k) { const double2 v = p[k]; r[2 * k] = v.x; r[2 * k + 1] = v.y; }
        };
#pragma unroll
        for (int k = 0; k < 18; ++k) wa[k] = 0;
        if (e < ch.z) {
            const int4 ob = pair_rec[e];      // {edge on a, edge on b, landmark, either edge excluded}
            if (!ob.w) {
                live = true;
                lm = ob.z;
                same = ob.x == ob.y;             // the records of a diagonal pair name the same edge twice (uniform over such a chunk)
                pa = reinterpret_cast<const double2*>(rec + ER::kSize * (size_t)ob.x);
                if (kLoadAFirst || same) load_rec(pa, ra);
                if (!same) load_rec(reinterpret_cast<const double2*>(rec + ER::kSize * (size_t)ob.y), rb);
                const double2* ph = reinterpret_cast<const double2*>(Hll + 6 * (size_t)lm);
#pragma unroll
                for (int k = 0; k < 3; ++k) { const double2 v = ph[k]; hl[2 * k] = v.x; hl[2 * k + 1] = v.y; }
                if (diag) { gl[0] = bl[3 * (size_t)lm]; gl[1] = bl[3 * (size_t)lm + 1]; gl[2] = bl[3 * (size_t)lm + 2]; }
                da = edge_dim<R>(P, ob.x); db = edge_dim<R>(P, ob.y);
            }
        }
        // B operand: element (column c, K slot 3 en + kc) = Hpl_b[c][kc] (c < 6), bl[kc] (c = 6); column 7 is never read
        int sb[3];
#pragma unroll
        for (int kc = 0; kc < 3; ++kc) { const int kk = 3 * (lane & 3) + kc; sb[kc] = (lane >> 2) * kSGW + (kk >> 2) * 28 + (kk & 3); }
        auto park = [&](int c, int kc, double v) { sWw[sb[kc] + 4 * c] = v; };
        if (!live) {
#pragma unroll
            for (int c = 0; c < 6; ++c)
#pragma unroll
                for (int kc = 0; kc < 3; ++kc) park(c, kc, 0.0);
        } else if (same) {
            ovs::edge_hpl_each<R>(ra, ra + ER::kJl, ra[ER::kWw], da, park);
        } else {
            ovs::edge_hpl_each<R>(rb, rb + ER::kJl, rb[ER::kWw], db, park);
        }
#pragma unroll
        for (int kc = 0; kc < 3; ++kc) sWw[sb[kc] + 24] = gl[kc];
        if (live) {
            if (!kLoadAFirst && !same) load_rec(pa, ra);
            ovs::edge_hpl<R>(ra, ra + ER::kJl, ra[ER::kWw], da, wa);
        }
    }
    // (Hll + lambda I)^-1 of this lane's landmark for damping value bt (zeros for an inactive lane or a singular block: the
    // back-substitution kernel flags the trial as failed in that case)
    double lam[kSpec];
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) lam[bt] = ctl->lam[bt];
    auto make_dinv = [&](int bt, double (&di)[6]) {
        double D[6] = {hl[0] + lam[bt], hl[1], hl[2], hl[3] + lam[bt], hl[4], hl[5] + lam[bt]};
        if (lm < 0 || !ovs::inv3_sym(D, di)) {
#pragma unroll
            for (int q = 0; q < 6; ++q) di[q] = 0.0;
        }
    };
    // fragment coordinates of this lane: r = lane >> 2 is the row of A / the column of B (valid < 6; column 6 of B
    // carries bl), k = lane & 3 the K slot
    const int r = lane >> 2;
    int sbase[3];                                          // where this lane's co-observation parks element (row 0, kc)
#pragma unroll
    for (int kc = 0; kc < 3; ++kc) { const int kk = 3 * (lane & 3) + kc; sbase[kc] = (lane >> 2) * kSGY + (kk >> 2) * 24 + (kk & 3); }
    const bool rowA = r < 6, colB = r < 6 || (r == 6 && diag);
    double acc[kSpec][2];
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) { acc[bt][0] = 0; acc[bt][1] = 0; }
    // A keyframe pair with a few more than 128 co-observations leaves a second chunk that fills one warp or less; warps (and second
    // halves of warps) without records skip the products -- they would only add zeros (same bits).
    const int nrec_w = min(32, max(0, ch.z - (ch.y + 32 * wid)));     // records of this warp (warp-uniform)
    const bool second_half = nrec_w > 16;
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) {
        if (bt < nbatch && nrec_w > 0) {         // block-uniform && warp-uniform
            double di[6];
            make_dinv(bt, di);
            // Y_a = Hpl_a (Hll + lambda_bt I)^-1 for this lane's co-observation
            double ya[18];
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                const double w0 = wa[3 * a], w1 = wa[3 * a + 1], w2 = wa[3 * a + 2];
                ya[3 * a] = w0 * di[0] + w1 * di[1] + w2 * di[2];
                ya[3 * a + 1] = w0 * di[1] + w1 * di[3] + w2 * di[4];
                ya[3 * a + 2] = w0 * di[2] + w1 * di[4] + w2 * di[5];
            }
            __syncwarp();                           // the previous damping value's reads of Y are done
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                sYw[sbase[0] + 4 * a] = ya[3 * a]; sYw[sbase[1] + 4 * a] = ya[3 * a + 1]; sYw[sbase[2] + 4 * a] = ya[3 * a + 2];
            }
            __syncwarp();
            // four independent accumulator chains (groups 0/4, 1/5, 2/6, 3/7), added in a fixed order at the end
            double c0[2] = {0, 0}, c1[2] = {0, 0}, c2[2] = {0, 0}, c3[2] = {0, 0};
            const double* yb = sYw + lane;
            const double* wb = sWw + lane;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                if (half == 1 && !second_half) break;       // groups 4..7 hold the warp's records 16..31
#pragma unroll
                for (int t = 0; t < 3; ++t) {
                    const int oy = (4 * half) * kSGY + t * 24, ow = (4 * half) * kSGW + t * 28;   // groups 4 half .. 4 half + 3, DMMA t of each
                    const double a0 = rowA ? yb[oy] : 0.0, b0 = colB ? wb[ow] : 0.0;
                    const double a1 = rowA ? yb[oy + kSGY] : 0.0, b1 = colB ? wb[ow + kSGW] : 0.0;
                    const double a2 = rowA ? yb[oy + 2 * kSGY] : 0.0, b2 = colB ? wb[ow + 2 * kSGW] : 0.0;
                    const double a3 = rowA ? yb[oy + 3 * kSGY] : 0.0, b3 = colB ? wb[ow + 3 * kSGW] : 0.0;
                    dmma_m8n8k4(c0[0], c0[1], a0, b0);       // D[i][j] += sum_kk Y[i][kk] W[j][kk]  (j = 6: bl)
                    dmma_m8n8k4(c1[0], c1[1], a1, b1);
                    dmma_m8n8k4(c2[0], c2[1], a2, b2);
                    dmma_m8n8k4(c3[0], c3[1], a3, b3);
                }
            }
            acc[bt][0] = (c0[0] + c1[0]) + (c2[0] + c3[0]);
            acc[bt][1] = (c0[1] + c1[1]) + (c2[1] + c3[1]);
        }
    }
    // D[r][2k], D[r][2k+1] of every damping value live in this lane; combine the four warps in a fixed order
    __syncthreads();                                // every warp is done with its Y slice: the region becomes the reduction buffer
    double* red = s_y;                              // [bt][warp][64]
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt)
        if (bt < nbatch) { red[(bt * 4 + wid) * 64 + 2 * lane] = acc[bt][0]; red[(bt * 4 + wid) * 64 + 2 * lane + 1] = acc[bt][1]; }
    __syncthreads();
    for (int idx = threadIdx.x; idx < 42 * nbatch; idx += 128) {
        const int bt = idx / 42, t = idx - 42 * bt;
        // S block element (i, j): lane 4 i + j / 2, slot j & 1; rhs element i: column 6 = lane 4 i + 3, slot 0
        const int i = t < 36 ? t / 6 : t - 36;
        const int j = t < 36 ? t % 6 : 6;
        const int src = 2 * (4 * i + (j >> 1)) + (j & 1);
        const double* rb = red + (size_t)bt * 4 * 64;
        double v = rb[src] + rb[64 + src] + rb[128 + src] + rb[192 + src];
        if (j == 6 && !diag) v = 0.0;
        spart[(size_t)bt * spart_stride + 42 * (size_t)blockIdx.x + t] = v;
    }
}

// marks the co-observation records whose edges have left the graph (outlier cut between the rounds): rec.w = excluded
__global__ void __launch_bounds__(256) k_ba_pair_flags(const unsigned char* __restrict__ level, int4* __restrict__ rec, int n) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    int4 r = rec[i];
    r.w = (level[r.x] | level[r.y]) ? 1 : 0;
    rec[i] = r;
}

// Stage 2: one block per keyframe pair sums its chunks in order and writes S_ab (transposed into the
// lower triangle of the (n + 1) x n system matrix) and, on diagonal pairs, b_S (row n).
__global__ void __launch_bounds__(64) k_ba_schur_final(int n, const LmCtl* __restrict__ ctl, const int* __restrict__ pair_chunk_begin, const int2* __restrict__ pair_ab,
                                                        const double* __restrict__ spart, size_t spart_stride, const double* __restrict__ Hpp,
                                                        const double* __restrict__ bp, double* __restrict__ S, size_t S_stride) {
    const int pid = blockIdx.x, t = threadIdx.x;
    if ((int)blockIdx.y >= ctl->nbatch) return;
    const double lambda = ctl->lam[blockIdx.y];
    spart += (size_t)blockIdx.y * spart_stride; S += (size_t)blockIdx.y * S_stride;
    double* bS = S + (size_t)n * n;
    if (t >= 42) return;
    const int a = pair_ab[pid].x, b = pair_ab[pid].y;
    const bool diag = a == b;
    if (t >= 36 && !diag) return;
    double s = 0;
    const int c0 = pair_chunk_begin[pid], c1 = pair_chunk_begin[pid + 1];
#pragma unroll 4
    for (int c = c0; c < c1; ++c) s += spart[42 * (size_t)c + t];     // same order of additions, four loads in flight
    if (t < 36) {
        const int i = t / 6, j = t % 6;
        double v = -s;
        if (diag) v += Hpp[21 * (size_t)a + ovs::sym6(i, j)] + (i == j ? lambda : 0.0);
        S[(size_t)(6 * b + j) * n + 6 * a + i] = v;   // element (6a+i, 6b+j), stored at its transpose position
    } else {
        bS[6 * a + t - 36] = bp[6 * (size_t)a + t - 36] - s;
    }
}

// Blocked (32) Cholesky of the reduced camera system on a thread-block cluster, with the right-hand
// side carried as an extra matrix row so the forward substitution costs nothing:
//   A is (n + 1) x n row-major; rows 0..n-1 hold the lower triangle of S, row n holds b_S.
//   After the factorisation row n holds y = L^-1 b; a blocked back-substitution gives x.
// The critical path of a dense Cholesky is the chain of n dependent pivots (reciprocal square root,
// scale, broadcast).  It runs on ONE warp per CTA, redundantly in every CTA of the cluster (so the only
// inter-CTA traffic is the trailing matrix itself, in global memory / L2), and it runs ONE BLOCK AHEAD
// (look-ahead): while the other warps apply block step k to the trailing matrix, warp 0 updates the
// next 32 x 32 diagonal block itself (10 lower 8 x 8 tiles, DMMA) and factorises it.
// Per block step (all blocks but possibly the last are 32 wide):
//   warps 2..  panel rows (and the rhs row) by cp.async, row-major with a pitch of 36 doubles (every
//              access pattern below is then at most 2-way bank conflicted), then L21 = A21 L11^-T by
//              substitution, one row per thread, L11 read through a transposed copy with 128-bit
//              broadcast loads
//   warp 1     (CTA 0) inverse of the factorised diagonal block for the back-substitution
//   warp 0     look-ahead: next diagonal block -= its panel rows' outer product; factorisation with one
//              matrix row per lane in registers (identity padding when narrower than 32); the pivot of
//              column j+1 is formed in its own lane from the lane's own factor, so the chain per column
//              is fma -> shuffle -> rsqrt -> mul
//   warps 1..  the solved panel goes back to global memory (rows dealt over the cluster); trailing update
//              A22 -= L21 L21' on the FP64 tensor cores, one warp per 16 x 32 macro-tile = 2 x 4 DMMA
//              (m8n8k4) tiles whose accumulators start from the old values with negated A fragments;
//              the elements of the next diagonal block are left to warp 0 (never written here)
//   cluster barrier (release/acquire): the trailing matrix is complete and visible to every CTA.
// Dynamic shared memory: LdT (32 x 33) + invd (32) + vec (npad) + scr (32 x 33) + IL (32 x 36) + panel.
constexpr int kPP = 36;   // panel row pitch in doubles: 4 mod 16 makes DMMA fragment loads conflict free
__host__ __device__ __forceinline__ size_t chol_fixed_doubles(int n) { return (size_t)32 * 33 + 32 + ((n + 1 + 31) / 32) * 32 + 32 * 33 + 32 * kPP; }
__host__ __device__ __forceinline__ size_t chol_panel_doubles(int n) { return (size_t)(n + 4) * kPP; }
__host__ __device__ __forceinline__ int chol_back_pitch(int n) { return ((n + 3) / 4) * 4 + 4; }
__host__ __device__ __forceinline__ size_t chol_back_doubles(int n) { return (size_t)32 * 33 + (size_t)32 * chol_back_pitch(n); }

__global__ void __launch_bounds__(kCholThreads, 1)
k_ba_cholesky_solve(const LmCtl* __restrict__ ctl, double* __restrict__ A, size_t A_stride, int n, double* __restrict__ x, double* __restrict__ invL, size_t invL_stride,
                    int* __restrict__ fail, int dbuf) {
    {
        const int bt = blockIdx.x / (int)cluster_size();   // one cluster per speculative trial
        if (bt >= ctl->nbatch) return;                      // the whole cluster leaves together
        A += (size_t)bt * A_stride; x += (size_t)bt * n; invL += (size_t)bt * invL_stride; fail += bt;
    }
    extern __shared__ __align__(16) double sh[];
    const int npad = ((n + 1 + 31) / 32) * 32;
    double* LdT = sh;                       // 32 x 32 used: LdT[c * 32 + r] = L11[r][c] (the region is 32 x 33 for the back-substitution)
    double* invd = LdT + 32 * 33;           // 32 reciprocal pivots
    double* vec = invd + 32;                // npad
    double* scr = vec + npad;               // 32 x 33 scratch of warp 0: look-ahead tile in row layout, then the factor's columns
    double* IL = scr + 32 * 33;             // 32 x kPP: inverse of the current diagonal block (row-major), B operand of the panel GEMM
    double* P = IL + 32 * kPP;              // panel, row-major, pitch kPP                  // panel, row-major, pitch kPP
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int rank = (int)cluster_rank();
    const int ncta = (int)cluster_size();   // cluster width is a launch attribute (1, 2, 4 or 8)
    const int g = lane >> 2, q = lane & 3;
    __shared__ int s_fail;
    if (tid == 0) s_fail = 0;
    __syncthreads();
    const int nblk = (n + kNB - 1) / kNB;

    // factorisation of the 32 x 32 block held one row per lane in a[] (warp 0 only).  Column j of the factor goes to
    // cs[j * 32 + lane] as soon as it is final (that store is also how the lanes exchange it), so a[j] is dead after
    // step j; returns the lane's reciprocal pivot, raises s_fail on a non-positive pivot
    auto factor_block = [&](double (&a)[kNB], double* cs) {
        bool bad = false;
        double my_inv = 1.0;
        double ajj = __shfl_sync(0xffffffffu, a[0], 0);
        double inv = rsqrt(ajj);
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
            bad = bad || !(ajj > 0.0) || !isfinite(ajj);
            const double l = (lane >= j) ? a[j] * inv : 0.0;   // L[lane][j]
            if (lane == j) my_inv = inv;
            double* col = cs + j * 32;
            col[lane] = l;
            if (j + 1 < kNB) {
                // next pivot first, without the shared-memory round trip: in lane j+1 the factor L[j+1][j] is the
                // lane's own l, so fma(-l, l, a[j+1]) there IS the updated pivot (the bulk update below recomputes
                // the same value); its broadcast and reciprocal square root overlap the bulk update
                ajj = __shfl_sync(0xffffffffu, fma(-l, l, a[j + 1]), j + 1);
                inv = rsqrt(ajj);
            }
            __syncwarp();
#pragma unroll
            for (int c = j + 1; c < kNB; ++c) a[c] = fma(-l, col[c], a[c]);
        }
        if (bad && lane == 0) s_fail = 1;
        return my_inv;
    };

    // Iteration -1 is the prologue: no panel, only warp 0's look-ahead path, which then factorises block 0 straight
    // from global memory.  It shares the (fully unrolled, ~64 KB) factorisation code with the steady state, so that
    // code is fetched cold once per launch, not twice (a cold pass costs ~3x a warm one).
    for (int blk = -1; blk < nblk; ++blk) {
        const bool pro = blk < 0;
        const int kb = pro ? 0 : blk * kNB;
        const int nb = pro ? 0 : min(kNB, n - kb);
        const int rem = n - kb - nb;          // matrix rows below the block; the rhs row is row `rem` of the panel
        const int prow = rem + 1;             // panel rows including the rhs row
        const int nbn = min(kNB, rem);        // width of the next diagonal block (rows/cols 0..nbn-1 of the trailing matrix)
        // ---- panel rows (and the rhs row): one warp per row, lane = column: a coalesced 256 B global read and a
        //      conflict-free shared write per instruction
        if (wid >= 2 && !pro) {
            for (int r = wid - 2; r < prow; r += kCholThreads / 32 - 2) {
                if (lane < nb) {
                    const unsigned dst = (unsigned)__cvta_generic_to_shared(P + r * kPP + lane);
                    const double* src = A + (size_t)(kb + nb + r) * n + kb + lane;
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(dst), "l"(src));
                } else {
                    P[r * kPP + lane] = 0.0;      // columns of the identity padding of a narrow last block
                }
            }
            asm volatile("cp.async.commit_group;\n" ::);
            asm volatile("cp.async.wait_group 0;\n" ::);
        }
        if (!pro) {
            __syncthreads();                  // panel loaded; LdT / invd / s_fail of this block (look-ahead) visible
            if (s_fail) break;
        }
        // ---- panel: L21 = A21 L11^-T (rows below + rhs row) by substitution, one row per thread.  Warp 0 takes the
        //      first 32 rows itself -- they are all the look-ahead needs, so the chain diagonal block -> its 32 panel
        //      rows -> next diagonal block never waits for the rest of the panel; worker warps take the other rows.
        //      Warps 4, 8, 12 share warp 0's scheduler and FP64 pipe and sit these phases out: their FP64 work
        //      stretches the latency-bound chain (measured: 2.6x), and the chain is what a block step waits for.
        const bool worker = wid >= 2 && (wid & 3) != 0;
        const int nw = 11;                                   // worker warps per CTA: 2 3 5 6 7 9 10 11 13 14 15
        const int wk = wid - 2 - (wid >> 2);                 // 0 .. nw-1 for a worker
        if (wid == 0) {
            // old values of the next diagonal block: in flight (cp.async into scr) while the 32 rows are solved
            if (rem > 0) {
                for (int r = 0; r < nbn; ++r)
                    if (lane <= r) {
                        const unsigned dst = (unsigned)__cvta_generic_to_shared(scr + r * 33 + lane);
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(dst), "l"(A + (size_t)(kb + nb + r) * n + kb + nb + lane));
                    }
                asm volatile("cp.async.commit_group;\n" ::);
            }
            if (lane < prow && !pro) {
                const int r = lane;
                double xr[kNB];
                double* row = P + r * kPP;
#pragma unroll
                for (int c = 0; c < kNB; c += 2) {
                    const double2 v = *reinterpret_cast<const double2*>(row + c);
                    xr[c] = v.x; xr[c + 1] = v.y;
                }
#pragma unroll
                for (int c = 0; c < kNB; ++c) {
                    const double xc = xr[c] * invd[c];
                    xr[c] = xc;
#pragma unroll
                    for (int c2 = c + 1; c2 < kNB; ++c2) xr[c2] = fma(-xc, LdT[c * 32 + c2], xr[c2]);
                }
#pragma unroll
                for (int c = 0; c < kNB; c += 2) *reinterpret_cast<double2*>(row + c) = make_double2(xr[c], xr[c + 1]);
            }
            __syncwarp();
            if (rem == 0) {
                // last block: only the rhs row was left; there is no cluster barrier before the back-substitution,
                // so CTA 0 writes it itself
                if (rank == 0 && lane < nb) A[(size_t)(kb + nb) * n + kb + lane] = P[lane];
            } else {
                if (!pro) asm volatile("bar.arrive 3, 480;\n" ::: "memory");   // rows 0..31 of the panel are solved (workers wait on 3)
            // ---- look-ahead: next diagonal block (lower 8 x 8 tiles) -= P[0..31] P[0..31]', then its factorisation
            asm volatile("cp.async.wait_group 0;\n" ::: "memory");
            __syncwarp();
            double acc[4][4][2];
#pragma unroll
            for (int ti = 0; ti < 4; ++ti)
#pragma unroll
                for (int tj = 0; tj <= ti; ++tj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int rr = 8 * ti + g, cc = 8 * tj + 2 * q + e;
                        acc[ti][tj][e] = (rr < nbn && cc <= rr) ? scr[rr * 33 + cc] : 0.0;
                    }
            __syncwarp();                                        // scr is rewritten below
#pragma unroll 2
            for (int k4 = pro ? kNB : 0; k4 < kNB; k4 += 4) {
                double pv[4];
#pragma unroll
                for (int ti = 0; ti < 4; ++ti) pv[ti] = P[(8 * ti + g) * kPP + k4 + q];
#pragma unroll
                for (int ti = 0; ti < 4; ++ti)
#pragma unroll
                    for (int tj = 0; tj <= ti; ++tj) dmma_m8n8k4(acc[ti][tj][0], acc[ti][tj][1], -pv[ti], pv[tj]);
            }
#pragma unroll
            for (int ti = 0; ti < 4; ++ti)
#pragma unroll
                for (int tj = 0; tj <= ti; ++tj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) scr[(8 * ti + g) * 33 + 8 * tj + 2 * q + e] = acc[ti][tj][e];
            __syncwarp();
            double a[kNB];
#pragma unroll
            for (int c = 0; c < kNB; ++c) a[c] = (lane < nbn && c <= lane) ? scr[lane * 33 + c] : ((c == lane) ? 1.0 : 0.0);
            __syncwarp();                                        // every lane has its row: scr becomes the column store
            const double my_inv = factor_block(a, scr);
            if (!pro) asm volatile("bar.sync 2, 64;\n" ::: "memory");      // warp 1 is done reading LdT / invd
#pragma unroll
            for (int c = 0; c < kNB; ++c) LdT[c * 32 + lane] = scr[c * 32 + lane];
            invd[lane] = my_inv;
            }
        } else if (pro) {
            // prologue: nothing to do for the other warps
        } else if (wid == 1) {
            // ---- inverse of the diagonal block, column `lane`: L x = e_lane, right-looking.  Every CTA needs it
            //      (B operand of its panel GEMM); CTA 0 also keeps it in global memory for the back-substitution
            double r[kNB];
#pragma unroll
            for (int i = 0; i < kNB; ++i) r[i] = (i == lane) ? 1.0 : 0.0;
#pragma unroll
            for (int i = 0; i < kNB; ++i) {
                const double xi = r[i] * invd[i];
                r[i] = xi;
#pragma unroll
                for (int i2 = i + 1; i2 < kNB; ++i2) r[i2] = fma(-LdT[i * 32 + i2], xi, r[i2]);
            }
#pragma unroll
            for (int i = 0; i < kNB; ++i) IL[i * kPP + lane] = r[i];
            asm volatile("bar.arrive 4, 384;\n" ::: "memory");      // IL is ready (the 11 worker warps wait on 4)
            if (rank == 0) {
#pragma unroll
                for (int i = 0; i < kNB; ++i) invL[((size_t)blk * kNB + i) * kNB + lane] = r[i];
            }
            // LdT / invd may be overwritten by the look-ahead from here on (warp 0 waits on barrier 2)
            if (rem > 0) asm volatile("bar.arrive 2, 64;\n" ::: "memory");
        } else {
            if (worker) {
                // ---- panel rows 32.. : X = A21 invL11' as a GEMM on the FP64 tensor cores, 8 rows x 32 columns per warp
                //      and pass, in place.  invL11' is upper triangular: column tile jt needs k < 8 (jt + 1) only,
                //      20 DMMAs per 8 rows; the 20 B fragments (invL) stay in registers for the whole step.
                asm volatile("bar.sync 4, 384;\n" ::: "memory");     // IL written by warp 1
                double bfr[4][8];   // [jt][k4 / 4], used for k4 / 4 < 2 (jt + 1)
#pragma unroll
                for (int jt = 0; jt < 4; ++jt)
#pragma unroll
                    for (int ks = 0; ks < 8; ++ks)
                        bfr[jt][ks] = (ks < 2 * (jt + 1)) ? IL[(8 * jt + g) * kPP + 4 * ks + q] : 0.0;
                const int ntile = (prow - 32 + 7) / 8;
                for (int t = wk; t < ntile; t += nw) {
                    const int r0 = 32 + 8 * t;
                    const double* arow = P + (size_t)min(r0 + g, prow - 1) * kPP + q;
                    double af[8];
#pragma unroll
                    for (int ks = 0; ks < 8; ++ks) af[ks] = arow[4 * ks];
                    __syncwarp();                                    // all fragments read before the rows are overwritten
                    double d[4][2];
#pragma unroll
                    for (int jt = 0; jt < 4; ++jt) {
                        d[jt][0] = 0.0; d[jt][1] = 0.0;
#pragma unroll
                        for (int ks = 0; ks < 2 * (jt + 1); ++ks) dmma_m8n8k4(d[jt][0], d[jt][1], af[ks], bfr[jt][ks]);
                    }
                    if (r0 + g < prow) {
#pragma unroll
                        for (int jt = 0; jt < 4; ++jt)
                            *reinterpret_cast<double2*>(P + (size_t)(r0 + g) * kPP + 8 * jt + 2 * q) = make_double2(d[jt][0], d[jt][1]);
                    }
                }
            }
            if (rem > 0) asm volatile("bar.sync 3, 480;\n" ::: "memory");   // whole panel solved (warps 0, 2..15)
            if (rem > 0 && worker) {
                // ---- the solved panel goes back to global memory (it is L, needed by the back-substitution): rows dealt
                //      round-robin to the worker warps of all CTAs (every CTA holds the whole panel), 256 B per instruction
                for (int r = rank * nw + wk; r < prow; r += ncta * nw)
                    if (lane < nb) A[(size_t)(kb + nb + r) * n + kb + lane] = P[r * kPP + lane];
                // ---- trailing update: rows < prow (rhs included), columns < rem, lower triangle only.
                //      A[i][k] = P[r0 + i][k], B[k][j] = P[c0 + j][k]: per k-step of 4 a warp reads 6 fragments for
                //      8 DMMAs (2048 multiply-adds).  Row indices beyond the panel are clamped (their products are
                //      never stored).
                const int nmr = (prow + 15) / 16, nmc = (rem + 31) / 32;
                // macro-tiles that touch the lower triangle: row-block mi holds min(nmc, (16 mi + 15) / 32 + 1) of them;
                // they are numbered consecutively and dealt round-robin to the warps of the cluster (balanced)
                int total_tiles = 0;
                for (int mi = 0; mi < nmr; ++mi) total_tiles += min(nmc, (16 * mi + 15) / 32 + 1);
                for (int w = rank * nw + wk; w < total_tiles; w += ncta * nw) {
                    int mi = 0, base = 0;
                    for (;; ++mi) { const int cnt = min(nmc, (16 * mi + 15) / 32 + 1); if (w < base + cnt) break; base += cnt; }
                    const int mj = w - base;
                    const int R0 = mi * 16, C0 = mj * 32;
                    double acc[2][4][2];
#pragma unroll
                    for (int ti = 0; ti < 2; ++ti)
#pragma unroll
                        for (int tj = 0; tj < 4; ++tj)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int rr = R0 + 8 * ti + g, cc = C0 + 8 * tj + 2 * q + e;
                                const bool mine = rr < prow && cc < rem && cc <= rr && !(rr < nbn);   // rows < nbn: next diagonal block (warp 0)
                                acc[ti][tj][e] = mine ? A[(size_t)(kb + nb + rr) * n + kb + nb + cc] : 0.0;
                            }
                    const double* pa0 = P + (size_t)min(R0 + g, prow - 1) * kPP + q;
                    const double* pa1 = P + (size_t)min(R0 + 8 + g, prow - 1) * kPP + q;
                    const double* pb[4];
#pragma unroll
                    for (int tj = 0; tj < 4; ++tj) pb[tj] = P + (size_t)min(C0 + 8 * tj + g, prow - 1) * kPP + q;
#pragma unroll 2
                    for (int k4 = 0; k4 < kNB; k4 += 4) {
                        const double af0 = -pa0[k4], af1 = -pa1[k4];
                        double bf[4];
#pragma unroll
                        for (int tj = 0; tj < 4; ++tj) bf[tj] = pb[tj][k4];
#pragma unroll
                        for (int tj = 0; tj < 4; ++tj) {
                            dmma_m8n8k4(acc[0][tj][0], acc[0][tj][1], af0, bf[tj]);
                            dmma_m8n8k4(acc[1][tj][0], acc[1][tj][1], af1, bf[tj]);
                        }
                    }
#pragma unroll
                    for (int ti = 0; ti < 2; ++ti)
#pragma unroll
                        for (int tj = 0; tj < 4; ++tj)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int rr = R0 + 8 * ti + g, cc = C0 + 8 * tj + 2 * q + e;
                                const bool mine = rr < prow && cc < rem && cc <= rr && !(rr < nbn);
                                if (mine) A[(size_t)(kb + nb + rr) * n + kb + nb + cc] = acc[ti][tj][e];
                            }
                }
            }
        }
        if (rem == 0) break;
        if (pro) continue;
        cluster_sync_all();   // the trailing matrix (global) is complete and visible to every CTA
    }
    __syncthreads();
    if (s_fail) { if (tid == 0 && rank == 0) *fail = 1; return; }
    if (rank != 0) return;   // no cluster barrier below this point

    // ---- y = row n of A; back-substitution L' x = y, right-looking from the last block:
    //      x_blk = invL_blk' y_blk ;  y_i -= sum_j L[kb + j][i] x_j  for i < kb.
    //      The 32 rows of a block and its inverse are staged in shared memory by cp.async (the panel is
    //      free now); when a second buffer fits (dbuf), block blk-1 is in flight while block blk is applied.
    for (int i = tid; i < n; i += kCholThreads) vec[i] = A[(size_t)n * n + i];
    const int bp = chol_back_pitch(n);
    double* const R0buf = P;
    double* const L1buf = P + 32 * (size_t)bp;
    double* const R1buf = L1buf + 32 * 33;
    double* const red = scr;
    auto stage = [&](int b, int which) {
        const int kb = b * kNB;
        const int nb = min(kNB, n - kb);
        double* Ldst = which ? L1buf : LdT;
        double* Rdst = which ? R1buf : R0buf;
        for (int i = tid; i < kNB * kNB; i += kCholThreads) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(Ldst + (i >> 5) * 33 + (i & 31));
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(dst), "l"(invL + (size_t)b * kNB * kNB + i));
        }
        // row starts are 16 B aligned (n = 6 x keyframes is even, kb is a multiple of 32): 16-byte copies, L2 only
        for (int j = wid; j < nb; j += kCholThreads / 32)
            for (int c = 2 * lane; c < kb; c += 64) {
                const unsigned dst = (unsigned)__cvta_generic_to_shared(Rdst + j * bp + c);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(dst), "l"(A + (size_t)(kb + j) * n + c));
            }
        asm volatile("cp.async.commit_group;\n" ::);
    };
    __syncthreads();   // LdT / panel are free
    stage(nblk - 1, 0);
    for (int blk = nblk - 1; blk >= 0; --blk) {
        const int kb = blk * kNB;
        const int nb = min(kNB, n - kb);
        const int cur = dbuf ? ((nblk - 1 - blk) & 1) : 0;
        if (dbuf && blk > 0) {
            stage(blk - 1, cur ^ 1);
            asm volatile("cp.async.wait_group 1;\n" ::);
        } else {
            asm volatile("cp.async.wait_group 0;\n" ::);
        }
        __syncthreads();
        const double* Lc = cur ? L1buf : LdT;
        const double* rows = cur ? R1buf : R0buf;
        if (wid == 0) {
            const double t = (lane < nb) ? vec[kb + lane] : 0.0;
            double acc0 = 0, acc1 = 0;
#pragma unroll
            for (int j = 0; j < kNB; j += 2) {
                acc0 = fma(Lc[j * 33 + lane], __shfl_sync(0xffffffffu, t, j), acc0);         // invL is lower triangular
                acc1 = fma(Lc[(j + 1) * 33 + lane], __shfl_sync(0xffffffffu, t, j + 1), acc1);
            }
            red[lane] = acc0 + acc1;
            if (lane < nb) vec[kb + lane] = acc0 + acc1;
        }
        __syncthreads();
        for (int i = tid; i < kb; i += kCholThreads) {
            double s0 = 0, s1 = 0;
#pragma unroll 8
            for (int j = 0; j < kNB; j += 2) {
                if (j < nb) s0 = fma(rows[j * bp + i], red[j], s0);
                if (j + 1 < nb) s1 = fma(rows[(j + 1) * bp + i], red[j + 1], s1);
            }
            vec[i] -= s0 + s1;
        }
        __syncthreads();
        if (!dbuf && blk > 0) stage(blk - 1, 0);
    }
    for (int i = tid; i < n; i += kCholThreads) x[i] = vec[i];
}

// ---- Reduced systems too large for the shared-memory panel of k_ba_cholesky_solve (n > kMaxReducedDim, i.e. more than
// 114 free keyframes): the same blocked algorithm -- rhs as an extra row, 32-wide blocks, block inverse, DMMA trailing
// update -- with the panel left in global memory (L2) and one launch per phase of a block step.  A fallback for
// unusually large local maps: simple and correct, not tuned.  grid.y / blockIdx.y = speculative trial.
__global__ void __launch_bounds__(64) k_chol_big_diag(const LmCtl* __restrict__ ctl, double* __restrict__ A, size_t A_stride, int n, int kb, int nb,
                                                      double* __restrict__ invL, size_t invL_stride, int* __restrict__ fail) {
    if ((int)blockIdx.y >= ctl->nbatch) return;
    A += (size_t)blockIdx.y * A_stride; invL += (size_t)blockIdx.y * invL_stride + (size_t)(kb / kNB) * kNB * kNB; fail += blockIdx.y;
    __shared__ double cs[kNB * kNB];     // cs[c * 32 + r] = L[r][c]
    __shared__ double sinv[kNB];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (wid == 0) {
        double a[kNB];
#pragma unroll
        for (int c = 0; c < kNB; ++c) {
            double v = (c == lane) ? 1.0 : 0.0;
            if (lane < nb && c <= lane) v = A[(size_t)(kb + lane) * n + kb + c];
            a[c] = v;
        }
        bool bad = false;
        double my_inv = 1.0;
        double ajj = __shfl_sync(0xffffffffu, a[0], 0);
        double inv = rsqrt(ajj);
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
            bad = bad || !(ajj > 0.0) || !isfinite(ajj);
            const double l = (lane >= j) ? a[j] * inv : 0.0;
            if (lane == j) my_inv = inv;
            cs[j * 32 + lane] = l;
            if (lane < nb && j <= lane && j < nb) A[(size_t)(kb + lane) * n + kb + j] = l;
            if (j + 1 < kNB) {
                ajj = __shfl_sync(0xffffffffu, fma(-l, l, a[j + 1]), j + 1);
                inv = rsqrt(ajj);
            }
            __syncwarp();
#pragma unroll
            for (int c = j + 1; c < kNB; ++c) a[c] = fma(-l, cs[j * 32 + c], a[c]);
        }
        if (bad && lane == 0) *fail = 1;
        sinv[lane] = my_inv;
    }
    __syncthreads();
    if (wid == 1) {
        // inverse of the block, column `lane`
        double r[kNB];
#pragma unroll
        for (int i = 0; i < kNB; ++i) r[i] = (i == lane) ? 1.0 : 0.0;
#pragma unroll
        for (int i = 0; i < kNB; ++i) {
            const double xi = r[i] * sinv[i];
            r[i] = xi;
#pragma unroll
            for (int i2 = i + 1; i2 < kNB; ++i2) r[i2] = fma(-cs[i * 32 + i2], xi, r[i2]);
        }
#pragma unroll
        for (int i = 0; i < kNB; ++i) invL[i * kNB + lane] = r[i];
    }
}

// panel rows (and the rhs row) below the block: X = A21 invL11', one row per thread
__global__ void __launch_bounds__(128) k_chol_big_panel(const LmCtl* __restrict__ ctl, double* __restrict__ A, size_t A_stride, int n, int kb, int nb,
                                                        const double* __restrict__ invL, size_t invL_stride) {
    if ((int)blockIdx.y >= ctl->nbatch) return;
    A += (size_t)blockIdx.y * A_stride; invL += (size_t)blockIdx.y * invL_stride + (size_t)(kb / kNB) * kNB * kNB;
    __shared__ double IL[kNB][kNB + 1];
    for (int i = threadIdx.x; i < kNB * kNB; i += 128) IL[i >> 5][i & 31] = invL[i];
    __syncthreads();
    const int prow = n - kb - nb + 1;
    const int r = blockIdx.x * 128 + threadIdx.x;
    if (r >= prow) return;
    double* row = A + (size_t)(kb + nb + r) * n + kb;
    double xr[kNB];
#pragma unroll
    for (int c = 0; c < kNB; ++c) xr[c] = (c < nb) ? row[c] : 0.0;
#pragma unroll
    for (int j = 0; j < kNB; ++j) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k <= j; ++k) acc = fma(xr[k], IL[j][k], acc);
        if (j < nb) row[j] = acc;
    }
}

// trailing update A22 -= L21 L21' (rhs row included), one warp per 16 x 32 macro-tile, fragments read from global memory
__global__ void __launch_bounds__(128) k_chol_big_trailing(const LmCtl* __restrict__ ctl, double* __restrict__ A, size_t A_stride, int n, int kb, int nb) {
    if ((int)blockIdx.y >= ctl->nbatch) return;
    A += (size_t)blockIdx.y * A_stride;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int rem = n - kb - nb, prow = rem + 1;
    const int nmr = (prow + 15) / 16, nmc = (rem + 31) / 32;
    const int w = blockIdx.x * 4 + wid;
    int mi = 0, base = 0;
    for (;; ++mi) {
        if (mi >= nmr) return;
        const int cnt = min(nmc, (16 * mi + 15) / 32 + 1);
        if (w < base + cnt) break;
        base += cnt;
    }
    const int mj = w - base;
    const int R0 = mi * 16, C0 = mj * 32;
    const double* P = A + (size_t)(kb + nb) * n + kb;      // solved panel: P[r * n + k]
    double* T = A + (size_t)(kb + nb) * n + kb + nb;        // trailing matrix: T[r * n + c]
    double acc[2][4][2];
#pragma unroll
    for (int ti = 0; ti < 2; ++ti)
#pragma unroll
        for (int tj = 0; tj < 4; ++tj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int rr = R0 + 8 * ti + g, cc = C0 + 8 * tj + 2 * q + e;
                acc[ti][tj][e] = (rr < prow && cc < rem && cc <= rr) ? T[(size_t)rr * n + cc] : 0.0;
            }
    const double* pa0 = P + (size_t)min(R0 + g, prow - 1) * n;
    const double* pa1 = P + (size_t)min(R0 + 8 + g, prow - 1) * n;
    const double* pb[4];
#pragma unroll
    for (int tj = 0; tj < 4; ++tj) pb[tj] = P + (size_t)min(C0 + 8 * tj + g, prow - 1) * n;
#pragma unroll 2
    for (int k4 = 0; k4 < kNB; k4 += 4) {
        const bool kin = k4 + q < nb;
        const double af0 = kin ? -pa0[k4 + q] : 0.0, af1 = kin ? -pa1[k4 + q] : 0.0;
        double bf[4];
#pragma unroll
        for (int tj = 0; tj < 4; ++tj) bf[tj] = kin ? pb[tj][k4 + q] : 0.0;
#pragma unroll
        for (int tj = 0; tj < 4; ++tj) {
            dmma_m8n8k4(acc[0][tj][0], acc[0][tj][1], af0, bf[tj]);
            dmma_m8n8k4(acc[1][tj][0], acc[1][tj][1], af1, bf[tj]);
        }
    }
#pragma unroll
    for (int ti = 0; ti < 2; ++ti)
#pragma unroll
        for (int tj = 0; tj < 4; ++tj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int rr = R0 + 8 * ti + g, cc = C0 + 8 * tj + 2 * q + e;
                if (rr < prow && cc < rem && cc <= rr) T[(size_t)rr * n + cc] = acc[ti][tj][e];
            }
}

// y = row n of A (L^-1 b after the factorisation); L' x = y by blocks from the last one, one CTA per trial
__global__ void __launch_bounds__(512) k_chol_big_backsolve(const LmCtl* __restrict__ ctl, const double* __restrict__ A, size_t A_stride, int n, const double* __restrict__ invL,
                                                            size_t invL_stride, double* __restrict__ x, int* __restrict__ fail) {
    if ((int)blockIdx.x >= ctl->nbatch) return;
    A += (size_t)blockIdx.x * A_stride; invL += (size_t)blockIdx.x * invL_stride; x += (size_t)blockIdx.x * n; fail += blockIdx.x;
    extern __shared__ __align__(16) double sh[];
    double* vec = sh;                         // n
    double* IL = sh + ((n + 31) / 32) * 32;   // 32 x 33
    double* red = IL + 32 * 33;               // 32
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < n; i += 512) vec[i] = A[(size_t)n * n + i];
    const int nblk = (n + kNB - 1) / kNB;
    for (int blk = nblk - 1; blk >= 0; --blk) {
        const int kb = blk * kNB, nb = min(kNB, n - kb);
        __syncthreads();
        for (int i = tid; i < kNB * kNB; i += 512) IL[(i >> 5) * 33 + (i & 31)] = invL[(size_t)blk * kNB * kNB + i];
        __syncthreads();
        if (wid == 0) {
            const double t = (lane < nb) ? vec[kb + lane] : 0.0;
            double a0 = 0, a1 = 0;
#pragma unroll
            for (int j = 0; j < kNB; j += 2) {
                a0 = fma(IL[j * 33 + lane], __shfl_sync(0xffffffffu, t, j), a0);
                a1 = fma(IL[(j + 1) * 33 + lane], __shfl_sync(0xffffffffu, t, j + 1), a1);
            }
            red[lane] = a0 + a1;
            if (lane < nb) vec[kb + lane] = a0 + a1;
        }
        __syncthreads();
        for (int i = tid; i < kb; i += 512) {
            double s0 = 0, s1 = 0;
            for (int j = 0; j + 1 < nb; j += 2) {
                s0 = fma(A[(size_t)(kb + j) * n + i], red[j], s0);
                s1 = fma(A[(size_t)(kb + j + 1) * n + i], red[j + 1], s1);
            }
            if (nb & 1) s0 = fma(A[(size_t)(kb + nb - 1) * n + i], red[nb - 1], s0);
            vec[i] -= s0 + s1;
        }
    }
    __syncthreads();
    if (*fail) return;
    for (int i = tid; i < n; i += 512) x[i] = vec[i];
}

// Landmarks: xl = Dinv (bl - sum Hpl' x_kf), candidate point; keyframes: candidate pose.
// Also the LM scale term sum x (lambda x + b), one partial per block and damping value.
// All damping values of the batch are handled by the same thread: the Jacobian blocks and the edge indices of a landmark
// are read once, only x, (Hll + lambda I)^-1 and the candidate slot differ.
template <int R>
__global__ void __launch_bounds__(128) k_ba_update(BaDev P, const LmCtl* __restrict__ ctl, const double* __restrict__ rec, const double* __restrict__ Hll,
                                                    const double* __restrict__ bl, const double* __restrict__ bp, const double* __restrict__ x,
                                                    double* poses_ring, double* points_ring,
                                                    double* __restrict__ partial_scale, int* __restrict__ fail) {
    __shared__ double sm[36];
    const int nbatch = ctl->nbatch;
    if (nbatch == 0) return;
    double lambda[kSpec]; int buf[kSpec];
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) { lambda[bt] = ctl->lam[bt]; buf[bt] = ctl->buf[bt]; }
    P.poses = P.poses_ring + (size_t)ctl->cur * 12 * P.K; P.points = P.points_ring + (size_t)ctl->cur * 3 * P.L;
    const int t = blockIdx.x * 128 + threadIdx.x;
    double sc[kSpec];
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) sc[bt] = 0;
    if (t < P.L) {
        const int l = t;
        const double b0 = bl[3 * (size_t)l], b1 = bl[3 * (size_t)l + 1], b2 = bl[3 * (size_t)l + 2];
        double r[kSpec][3];
#pragma unroll
        for (int bt = 0; bt < kSpec; ++bt) { r[bt][0] = b0; r[bt][1] = b1; r[bt][2] = b2; }
        for (int p = P.lm_first[l]; p < P.lm_first[l + 1]; ++p) {
            const int fi = P.free_idx[P.obs_kf[p]];
            if (P.level[p] || fi < 0) continue;
            using ER = EdgeRec<R>;
            double W[18], er[2 * ER::kHpl2];
            const double2* pw = reinterpret_cast<const double2*>(rec + ER::kSize * (size_t)p);
#pragma unroll
            for (int k = 0; k < ER::kHpl2; ++k) { const double2 v = pw[k]; er[2 * k] = v.x; er[2 * k + 1] = v.y; }
            ovs::edge_hpl<R>(er, er + ER::kJl, er[ER::kWw], edge_dim<R>(P, p), W);
#pragma unroll
            for (int bt = 0; bt < kSpec; ++bt) {
                if (bt < nbatch) {
                    const double* xb = x + (size_t)bt * P.n + 6 * fi;
#pragma unroll
                    for (int a = 0; a < 6; ++a) {
                        const double xa = xb[a];
                        r[bt][0] -= W[3 * a] * xa; r[bt][1] -= W[3 * a + 1] * xa; r[bt][2] -= W[3 * a + 2] * xa;
                    }
                }
            }
        }
        const double p0 = P.points[3 * (size_t)l], p1 = P.points[3 * (size_t)l + 1], p2 = P.points[3 * (size_t)l + 2];
#pragma unroll
        for (int bt = 0; bt < kSpec; ++bt) {
            if (bt < nbatch) {
                const double D[6] = {Hll[6 * (size_t)l] + lambda[bt], Hll[6 * (size_t)l + 1], Hll[6 * (size_t)l + 2], Hll[6 * (size_t)l + 3] + lambda[bt],
                                     Hll[6 * (size_t)l + 4], Hll[6 * (size_t)l + 5] + lambda[bt]};
                double Di[6];
                if (!ovs::inv3_sym(D, Di)) {       // singular landmark block: the trial counts as failed (g2o: solver returns false)
                    fail[bt] = 1;
#pragma unroll
                    for (int q = 0; q < 6; ++q) Di[q] = 0.0;
                }
                const double d0 = Di[0] * r[bt][0] + Di[1] * r[bt][1] + Di[2] * r[bt][2];
                const double d1 = Di[1] * r[bt][0] + Di[3] * r[bt][1] + Di[4] * r[bt][2];
                const double d2 = Di[2] * r[bt][0] + Di[4] * r[bt][1] + Di[5] * r[bt][2];
                double* cand_points = points_ring + (size_t)buf[bt] * 3 * P.L;
                cand_points[3 * (size_t)l] = p0 + d0;
                cand_points[3 * (size_t)l + 1] = p1 + d1;
                cand_points[3 * (size_t)l + 2] = p2 + d2;
                sc[bt] = d0 * (lambda[bt] * d0 + b0) + d1 * (lambda[bt] * d1 + b1) + d2 * (lambda[bt] * d2 + b2);
            }
        }
    } else if (t < P.L + P.K) {
        const int k = t - P.L;
        const int fi = P.free_idx[k];
        double pose[12];
#pragma unroll
        for (int j = 0; j < 12; ++j) pose[j] = P.poses[12 * (size_t)k + j];
#pragma unroll
        for (int bt = 0; bt < kSpec; ++bt) {
            if (bt < nbatch) {
            double out[12];
            if (fi >= 0) {
                double u[6];
#pragma unroll
                for (int j = 0; j < 6; ++j) { u[j] = x[(size_t)bt * P.n + 6 * fi + j]; sc[bt] += u[j] * (lambda[bt] * u[j] + bp[6 * (size_t)fi + j]); }
                ovs::pose_oplus(pose, u, out);
            } else {
#pragma unroll
                for (int j = 0; j < 12; ++j) out[j] = pose[j];
            }
            double* cand_poses = poses_ring + (size_t)buf[bt] * 12 * P.K;
#pragma unroll
            for (int j = 0; j < 12; ++j) cand_poses[12 * (size_t)k + j] = out[j];
            }
        }
    }
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) {
        if (bt < nbatch) {          // block-uniform
            const double tot = block_sum(sc[bt], sm);
            if (threadIdx.x == 0) partial_scale[(size_t)bt * gridDim.x + blockIdx.x] = tot;
        }
    }
}

// at_current != 0: computeActiveErrors at the current estimate (start of an optimize()), errors to slot 0.
__global__ void __launch_bounds__(128) k_ba_errors(BaDev P, const LmCtl* __restrict__ ctl, int at_current,
                                                    double* __restrict__ err, double* __restrict__ partial_chi) {
    __shared__ double sm[36];
    int slot;
    if (at_current) {
        if (!ctl->active) return;
        slot = ctl->cur;
    } else {
        if ((int)blockIdx.y >= ctl->nbatch) return;
        slot = ctl->buf[blockIdx.y];
    }
    P.use_huber = ctl->use_huber;
    P.poses = P.poses_ring + (size_t)slot * 12 * P.K;
    P.points = P.points_ring + (size_t)slot * 3 * P.L;
    err += (size_t)blockIdx.y * 3 * P.M; partial_chi += (size_t)blockIdx.y * gridDim.x;
    const int i = blockIdx.x * 128 + threadIdx.x;
    double c = 0;
    if (i < P.M && !P.level[i]) {
        const int kf = P.obs_kf[i];
        const float xr = P.obs_xr ? P.obs_xr[i] : -1.0f;
        const bool stereo = xr >= 0.0f;
        const float2 xy = P.obs_xy[i];
        const double obs[3] = {(double)xy.x, (double)xy.y, (double)xr};
        double pose[12], pw[3], e[3] = {0, 0, 0};
#pragma unroll
        for (int k = 0; k < 12; ++k) pose[k] = P.poses[12 * (size_t)kf + k];
        const size_t pi = P.obs_lm ? (size_t)P.obs_lm[i] : (size_t)i;
#pragma unroll
        for (int k = 0; k < 3; ++k) pw[k] = P.points[3 * pi + k];
        ovs::edge_eval(P.cam, pose, pw, obs, stereo, e, nullptr, nullptr);
        err[3 * (size_t)i] = e[0]; err[3 * (size_t)i + 1] = e[1]; err[3 * (size_t)i + 2] = stereo ? e[2] : 0.0;
        const double w = (double)P.inv_sigma_sq[i];
        double chi = w * (e[0] * e[0] + e[1] * e[1]);
        if (stereo) chi += w * e[2] * e[2];
        c = chi;
        if (P.use_huber) { double r1; ovs::huber(chi, P.delta, &c, &r1); }
    }
    const double tot = block_sum(c, sm);
    if (threadIdx.x == 0) partial_chi[blockIdx.x] = tot;
}

// what the host needs to know when it does look: [0] nbatch, [1] active, [3] need_more, [4] iterations completed
// ([2] is the stop word, written by the host)
__device__ __forceinline__ void mirror_state(const LmCtl& c, volatile int* mirror) {
    if (!mirror) return;
    mirror[0] = c.nbatch; mirror[1] = c.active; mirror[3] = c.need_more; mirror[4] = c.it;   // read by the host after a stream synchronisation
}

// Final sums of a trial batch and the Levenberg decision, on the device.
// One block of kSpec x 256 threads: group t = threadIdx.x / 256 sums the partials of trial t deterministically (thread-
// strided partial sums, butterfly per warp, the 8 warp sums in order); thread 0 then walks the trials exactly as g2o's
//   do { solve; rho = (currentChi - tempChi) / scale; accept or lambda *= ni, ni *= 2 } while (rho < 0 && qmax < 10 && !terminate)
// would have produced them, and leaves in *ctl either the next batch of damping values (all trials rejected so far) or
// nbatch = 0 and the bookkeeping of the finished iteration.
// mode 0: robust chi2 at the current estimate (computeActiveErrors at the start of optimize()) -> currentChi.
__global__ void __launch_bounds__(kSpec * 256) k_ba_reduce(LmCtl* ctl, int mode, const double* __restrict__ partial_chi, int nchi,
                                                           const double* __restrict__ partial_scale, int nscale, int* fail,
                                                           const volatile int* stop_word, int batch_index, int* exec_log, volatile int* mirror,
                                                           int halt_if_undecided, int next_width_cap) {
    __shared__ double sm[kSpec][2][8];
    const int nb = mode == 0 ? (ctl->active ? 1 : 0) : ctl->nbatch;
    if (nb == 0) {
        if (threadIdx.x == 0 && mode == 1 && exec_log && batch_index >= 0) exec_log[batch_index] = 0;
        return;
    }
    const int t = threadIdx.x >> 8, tl = threadIdx.x & 255, lane = tl & 31, w = tl >> 5;
    double a = 0, b = 0;
    if (t < nb) {
        const double* pc = partial_chi + (size_t)t * nchi;
        for (int i = tl; i < nchi; i += 256) a += pc[i];
        if (mode == 1) {
            const double* ps = partial_scale + (size_t)t * nscale;
            for (int i = tl; i < nscale; i += 256) b += ps[i];
        }
    }
    a = warp_sum(a); b = warp_sum(b);
    if (lane == 0) { sm[t][0][w] = a; sm[t][1][w] = b; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    double chi[kSpec], sc[kSpec];
    for (int k = 0; k < nb; ++k) {
        double x = 0, y = 0;
        for (int j = 0; j < 8; ++j) { x += sm[k][0][j]; y += sm[k][1][j]; }
        chi[k] = x; sc[k] = y;
    }
    if (mode == 0) { ctl->currentChi = chi[0]; ctl->err_slot = 0; return; }
    // the control block is read and written back as a whole (a handful of wide transactions instead of a chain of dependent
    // scalar round trips to L2: this thread is the critical path between two trial batches)
    LmCtl c = *ctl;
    const bool stop = stop_word && *stop_word != 0;
    double lambda = c.lambda, ni = c.ni, currentChi = c.currentChi, rho = c.rho;
    int qmax = c.qmax, cur = c.cur, es = c.err_slot, ntr = c.num_trials;
    bool done = false;
#pragma unroll
    for (int k = 0; k < kSpec; ++k) {
        if (k < nb && !done) {
            const bool ok2 = fail[k] == 0;
            const double tempChi = ok2 ? chi[k] : DBL_MAX;
            rho = currentChi - tempChi;
            double scale = ok2 ? sc[k] : 0.0;
            scale += 1e-3;
            rho /= scale;
            es = k;                                                 // edge->_error as of this trial
            ++qmax; ++ntr;
            if (rho > 0 && isfinite(tempChi)) {
                double alpha = 1. - pow(2 * rho - 1, 3.0);
                alpha = fmin(alpha, 2. / 3.);
                lambda = c.lam[k] * fmax(1. / 3., alpha);
                ni = 2;
                currentChi = tempChi;
                cur = c.buf[k];                                     // discardTop: the candidate becomes the estimate
                done = true;
            } else {
                lambda = c.lam[k] * c.ni_after[k];                  // pop: candidate dropped
                ni = c.ni_after[k] * 2;
                if (!(rho < 0) || qmax >= kMaxTrials || stop) done = true;
            }
        }
    }
    c.lambda = lambda; c.ni = ni; c.currentChi = currentChi; c.rho = rho;
    c.qmax = qmax; c.cur = cur; c.err_slot = es; c.num_trials = ntr;
    c.batches += 1; c.solver_trials += nb;
    if (exec_log && batch_index >= 0) exec_log[batch_index] = nb;
#pragma unroll
    for (int k = 0; k < kSpec; ++k) fail[k] = 0;
    if (done) {
        c.nbatch = 0;
        c.last_chi2 = currentChi; c.last_lambda = lambda;
        const int it = c.it + 1;
        c.it = it;
        if (qmax == kMaxTrials || rho == 0 || it >= c.iterations) c.active = 0;
        if (stop) { c.active = 0; c.stopped = 1; }
    } else {
        int nn = min(kSpec, kMaxTrials - qmax);
        if (next_width_cap > 0) nn = min(nn, next_width_cap);     // a statically enqueued follow-up batch of that width comes next
        double l = lambda, n2 = ni;
#pragma unroll
        for (int k = 0; k < kSpec; ++k)
            if (k < nn) { c.lam[k] = l; c.buf[k] = (cur + 1 + k) % (kSpec + 1); l *= n2; c.ni_after[k] = n2; n2 *= 2; }
        if (halt_if_undecided) {
            // no further batch of this iteration is enqueued: park the batch and halt until the host has enqueued it
            c.pending_nbatch = nn; c.nbatch = 0; c.active = 0; c.need_more = 1;
        } else {
            c.nbatch = nn;
        }
    }
    *ctl = c;
    mirror_state(c, mirror);
}

// the host has enqueued the parked trial batch behind this kernel
__global__ void k_lm_resume(LmCtl* ctl, volatile int* mirror) {
    LmCtl c = *ctl;
    if (!c.need_more) return;
    c.nbatch = c.pending_nbatch; c.pending_nbatch = 0; c.active = 1; c.need_more = 0;
    *ctl = c;
    mirror_state(c, mirror);
}

// ---- one-thread control kernels of the device-side Levenberg loop
__global__ void k_lm_init(LmCtl* ctl, int spec_width, int* fail, volatile int* mirror) {
    LmCtl c;
    memset(&c, 0, sizeof(c));
    c.ni = 2; c.spec_width = spec_width;
    *ctl = c;
    for (int k = 0; k < kSpec; ++k) fail[k] = 0;
    mirror_state(c, mirror);
}

// start of SparseOptimizer::optimize(iterations): all of g2o's per-call state is reset
__global__ void k_lm_round_begin(LmCtl* ctl, int iterations, int use_huber, const volatile int* stop_word, double* maxdiag, volatile int* mirror) {
    LmCtl c = *ctl;
    if (stop_word && *stop_word != 0) c.stopped = 1;
    c.iterations = iterations; c.use_huber = use_huber;
    c.it = 0; c.qmax = 0; c.rho = 0; c.lambda = 0; c.ni = 2; c.nbatch = 0;
    c.round_live = c.stopped ? 0 : 1;
    c.active = (iterations > 0 && !c.stopped) ? 1 : 0;
    *ctl = c;
    maxdiag[0] = 0; maxdiag[1] = 0;
    mirror_state(c, mirror);
}

__global__ void k_lm_round_end(LmCtl* ctl, const volatile int* stop_word, volatile int* mirror) {
    LmCtl c = *ctl;
    if (c.round_live || c.num_rounds == 0) {
        const int r = c.num_rounds;
        if (r < 8) c.round_iterations[r] = c.it;
        c.num_iterations += c.it;
        c.num_rounds = r + 1;
    }
    c.active = 0; c.nbatch = 0;
    if (stop_word && *stop_word != 0) c.stopped = 1;
    *ctl = c;
    mirror_state(c, mirror);
}

// Start of a Levenberg iteration (one thread): the damping values and ring slots of its first trial batch.  lambda_init is
// g2o's computeLambdaInit, used on the first iteration of a round.
__device__ void lm_plan_iteration(LmCtl* ctl, double lambda_init, const volatile int* stop_word, int* fail, volatile int* mirror) {
    LmCtl c = *ctl;
    if (c.active && stop_word && *stop_word != 0) { c.active = 0; c.stopped = 1; }
    if (!c.active) {
        c.nbatch = 0;
    } else {
        if (c.it == 0) {
            c.lambda = lambda_init;
            c.ni = 2;
            if (c.num_rounds < 8) c.lambda_init[c.num_rounds] = c.lambda;
        }
        c.qmax = 0; c.rho = 0;
        const int nn = min(max(c.spec_width, 1), kSpec);
        double l = c.lambda, n2 = c.ni;
#pragma unroll
        for (int k = 0; k < kSpec; ++k)
            if (k < nn) { c.lam[k] = l; c.buf[k] = (c.cur + 1 + k) % (kSpec + 1); l *= n2; c.ni_after[k] = n2; n2 *= 2; }
        c.nbatch = nn;
    }
    *ctl = c;
#pragma unroll
    for (int k = 0; k < kSpec; ++k) fail[k] = 0;
    mirror_state(c, mirror);
}

__global__ void __launch_bounds__(1024) k_ba_pose_final_plan(LmCtl* ctl, int nfree, const int* __restrict__ kf_chunk_begin, const double* __restrict__ ppart,
                                                              double* __restrict__ Hpp, double* __restrict__ bp, double* maxdiag, int* fail,
                                                              const volatile int* stop_word, volatile int* mirror) {
    __shared__ double smax[32];
    const bool active = ctl->active != 0, halted = ctl->need_more != 0;
    double md = 0;
    if (active) {
        for (int o = threadIdx.x; o < 27 * nfree; o += 1024) {
            const int a = o / 27, t = o - 27 * a;
            double v = 0;
            const int c0 = kf_chunk_begin[a], c1 = kf_chunk_begin[a + 1];
#pragma unroll 4
            for (int c = c0; c < c1; ++c) v += ppart[27 * (size_t)c + t];     // same order of additions, four loads in flight
            if (t < 21) {
                Hpp[21 * (size_t)a + t] = v;
                if (t == 0 || t == 6 || t == 11 || t == 15 || t == 18 || t == 20) md = fmax(md, fabs(v));
            } else {
                bp[6 * (size_t)a + t - 21] = v;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, o));
    if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = md;
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (halted) return;             // halted: the parked batch and the Hessian of the undecided iteration must survive
    for (int w = 0; w < 32; ++w) md = fmax(md, smax[w]);
    md = fmax(md, maxdiag[0]);      // the landmark blocks' share (k_ba_linearize)
    maxdiag[0] = 0; maxdiag[1] = 0;
    lm_plan_iteration(ctl, 1e-5 * md, stop_word, fail, mirror);
}

// Outlier classification from the stored edge errors (edge->chi2()) and depth_is_positive().
// mode 0: set level = 1 where outlier (between the two BA rounds; not when the call was stopped); mode 1: write outlier_out.
__global__ void __launch_bounds__(128) k_ba_classify(BaDev P, const LmCtl* __restrict__ ctl, const double* __restrict__ err_slots, double chi2_2d, double chi2_3d, int mode,
                                                      unsigned char* __restrict__ level_out, unsigned char* __restrict__ outlier_out) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= P.M || (mode == 0 && ctl->stopped)) return;
    const double* err = err_slots + (size_t)ctl->err_slot * 3 * P.M;
    P.poses = P.poses_ring + (size_t)ctl->cur * 12 * P.K; P.points = P.points_ring + (size_t)ctl->cur * 3 * P.L;
    const bool stereo = P.obs_xr && P.obs_xr[i] >= 0.0f;
    const double w = (double)P.inv_sigma_sq[i];
    const double e0 = err[3 * (size_t)i], e1 = err[3 * (size_t)i + 1], e2 = err[3 * (size_t)i + 2];
    double chi = w * (e0 * e0 + e1 * e1);
    if (stereo) chi += w * e2 * e2;
    bool depth_pos = true;
    if (P.cam.model != ovs::kCamEquirectangular) {
        const double* ps = P.poses + 12 * (size_t)P.obs_kf[i];
        const double* pw = P.points + 3 * (size_t)P.obs_lm[i];
        depth_pos = (ps[6] * pw[0] + ps[7] * pw[1] + ps[8] * pw[2] + ps[11]) > 0;
    }
    const bool outlier = (stereo ? chi2_3d : chi2_2d) < chi || !depth_pos;
    if (mode == 0) { if (outlier) level_out[i] = 1; }
    else outlier_out[i] = outlier ? 1 : 0;
}

// Edges excluded from the second round keep their first-round error (g2o never touches them again): replicate the
// errors of the last evaluated trial into every speculative slot so that they survive whichever slot ends up current.
__global__ void __launch_bounds__(256) k_ba_replicate_err(const LmCtl* __restrict__ ctl, double* err_slots, size_t n3) {
    if (ctl->stopped) return;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n3) return;
    const int src = ctl->err_slot;
    const double v = err_slots[(size_t)src * n3 + i];
#pragma unroll
    for (int k = 0; k < kSpec; ++k)
        if (k != src) err_slots[(size_t)k * n3 + i] = v;
}

// ------------------------------------------------------------------ graph bookkeeping
// What the reference does while it builds its g2o graph -- vertex ids of the free keyframes, the edges of every landmark,
// input validation -- as three small kernels over the uploaded index arrays, so that prepare has no O(M) host loop.
// counts[0] = free keyframes, [1] = co-observation entries, [2] = edges on free keyframes, [3] = error code
// (1 index out of range, 2 observations not grouped by landmark), [4] = first offending observation.
__global__ void __launch_bounds__(1024) k_ba_free_index(int K, const unsigned char* __restrict__ fixed, int* __restrict__ free_idx, long long* counts) {
    __shared__ int wsum[32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < K; base += 1024) {
        const int i = base + tid;
        const int c = (i < K && !fixed[i]) ? 1 : 0;
        int v = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
        if (lane == 31) wsum[wid] = v;
        __syncthreads();
        if (wid == 0) {
            int ws = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += u; }
            wsum[lane] = ws;
        }
        __syncthreads();
        const int excl = carry + (wid ? wsum[wid - 1] : 0) + v - c;
        if (i < K) free_idx[i] = c ? excl : -1;
        __syncthreads();
        if (tid == 1023) carry = excl + c;
        __syncthreads();
    }
    if (tid == 0) counts[0] = carry;
}

__global__ void __launch_bounds__(256) k_ba_landmark_index(int M, int L, int K, const int* __restrict__ obs_kf, const int* __restrict__ obs_lm,
                                                            const float* __restrict__ obs_xr, int* __restrict__ lm_first, long long* counts) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= M) return;
    if (obs_xr[i] >= 0.0f) counts[5] = 1;          // a stereo edge: the edge records have 3 rows
    const int l = obs_lm[i], k = obs_kf[i];
    int err = 0;
    if (l < 0 || l >= L || k < 0 || k >= K) err = 1;
    const int lp = i > 0 ? obs_lm[i - 1] : -1;
    if (!err && i > 0 && l < lp) err = 2;
    if (err) {
        // the FIRST offending observation is reported (64-bit min over (index << 2 | code))
        atomicMin(reinterpret_cast<unsigned long long*>(counts + 4), ((unsigned long long)i << 2) | (unsigned)err);
        return;
    }
    if (i == 0 || (lp >= -1 && lp < L && l != lp))
        for (int q = max(lp, -1) + 1; q <= l; ++q) lm_first[q] = i;      // landmarks without observations start where the next one does
    if (i == M - 1)
        for (int q = l + 1; q <= L; ++q) lm_first[q] = M;
}

// Landmark block table of k_ba_linearize: consecutive landmarks with at most 128 edges in all; a landmark with more than 128 edges
// gets a block of its own.  Entry = {first landmark, end landmark, first edge, end edge}.  The landmarks are split into segments
// by where their edges start (segment k: lm_first in [kLbSegEdges k, kLbSegEdges (k + 1))), and each segment is cut greedily in
// landmark order by one CTA, independently of the others; its entries go to blocks[k * kLbSegCap ..], their number to nblocks[k].
// Two consecutive blocks hold more than 128 edges together and all but the last block of a segment lie inside its edge window,
// so a segment has at most 2 (kLbSegEdges - 1) / 129 + 2 <= kLbSegCap blocks.
// Per CTA: lm_first is staged in shared memory kLbThreads landmarks at a time, warp 0 cuts it 32 landmarks per step (the first
// landmark that does not fit is found by a ballot).
__device__ __forceinline__ int lower_bound_first(const int* __restrict__ lm_first, int L, int v) {
    int lo = 0, hi = L;                                 // first landmark l with lm_first[l] >= v (L if none)
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (lm_first[mid] < v) lo = mid + 1; else hi = mid; }
    return lo;
}
__global__ void __launch_bounds__(kLbThreads) k_ba_landmark_blocks(int L, const int* __restrict__ lm_first, int4* __restrict__ blocks, int* __restrict__ nblocks) {
    __shared__ int s_first[kLbThreads + 1];
    __shared__ int s_range[2];
    const int lane = threadIdx.x & 31, seg = blockIdx.x;
    if (threadIdx.x < 2) s_range[threadIdx.x] = lower_bound_first(lm_first, L, (seg + (int)threadIdx.x) * kLbSegEdges);
    __syncthreads();
    const int l0 = s_range[0], l1 = (seg + 1 == (int)gridDim.x) ? L : s_range[1];
    blocks += (size_t)seg * kLbSegCap;
    int start = l0, s = l0 < L ? lm_first[l0] : 0, nb = 0;   // warp 0: first landmark and first edge of the open block, blocks emitted
    for (int c0 = l0; c0 < l1; c0 += kLbThreads) {
        __syncthreads();
        for (int q = threadIdx.x; q <= kLbThreads; q += kLbThreads)
            if (c0 + q <= l1) s_first[q] = lm_first[c0 + q];
        __syncthreads();
        if (threadIdx.x >= 32) continue;
        const int cn = min(kLbThreads, l1 - c0);
        for (int g = 0; g < cn; g += 32) {
            const int j = g + lane;
            const bool in = j < cn;
            const int eb = in ? s_first[j] : 0, ee = in ? s_first[j + 1] : 0;
            int cur = c0 + g;                           // first landmark of this step not placed yet
            for (;;) {
                const unsigned over = __ballot_sync(0xffffffffu, in && c0 + j >= cur && ee - s > 128);
                if (!over) break;
                const int f = __ffs(over) - 1, lf = c0 + g + f;
                const int bf = __shfl_sync(0xffffffffu, eb, f), ef = __shfl_sync(0xffffffffu, ee, f);
                if (lf == start) {                      // alone and still more than 128 edges: a block of its own
                    if (lane == 0) blocks[nb] = make_int4(start, lf + 1, s, ef);
                    start = lf + 1; s = ef;
                } else {
                    if (lane == 0) blocks[nb] = make_int4(start, lf, s, bf);
                    start = lf; s = bf;
                }
                cur = start;
                ++nb;
            }
        }
    }
    if (threadIdx.x == 0) {
        if (start < l1) blocks[nb++] = make_int4(start, l1, s, lm_first[l1]);
        nblocks[seg] = nb;
    }
}

// observations on free keyframes per landmark (one thread per landmark: the dependent index loads of 20 k landmarks overlap),
// left in pair_off[l] for the scan below
__global__ void __launch_bounds__(256) k_ba_pair_counts(int L, const int* __restrict__ lm_first, const int* __restrict__ obs_kf,
                                                         const int* __restrict__ free_idx, int* __restrict__ pair_off, const long long* __restrict__ counts) {
    if (counts[4] != 0x7fffffffffffffffll) return;      // invalid input: the index arrays cannot be trusted
    const int l = blockIdx.x * 256 + threadIdx.x;
    if (l >= L) return;
    int m = 0;
    for (int p = lm_first[l]; p < lm_first[l + 1]; ++p) m += free_idx[obs_kf[p]] >= 0;
    pair_off[l] = m;
}

__global__ void __launch_bounds__(1024) k_ba_pair_offsets(int L, int* __restrict__ pair_off, long long* counts) {
    // exclusive prefix of m (m + 1) / 2 over the landmarks, in place: every thread owns a contiguous run of landmarks
    // (local sum, ONE block scan of the 1024 run sums, offsets written back), 64-bit sums clamped to int on output
    __shared__ long long wsum[33];
    __shared__ long long edges;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (counts[4] != 0x7fffffffffffffffll) return;      // invalid input: the index arrays cannot be trusted
    if (tid == 0) edges = 0;
    const int run = (L + 1023) / 1024;
    const int b = min(L, tid * run), e = min(L, b + run);
    long long local = 0, my_edges = 0;
    for (int l = b; l < e; ++l) {
        const int m = pair_off[l];                   // k_ba_pair_counts
        local += (long long)m * (m + 1) / 2;
        my_edges += m;
    }
    long long v = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
    if (lane == 31) wsum[wid] = v;
    __syncthreads();
    if (wid == 0) {
        const long long x = wsum[lane];
        long long ws = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += u; }
        wsum[lane] = ws - x;                          // exclusive over the warps
        if (lane == 31) wsum[32] = ws;                // total
    }
    __syncthreads();
    long long excl = wsum[wid] + v - local;
    for (int l = b; l < e; ++l) {
        const int m = pair_off[l];
        pair_off[l] = (int)min(excl, (long long)0x7fffffff);
        excl += (long long)m * (m + 1) / 2;
    }
    my_edges = (long long)warp_sum((double)my_edges);       // exact: far below 2^53
    if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&edges), (unsigned long long)my_edges);
    __syncthreads();
    if (tid == 0) { const long long total = wsum[32]; pair_off[L] = (int)min(total, (long long)0x7fffffff); counts[1] = total; counts[2] = edges; }
}

__global__ void __launch_bounds__(256) k_fill_f32(float* p, size_t n, float v) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) p[i] = v;
}

// -------------------------------------------------------------------- co-observation lists
// For landmark l with free-keyframe observations o_0..o_{m-1} (in edge order) emit the m(m+1)/2
// entries (key = pair id of (min fa, max fb), value = (edge on a, edge on b)), at pair_off[l].
__global__ void __launch_bounds__(128) k_ba_emit_pairs(BaDev P, const int* __restrict__ pair_off, unsigned* __restrict__ keys,
                                                        unsigned long long* __restrict__ vals) {
    const int l = blockIdx.x * 128 + threadIdx.x;
    if (l >= P.L) return;
    int pos = pair_off[l];
    const int nf = P.nfree;
    for (int p = P.lm_first[l]; p < P.lm_first[l + 1]; ++p) {
        const int fa = P.free_idx[P.obs_kf[p]];
        if (fa < 0) continue;
        for (int q = p; q < P.lm_first[l + 1]; ++q) {
            const int fb = P.free_idx[P.obs_kf[q]];
            if (fb < 0) continue;
            int a = fa, b = fb, oa = p, ob = q;
            if (a > b) { a = fb; b = fa; oa = q; ob = p; }
            keys[pos] = (unsigned)(a * nf - a * (a - 1) / 2 + (b - a));
            vals[pos] = ((unsigned long long)(unsigned)ob << 32) | (unsigned)oa;
            ++pos;
        }
    }
}

__global__ void __launch_bounds__(256) k_ba_segments(const unsigned* __restrict__ keys, int n, int* __restrict__ seg_begin, int* __restrict__ seg_end) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const unsigned k = keys[i];
    if (i == 0 || keys[i - 1] != k) seg_begin[k] = i;
    if (i == n - 1 || keys[i + 1] != k) seg_end[k] = i + 1;
}

// sorted (edge on a, edge on b) -> one 16-byte record per co-observation {edge on a, edge on b, landmark, 0}
__global__ void __launch_bounds__(256) k_ba_pair_records(const unsigned long long* __restrict__ vals, int n, const int* __restrict__ obs_lm, int4* __restrict__ rec) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const unsigned long long v = vals[i];
    const int oa = (int)(unsigned)(v & 0xffffffffull), ob = (int)(unsigned)(v >> 32);
    rec[i] = make_int4(oa, ob, obs_lm[oa], 0);
}

// ---------------------------------------------------------------- stable radix sort of the co-observation list
// (pair id -> (edge on a, edge on b)), least-significant digit first, kSortBits bits per pass: ONE pass for up to 2048 keyframe
// pairs (63 free keyframes -- every local BA), two for up to 4 M pairs.  A pass is three launches:
//   k_sort_hist         digit histogram of every tile of kSortTile entries                      hist[tile][bin]
//   k_sort_tile_prefix  per bin: exclusive prefix over the tiles (one warp per bin), bin totals  hist[tile][bin], bin_total[bin]
//   k_sort_scatter      per tile: bin bases (scan of the totals) + the tile's prefix; the tile is walked by 8 warps x 8 chunks of 32
//                       consecutive entries; entries of one chunk with the same digit are ranked by lane (match.any), chunks of a
//                       warp by a running per-warp counter, warps by an exclusive prefix over the per-warp counts: the order of equal
//                       digits is the input order (stable), nothing depends on thread timing.
constexpr int kSortBits = 11, kSortBins = 1 << kSortBits, kSortTile = 2048, kSortThreads = 256, kSortWarps = kSortThreads / 32;
static_assert(kSortTile == kSortWarps * 8 * 32 && kSortBins == kSortThreads * 8, "tile / bin geometry");

__global__ void __launch_bounds__(kSortThreads) k_sort_hist(const unsigned* __restrict__ keys, int n, int shift, int* __restrict__ hist) {
    __shared__ int sh[kSortBins];
    for (int i = threadIdx.x; i < kSortBins; i += kSortThreads) sh[i] = 0;
    __syncthreads();
    const int base = blockIdx.x * kSortTile;
    for (int i = threadIdx.x; i < kSortTile; i += kSortThreads) {
        const int idx = base + i;
        if (idx < n) atomicAdd(&sh[(keys[idx] >> shift) & (kSortBins - 1)], 1);      // integer counts: order free
    }
    __syncthreads();
    int* out = hist + (size_t)blockIdx.x * kSortBins;
    for (int i = threadIdx.x; i < kSortBins; i += kSortThreads) out[i] = sh[i];
}

__global__ void __launch_bounds__(256) k_sort_tile_prefix(int* __restrict__ hist, int ntiles, int* __restrict__ bin_total) {
    const int bin = (int)((blockIdx.x * 256u + threadIdx.x) >> 5), lane = threadIdx.x & 31;     // grid = kSortBins / 8
    int run = 0;
    for (int t0 = 0; t0 < ntiles; t0 += 32) {
        const int t = t0 + lane;
        int* p = hist + (size_t)min(t, ntiles - 1) * kSortBins + bin;
        const int v = t < ntiles ? *p : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
        if (t < ntiles) *p = run + inc - v;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) bin_total[bin] = run;
}

__global__ void __launch_bounds__(kSortThreads) k_sort_scatter(const unsigned* __restrict__ keys, const unsigned long long* __restrict__ vals, int n, int shift,
                                                               const int* __restrict__ hist, const int* __restrict__ bin_total,
                                                               unsigned* __restrict__ keys_out, unsigned long long* __restrict__ vals_out) {
    __shared__ int s_base[kSortBins];                         // first output slot of (bin, this tile)
    __shared__ unsigned short s_cnt[kSortWarps][kSortBins];   // per warp: entries per bin, then the running offset inside the tile
    __shared__ int s_warp[kSortWarps];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    for (int i = tid; i < kSortWarps * kSortBins / 2; i += kSortThreads) reinterpret_cast<unsigned*>(&s_cnt[0][0])[i] = 0;
    // bin bases: exclusive scan of the bin totals (8 consecutive bins per thread) + this tile's prefix
    int tot[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { tot[k] = bin_total[tid * 8 + k]; sum += tot[k]; }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) s_warp[w] = inc;
    // the tile: warp w owns entries [256 w, 256 w + 256), chunk c = 32 consecutive entries
    const int base = blockIdx.x * kSortTile + w * 256;
    unsigned key[8];
    unsigned long long val[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int idx = base + c * 32 + lane;
        key[c] = idx < n ? keys[idx] : 0u;
        val[c] = idx < n ? vals[idx] : 0ull;
    }
    __syncthreads();
    {
        int run = inc - sum;
        for (int ww = 0; ww < w; ++ww) run += s_warp[ww];
        const int* hrow = hist + (size_t)blockIdx.x * kSortBins;
#pragma unroll
        for (int k = 0; k < 8; ++k) { s_base[tid * 8 + k] = run + hrow[tid * 8 + k]; run += tot[k]; }
    }
    // per-warp digit counts (one leader lane per distinct digit of a chunk: plain read-modify-write, the warp owns its row)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const bool valid = base + c * 32 + lane < n;
        const unsigned d = valid ? (key[c] >> shift) & (kSortBins - 1) : (unsigned)kSortBins;     // invalid lanes: a group of their own
        const unsigned m = __match_any_sync(0xffffffffu, d);
        if (valid && lane == __ffs(m) - 1) s_cnt[w][d] = (unsigned short)(s_cnt[w][d] + __popc(m));
        __syncwarp();
    }
    __syncthreads();
    for (int bin = tid; bin < kSortBins; bin += kSortThreads) {
        unsigned r = 0;
#pragma unroll
        for (int ww = 0; ww < kSortWarps; ++ww) { const unsigned t = s_cnt[ww][bin]; s_cnt[ww][bin] = (unsigned short)r; r += t; }
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const bool valid = base + c * 32 + lane < n;
        const unsigned d = valid ? (key[c] >> shift) & (kSortBins - 1) : (unsigned)kSortBins;
        const unsigned m = __match_any_sync(0xffffffffu, d);
        if (valid) {
            const int pos = s_base[d] + (int)s_cnt[w][d] + __popc(m & ((1u << lane) - 1u));
            keys_out[pos] = key[c];
            vals_out[pos] = val[c];
        }
        __syncwarp();
        if (valid && lane == __ffs(m) - 1) s_cnt[w][d] = (unsigned short)(s_cnt[w][d] + __popc(m));
        __syncwarp();
    }
}

// sorts (keys, vals) by the low end_bit bits of the keys, stable; the result is in *keys_sorted / *vals_sorted (one of the two
// buffer pairs).  hist: ntiles x kSortBins + kSortBins ints of scratch.
size_t sort_scratch_ints(long long n) { return (size_t)((n + kSortTile - 1) / kSortTile) * kSortBins + kSortBins; }
int sort_pairs(cudaStream_t st, unsigned* k0, unsigned* k1, unsigned long long* v0, unsigned long long* v1, int n, int end_bit, int* scratch,
               unsigned** keys_sorted, unsigned long long** vals_sorted) {
    const int ntiles = (n + kSortTile - 1) / kSortTile;
    int* hist = scratch;
    int* bin_total = scratch + (size_t)ntiles * kSortBins;
    unsigned *kin = k0, *kout = k1;
    unsigned long long *vin = v0, *vout = v1;
    for (int shift = 0; shift < end_bit; shift += kSortBits) {
        k_sort_hist<<<ntiles, kSortThreads, 0, st>>>(kin, n, shift, hist);
        OVS_LAUNCH_CHECK();
        k_sort_tile_prefix<<<kSortBins / 8, 256, 0, st>>>(hist, ntiles, bin_total);
        OVS_LAUNCH_CHECK();
        k_sort_scatter<<<ntiles, kSortThreads, 0, st>>>(kin, vin, n, shift, hist, bin_total, kout, vout);
        OVS_LAUNCH_CHECK();
        std::swap(kin, kout); std::swap(vin, vout);
    }
    *keys_sorted = kin; *vals_sorted = vin;
    return OVS_OK;
}

// pair id -> (a, b), a <= b, ids numbered row by row; diag[a] = id of (a, a)
__global__ void __launch_bounds__(128) k_ba_pair_table(int nfree, int2* __restrict__ pair_ab, int* __restrict__ diag) {
    const int a = blockIdx.x;
    const int base = a * nfree - a * (a - 1) / 2;
    for (int b = a + threadIdx.x; b < nfree; b += 128) pair_ab[base + (b - a)] = make_int2(a, b);
    if (threadIdx.x == 0) diag[a] = base;
}

// Chunk tables of the two-stage reductions, built on the device (no host round trip in prepare): item i (a keyframe
// pair, or -- with `ids` -- the diagonal pair of free keyframe i) owns ceil(len / 128) chunks of its segment of the
// sorted co-observation list.  One block: exclusive scan of the chunk counts in tiles of 1024 with a running carry.
__global__ void __launch_bounds__(1024) k_ba_chunk_scan(const int* __restrict__ ids, int count, const int* __restrict__ seg_begin,
                                                         const int* __restrict__ seg_end, int* __restrict__ chunk_begin, int* __restrict__ total) {
    __shared__ int wsum[32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < count; base += 1024) {
        const int i = base + tid;
        int c = 0;
        if (i < count) { const int id = ids ? ids[i] : i; c = (seg_end[id] - seg_begin[id] + 127) / 128; }
        int v = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
        if (lane == 31) wsum[wid] = v;
        __syncthreads();
        if (wid == 0) {
            int ws = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += u; }
            wsum[lane] = ws;      // inclusive over warps
        }
        __syncthreads();
        const int excl = carry + (wid ? wsum[wid - 1] : 0) + v - c;
        if (i < count) chunk_begin[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + c;
        __syncthreads();
    }
    if (tid == 0) { chunk_begin[count] = carry; *total = carry; }
}

// chunk = {tag, begin, end, 0}; tag = the pair id (Schur) or the free keyframe index (Hpp accumulation)
__global__ void __launch_bounds__(128) k_ba_chunk_fill(const int* __restrict__ ids, int count, const int* __restrict__ seg_begin,
                                                        const int* __restrict__ seg_end, const int* __restrict__ chunk_begin, int4* __restrict__ chunks) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= count) return;
    const int id = ids ? ids[i] : i;
    const int e1 = seg_end[id];
    int c = chunk_begin[i];
    for (int e0 = seg_begin[id]; e0 < e1; e0 += 128, ++c) chunks[c] = make_int4(i, e0, min(e0 + 128, e1), 0);
}

// ------------------------------------------------------------------------- pose optimiser
struct PoseOptArgs {
    CameraD cam;
    int n;
    const double* pts_w; const float2* obs_xy; const float* obs_xr; const float* inv_sigma_sq;
    double* pose;              // 12, in/out
    unsigned char* outlier;    // n, out
    int num_trials, num_each_iter;
    double delta, chi2_2d, chi2_3d;
    double* stats;             // [0] iterations [1] trials(solves) [2] rounds [3] final chi2 [4] inliers [5..] lambda_init per round
};

struct LmRoundStats {
    int iterations, trials;      // iterations run, trials (solves) over them
    double lambda_init;          // set when iterations > 0
    double lambda, chi2;         // after the last iteration; set when iterations > 0
};

// SparseOptimizer::optimize(iterations) of g2o's OptimizationAlgorithmLevenberg with a fresh initializeOptimization (lambda_init
// again) for one vertex of D parameters (an estimate of P doubles in shared memory, est), run redundantly by every CTA of the
// cluster on the sums `reduce` leaves in every CTA.  build(est, acc) is the kernel's edge pass at an estimate: the edge errors
// it stores and this thread's share of {H (packed D x D), b (D), robust chi2} in acc; oplus(est, x, out) applies an update.
// g2o evaluates the errors at the candidate of a trial and, once the trial is accepted, evaluates them again at the same
// estimate at the top of the next iteration, where it also linearises.  Here the trial's pass over the edges already forms H
// and b at the candidate (same code, same summation order as the pass at the top of an iteration), so an accepted trial hands
// the next iteration its system: one pass over the edges and one cluster reduction per iteration instead of two.  A round
// starts with a fresh pass.
template <int D, int P, class Reduce, class Build, class Oplus>
__device__ __forceinline__ LmRoundStats cluster_lm_round(int iterations, double* est, Reduce& reduce, Build&& build, Oplus&& oplus) {
    constexpr int NH = D * (D + 1) / 2, NS = NH + D + 1;
    __shared__ double s_cand[P], s_x[D];
    __shared__ int s_flag;
    const int tid = threadIdx.x;
    LmRoundStats st{0, 0, 0.0, 0.0, 0.0};
    double lambda = 0, ni = 2;
    bool ok = true, have_sys = false;
    int it = 0;
    double Hs[NH], bs[D], currentChi = 0;
    for (; it < iterations && ok; ++it) {
        if (!have_sys) {
            double acc[NS];
            build(est, acc);
            const double* sys = reduce(acc, NS);
#pragma unroll
            for (int k = 0; k < NH; ++k) Hs[k] = sys[k];
#pragma unroll
            for (int k = 0; k < D; ++k) bs[k] = sys[NH + k];
            currentChi = sys[NH + D];
            have_sys = true;
        }
        if (it == 0) {
            double md = 0;
#pragma unroll
            for (int k = 0; k < D; ++k) md = fmax(md, fabs(Hs[ovs::sym<D>(k, k)]));
            lambda = 1e-5 * md;
            ni = 2;
            st.lambda_init = lambda;
        }
        double rho = 0;
        int qmax = 0;
        do {
            if (tid == 0) {
                double xs[D];
                const bool ok2 = ovs::solve_spd<D>(Hs, lambda, bs, xs);
                s_flag = ok2 ? 1 : 0;
                if (ok2) {
                    for (int k = 0; k < D; ++k) s_x[k] = xs[k];
                    double out[P];
                    oplus(est, xs, out);
                    for (int k = 0; k < P; ++k) s_cand[k] = out[k];
                } else {
                    for (int k = 0; k < P; ++k) s_cand[k] = est[k];
                }
            }
            __syncthreads();
            const bool ok2 = s_flag != 0;
            const double* sys;
            {
                double acc[NS];
                build(s_cand, acc);
                sys = reduce(acc, NS);
            }
            double tempChi = sys[NH + D];
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0;
            if (ok2) for (int k = 0; k < D; ++k) scale += s_x[k] * (lambda * s_x[k] + bs[k]);
            scale += 1e-3;
            rho /= scale;
            const bool accept = rho > 0 && isfinite(tempChi);
            if (accept) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = fmin(alpha, 2. / 3.);
                lambda *= fmax(1. / 3., alpha);
                ni = 2;
                currentChi = tempChi;
#pragma unroll
                for (int k = 0; k < NH; ++k) Hs[k] = sys[k];      // the system at the accepted estimate
#pragma unroll
                for (int k = 0; k < D; ++k) bs[k] = sys[NH + k];
            } else {
                lambda *= ni;
                ni *= 2;
            }
            __syncthreads();                    // the sums, s_x, est and s_cand have been read by every thread
            if (accept && tid < P) est[tid] = s_cand[tid];
            __syncthreads();
            ++qmax; ++st.trials;
        } while (rho < 0 && qmax < kMaxTrials);
        if (qmax == kMaxTrials || rho == 0) ok = false;
    }
    st.iterations = it;
    st.lambda = lambda; st.chi2 = currentChi;
    return st;
}

// pose_optimizer::optimize: the whole call is ONE kernel on a thread-block cluster of kPoseCluster
// CTAs (the edge linearisation is FP64-throughput bound on one SM).  Every CTA owns a slice of the
// edges; the 6x6 normal equations and the chi2 sums are reduced across the cluster (ClusterSum),
// so every CTA then takes the same Levenberg decision redundantly (no broadcast needed).  Edge state
// lives in global scratch (err: n x 3 doubles, level: n bytes).
__global__ void __cluster_dims__(kPoseCluster, 1, 1) __launch_bounds__(kPoseThreads, 1)
k_pose_optimize(PoseOptArgs A, double* __restrict__ err, unsigned char* __restrict__ level) {
    __shared__ double s_pose[12];
    const int tid = threadIdx.x;
    const unsigned my_rank = cluster_rank();
    const int gtid = (int)my_rank * kPoseThreads + tid;
    constexpr int GS = kPoseCluster * kPoseThreads;
    const int n = A.n;
    if (tid < 12) s_pose[tid] = A.pose[tid];
    for (int i = gtid; i < n; i += GS) { level[i] = 0; A.outlier[i] = 0; }
    cluster_sync_mem();     // every CTA of the cluster is running before anyone writes into its shared memory
    ClusterSum<28, kPoseCluster, kPoseThreads> reduce_all;
    bool use_huber = true;

    // computeActiveErrors + buildSystem in one pass at pose `ps`: edge errors to err[], this thread's share of
    // {H (21), b (6), robust chi2} over its active edges into acc
    auto build_local = [&](const double* ps, double* acc) {
#pragma unroll
        for (int k = 0; k < 28; ++k) acc[k] = 0;
        double pose[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) pose[k] = ps[k];
        for (int i = gtid; i < n; i += GS) {
            if (level[i]) continue;
            const float xr = A.obs_xr ? A.obs_xr[i] : -1.0f;
            const bool stereo = xr >= 0.0f;
            const float2 xy = A.obs_xy[i];
            const double obs[3] = {(double)xy.x, (double)xy.y, (double)xr};
            const double pw[3] = {A.pts_w[3 * (size_t)i], A.pts_w[3 * (size_t)i + 1], A.pts_w[3 * (size_t)i + 2]};
            double e[3] = {0, 0, 0}, Jp[18];
            const int dim = ovs::edge_eval(A.cam, pose, pw, obs, stereo, e, Jp, nullptr);
            err[3 * (size_t)i] = e[0]; err[3 * (size_t)i + 1] = e[1]; err[3 * (size_t)i + 2] = stereo ? e[2] : 0.0;
            const double w = (double)A.inv_sigma_sq[i];
            double chi = 0;
            for (int d = 0; d < dim; ++d) chi += w * e[d] * e[d];
            double r0 = chi, r1 = 1.0;
            if (use_huber) ovs::huber(chi, A.delta, &r0, &r1);
            acc[27] += r0;
            const double ww = r1 * w;
            for (int a = 0; a < 6; ++a) {
                double g = 0;
                for (int d = 0; d < dim; ++d) g -= Jp[6 * d + a] * ww * e[d];
                acc[21 + a] += g;
                for (int b = a; b < 6; ++b) {
                    double hh = 0;
                    for (int d = 0; d < dim; ++d) hh += Jp[6 * d + a] * ww * Jp[6 * d + b];
                    acc[ovs::sym6(a, b)] += hh;
                }
            }
        }
    };

    int total_iters = 0, total_trials = 0, rounds = 0, num_bad = 0;
    for (int trial = 0; trial < A.num_trials; ++trial) {
        // ---- optimizer.optimize(num_each_iter); a round starts with a fresh pass (the outlier levels and the robust kernel
        // change between rounds)
        const LmRoundStats r = cluster_lm_round<6, 12>(A.num_each_iter, s_pose, reduce_all, build_local,
                                                       [](const double* ps, const double* x, double* out) { ovs::pose_oplus(ps, x, out); });
        if (r.iterations > 0 && gtid == 0 && rounds < 8) A.stats[5 + rounds] = r.lambda_init;
        total_iters += r.iterations; total_trials += r.trials; ++rounds;
        // ---- outlier re-classification
        {
            double pose[12];
#pragma unroll
            for (int k = 0; k < 12; ++k) pose[k] = s_pose[k];
            double bad[1] = {0};
            for (int i = gtid; i < n; i += GS) {
                const float xr = A.obs_xr ? A.obs_xr[i] : -1.0f;
                const bool stereo = xr >= 0.0f;
                if (level[i]) {  // edge->computeError() for current outliers
                    const float2 xy = A.obs_xy[i];
                    const double obs[3] = {(double)xy.x, (double)xy.y, (double)xr};
                    const double pw[3] = {A.pts_w[3 * (size_t)i], A.pts_w[3 * (size_t)i + 1], A.pts_w[3 * (size_t)i + 2]};
                    double e[3] = {0, 0, 0};
                    ovs::edge_eval(A.cam, pose, pw, obs, stereo, e, nullptr, nullptr);
                    err[3 * (size_t)i] = e[0]; err[3 * (size_t)i + 1] = e[1]; err[3 * (size_t)i + 2] = stereo ? e[2] : 0.0;
                }
                const double w = (double)A.inv_sigma_sq[i];
                const double e0 = err[3 * (size_t)i], e1 = err[3 * (size_t)i + 1], e2 = err[3 * (size_t)i + 2];
                double chi = w * (e0 * e0 + e1 * e1);
                if (stereo) chi += w * e2 * e2;
                const bool outl = (stereo ? A.chi2_3d : A.chi2_2d) < chi;
                level[i] = outl ? 1 : 0;
                A.outlier[i] = outl ? 1 : 0;
                bad[0] += outl ? 1.0 : 0.0;
            }
            num_bad = (int)(reduce_all(bad, 1)[0] + 0.5);
            __syncthreads();
        }
        if (trial == A.num_trials - 2) use_huber = false;
        if (n - num_bad < 5) break;
    }
    // final chi2 over inlier edges from the stored errors
    double fc[1] = {0};
    for (int i = gtid; i < n; i += GS) {
        if (level[i]) continue;
        const bool stereo = A.obs_xr && A.obs_xr[i] >= 0.0f;
        const double w = (double)A.inv_sigma_sq[i];
        const double e0 = err[3 * (size_t)i], e1 = err[3 * (size_t)i + 1], e2 = err[3 * (size_t)i + 2];
        fc[0] += w * (e0 * e0 + e1 * e1) + (stereo ? w * e2 * e2 : 0.0);
    }
    const double final_chi2 = reduce_all(fc, 1)[0];
    if (gtid == 0) {
        A.stats[0] = total_iters; A.stats[1] = total_trials; A.stats[2] = rounds; A.stats[3] = final_chi2; A.stats[4] = n - num_bad;
    }
    if (gtid < 12) A.pose[gtid] = s_pose[gtid];
}

}  // namespace

// ================================================================================= handle
struct ovs_ba_plan;
extern "C" void ovs_optimizer_destroy(ovs_optimizer* h);
struct ovs_optimizer {
    int device = 0;
    ovs_ba_plan* plan = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2]{};
    std::vector<cudaEvent_t> solver_ev;             // pairs around the reduced-system solver launches of one run
    // The launch sequence of one LM iteration (linearise + accumulate, plan, the trial batches) is STATIC -- damping
    // values, ring slots and "is there anything to do" are read from device memory (LmCtl) -- so it can be captured once
    // per run and replayed as one CUDA graph per iteration (ovs_optimizer_set_graphs).
    cudaGraphExec_t gx_iter = nullptr;
    int spec_width = kSpec;                         // LM trials evaluated speculatively in the first batch of an iteration (1..kSpec)
    int spec_width2 = 0;                            // > 0: a second batch of that width is enqueued statically behind the first (it
                                                    // returns at once when the first batch decided the iteration)
    int use_graphs = 0;
    int lm_host_sync = -1;                          // -1: automatic (only the multi-launch solver of very large systems syncs per
                                                    // batch, to skip its ~100-launch batches); 0 / 1: development override
    bool pending = false;                           // work enqueued on the stream that reads the pinned arena
    // grow-only byte arenas
    uint8_t* d_arena = nullptr; size_t d_cap = 0;
    uint8_t* h_arena = nullptr; size_t h_cap = 0;   // pinned
    uint8_t* d_work = nullptr; size_t w_cap = 0;    // local BA: buffers sized by the number of free keyframes / co-observations
    int* h_mirror = nullptr;                         // pinned, mapped: [0] nbatch, [1] active (written by the device), [2] stop word (host)
    int* d_mirror = nullptr;
    int chol_cluster = kCholCluster;                 // CTAs per Cholesky cluster (1, 2, 4 or 8)
};

namespace {

CameraD to_cam(const ovs_camera* c) {
    CameraD d;
    d.model = c->model; d.fx = c->fx; d.fy = c->fy; d.cx = c->cx; d.cy = c->cy; d.fb = c->focal_x_baseline; d.cols = c->cols; d.rows = c->rows;
    return d;
}

}  // namespace

static void invalidate_plan(ovs_optimizer* h);

// ------------------------------------------------------------------------ pose optimiser
extern "C" int ovs_pose_optimize_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int n, const double* pts_w,
                                      const float* obs_xy, const float* obs_x_right, const float* inv_sigma_sq,
                                      double* pose_cw, uint8_t* outlier_flags, int num_trials, int num_each_iter,
                                      int* num_inliers, ovs_ba_stats* stats) {
    OVS_REQUIRE(h && cam && pose_cw && num_inliers && n >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n == 0 || (pts_w && obs_xy && inv_sigma_sq && outlier_flags), OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(cam->model == ovs::kCamPerspective || cam->model == ovs::kCamEquirectangular, OVS_ERR_INVALID_ARG, "unknown camera model");
    OVS_REQUIRE(num_trials >= 1 && num_each_iter >= 0, OVS_ERR_INVALID_ARG, "bad iteration counts");
    if (stats) memset(stats, 0, sizeof(*stats));
    for (int i = 0; i < n; ++i) outlier_flags[i] = 0;
    *num_inliers = 0;
    if (n < 5) return OVS_OK;  // `if (num_init_obs < 5) return 0;`
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // The pose optimiser carves its buffers from the arenas a prepared local-BA problem lives in: that problem is gone.
    invalidate_plan(h);
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(h->stream)); h->pending = false; }
    const size_t N = (size_t)n;
    PoseOptArgs A;
    double *hp, *hpose, *hstats, *derr; float *hxy, *hxr, *hw; uint8_t *hout, *dlevel;
    ovs::Staging S;
    const int rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        A.pts_w = S.in(hp, 3 * N); A.obs_xy = (const float2*)S.in(hxy, 2 * N); A.obs_xr = S.in(hxr, N); A.inv_sigma_sq = S.in(hw, N);
        A.pose = S.io(hpose, 12); A.stats = S.io(hstats, 16); A.outlier = S.out(hout, N);
        derr = S.dev<double>(3 * N); dlevel = S.dev<uint8_t>(N);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hp, pts_w, 24 * N); memcpy(hxy, obs_xy, 8 * N); memcpy(hw, inv_sigma_sq, 4 * N);
    if (obs_x_right) memcpy(hxr, obs_x_right, 4 * N); else for (size_t i = 0; i < N; ++i) hxr[i] = -1.0f;
    memcpy(hpose, pose_cw, 96);
    memset(hstats, 0, 128);
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    A.cam = to_cam(cam); A.n = n; A.num_trials = num_trials; A.num_each_iter = num_each_iter;
    const float chi_sq_2D = 5.99146f, chi_sq_3D = 7.81473f;
    A.delta = (double)(setup_is_mono ? sqrtf(chi_sq_2D) : sqrtf(chi_sq_3D));
    A.chi2_2d = (double)chi_sq_2D; A.chi2_3d = (double)chi_sq_3D;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    k_pose_optimize<<<kPoseCluster, kPoseThreads, 0, st>>>(A, derr, dlevel);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(pose_cw, hpose, 96);
    memcpy(outlier_flags, hout, N);
    *num_inliers = (int)hstats[4];
    if (stats) {
        stats->num_iterations = (int)hstats[0]; stats->num_trials = (int)hstats[1]; stats->num_rounds = (int)hstats[2];
        stats->final_chi2 = hstats[3];
        for (int r = 0; r < 8 && r < stats->num_rounds; ++r) stats->lambda_init[r] = hstats[5 + r];
        float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
        stats->device_us = ms * 1000.f;
    }
    return OVS_OK;
}

// ----------------------------------------------------------------------- transform optimiser
namespace {

constexpr int kSim3Threads = 256;
constexpr int kSim3Cluster = 8;
constexpr int kSim3Stride = kSim3Threads * kSim3Cluster;   // pairs per grid-stride step: thread g takes pairs g, g + 2048, ...
constexpr int kSim3Sums = 36;                              // H (28, packed 7x7), b (7), robust chi2

struct Sim3OptArgs {
    CameraD cam1, cam2;
    double pose1[12], pose2[12];   // cam_pose_1w, cam_pose_2w
    int n;
    const double* pw1; const float2* xy1; const float* w1;   // lm_1 (world), keyframe 1's keypoint, its inv_level_sigma_sq
    const double* pw2; const float2* xy2; const float* w2;   // lm_2 (world), keyframe 2's keypoint, its inv_level_sigma_sq
    double* sim3;                  // 13, in / out (written only when the call succeeds)
    unsigned char* inlier;         // n, out
    int fix_scale, num_first_iter, num_iter;
    double delta, chi_sq;
    // [0] iterations [1] trials [2] rounds [3] final chi2 [4] inliers (the return value) [5..6] lambda_init per round
    // [7..8] iterations per round [9] last lambda [10] last chi2
    double* stats;
};

// transform_optimizer::optimize: the whole call is ONE kernel on a cluster of kSim3Cluster CTAs, organised as
// k_pose_optimize: every CTA owns a grid-stride slice of the pairs (both edges of a pair in one thread), the 7x7 system and the
// chi2 are reduced across the cluster (ClusterSum), so every CTA holds the same bits and takes the same Levenberg decision.
// err (n x 4: e12, e21) keeps the errors of the last evaluated trial, which the outlier tests read as g2o's chi2() does;
// level (n) is 1 for the pairs cut so far.
__global__ void __cluster_dims__(kSim3Cluster, 1, 1) __launch_bounds__(kSim3Threads, 1)
k_sim3_optimize(Sim3OptArgs A, double* __restrict__ err, unsigned char* __restrict__ level) {
    constexpr int NS = kSim3Sums;
    __shared__ double s_S[13];
    const int tid = threadIdx.x;
    const unsigned my_rank = cluster_rank();
    const int gtid = (int)my_rank * kSim3Threads + tid;
    const int n = A.n;
    if (tid < 13) s_S[tid] = A.sim3[tid];
    for (int i = gtid; i < n; i += kSim3Stride) { level[i] = 0; A.inlier[i] = 0; }
    cluster_sync_mem();     // every CTA of the cluster is running before anyone writes into its shared memory
    ClusterSum<NS, kSim3Cluster, kSim3Threads> reduce_all;

    // computeActiveErrors + buildSystem at S in one pass: errors to err[], this thread's share of {H, b, robust chi2}
    auto build_local = [&](const double* Sp, double* acc) {
#pragma unroll
        for (int k = 0; k < NS; ++k) acc[k] = 0;
        double S[13];
#pragma unroll
        for (int k = 0; k < 13; ++k) S[k] = Sp[k];
        for (int i = gtid; i < n; i += kSim3Stride) {
            if (level[i]) continue;
#pragma unroll 1
            for (int edge = 0; edge < 2; ++edge) {
                const double* pose = edge == 0 ? A.pose2 : A.pose1;
                const double* pwp = (edge == 0 ? A.pw2 : A.pw1) + 3 * (size_t)i;
                const float2 xy = edge == 0 ? A.xy1[i] : A.xy2[i];
                const double w = (double)(edge == 0 ? A.w1[i] : A.w2[i]);
                const double pw[3] = {pwp[0], pwp[1], pwp[2]};
                double pc[3];
                ovs::mat3_vec(pose, pw, pc);
                pc[0] += pose[9]; pc[1] += pose[10]; pc[2] += pose[11];
                const double obs[2] = {(double)xy.x, (double)xy.y};
                double e[2], J[14];
                if (edge == 0) ovs::sim3_edge_forward(A.cam1, S, pc, obs, e, J);
                else ovs::sim3_edge_backward(A.cam2, S, pc, obs, e, J);
                err[4 * (size_t)i + 2 * edge] = e[0]; err[4 * (size_t)i + 2 * edge + 1] = e[1];
                const double chi = w * (e[0] * e[0] + e[1] * e[1]);
                double r0, r1;
                ovs::huber(chi, A.delta, &r0, &r1);
                acc[35] += r0;
                const double ww = r1 * w;
                for (int a = 0; a < 7; ++a) {
                    acc[28 + a] -= J[a] * ww * e[0] + J[7 + a] * ww * e[1];
                    for (int c = a; c < 7; ++c) acc[ovs::sym<7>(a, c)] += J[a] * ww * J[c] + J[7 + a] * ww * J[7 + c];
                }
            }
        }
    };

    // pairs still active that fail chi_sq on the stored errors go to level 1; returns this thread's count of them
    auto cut_outliers = [&]() {
        double bad = 0;
        for (int i = gtid; i < n; i += kSim3Stride) {
            if (level[i]) continue;
            const double* e = err + 4 * (size_t)i;
            const double c12 = (double)A.w1[i] * (e[0] * e[0] + e[1] * e[1]);
            const double c21 = (double)A.w2[i] * (e[2] * e[2] + e[3] * e[3]);
            if (A.chi_sq < c12 || A.chi_sq < c21) { level[i] = 1; bad += 1.0; }
        }
        return bad;
    };

    // round 0: num_first_iter iterations and the outlier cut; fewer than 10 pairs left: return 0, g2o_Sim3_12 untouched.
    // round 1: num_iter iterations and the outlier cut.
    int total_iters = 0, total_trials = 0, rounds = 0, num_outliers = 0;
    double last_lambda = 0, last_chi = 0;
    bool success = true;
    for (; rounds < 2 && success; ++rounds) {
        const LmRoundStats r = cluster_lm_round<7, 13>(rounds == 0 ? A.num_first_iter : A.num_iter, s_S, reduce_all, build_local,
                                                       [&](const double* S, const double* x, double* out) {
                                                           ovs::sim3_oplus(S, x, A.fix_scale != 0, out);
                                                       });
        if (r.iterations > 0) {
            if (gtid == 0) A.stats[5 + rounds] = r.lambda_init;
            last_lambda = r.lambda; last_chi = r.chi2;
        }
        if (gtid == 0) A.stats[7 + rounds] = r.iterations;
        total_iters += r.iterations; total_trials += r.trials;
        const double cnt[1] = {cut_outliers()};
        num_outliers += (int)(reduce_all(cnt, 1)[0] + 0.5);
        if (rounds == 0) success = n - num_outliers >= 10;
    }
    const int num_inliers = success ? n - num_outliers : 0;
    double fc[1] = {0};
    for (int i = gtid; i < n; i += kSim3Stride) {
        A.inlier[i] = level[i] ? 0 : 1;
        if (level[i]) continue;
        const double* e = err + 4 * (size_t)i;
        fc[0] += (double)A.w1[i] * (e[0] * e[0] + e[1] * e[1]) + (double)A.w2[i] * (e[2] * e[2] + e[3] * e[3]);
    }
    const double final_chi2 = reduce_all(fc, 1)[0];
    if (gtid == 0) {
        A.stats[0] = total_iters; A.stats[1] = total_trials; A.stats[2] = rounds; A.stats[3] = final_chi2; A.stats[4] = num_inliers;
        A.stats[9] = last_lambda; A.stats[10] = last_chi;
    }
    if (success && gtid < 13) A.sim3[gtid] = s_S[gtid];
}

}  // namespace

extern "C" int ovs_transform_optimize_host(ovs_optimizer* h, const ovs_camera* cam_1, const ovs_camera* cam_2, const double* pose_1w,
                                           const double* pose_2w, int n, const double* pos_w_1, const float* obs_xy_1,
                                           const float* inv_sigma_sq_1, const double* pos_w_2, const float* obs_xy_2,
                                           const float* inv_sigma_sq_2, int fix_scale, float chi_sq, int num_first_iter, int num_iter,
                                           double* sim3_12, uint8_t* inlier_out, int* num_inliers, ovs_ba_stats* stats) {
    OVS_REQUIRE(h && cam_1 && cam_2 && pose_1w && pose_2w && sim3_12 && num_inliers && n >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(n == 0 || (pos_w_1 && obs_xy_1 && inv_sigma_sq_1 && pos_w_2 && obs_xy_2 && inv_sigma_sq_2 && inlier_out),
                OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE((cam_1->model == ovs::kCamPerspective || cam_1->model == ovs::kCamEquirectangular) &&
                (cam_2->model == ovs::kCamPerspective || cam_2->model == ovs::kCamEquirectangular), OVS_ERR_INVALID_ARG, "unknown camera model");
    OVS_REQUIRE(num_first_iter >= 0 && num_iter >= 0, OVS_ERR_INVALID_ARG, "bad iteration counts");
    OVS_REQUIRE(sim3_12[12] > 0.0 && std::isfinite(sim3_12[12]), OVS_ERR_INVALID_ARG, "the Sim3 scale must be positive");
    OVS_REQUIRE(chi_sq > 0.0f && std::isfinite(chi_sq), OVS_ERR_INVALID_ARG, "chi_sq must be positive");
    if (stats) memset(stats, 0, sizeof(*stats));
    for (int i = 0; i < n; ++i) inlier_out[i] = 0;
    *num_inliers = 0;
    if (n == 0) return OVS_OK;   // fewer than 10 pairs can survive: the reference returns 0 and leaves g2o_Sim3_12 as it is
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // carved from the same arenas as the pose optimiser: a prepared local-BA problem on this handle is gone
    invalidate_plan(h);
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(h->stream)); h->pending = false; }
    const size_t N = (size_t)n;
    Sim3OptArgs A;
    double *hp1, *hp2, *hS, *hstats, *derr; float *hxy1, *hw1, *hxy2, *hw2; uint8_t *hout, *dlevel;
    ovs::Staging S;
    const int rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        A.pw1 = S.in(hp1, 3 * N); A.xy1 = (const float2*)S.in(hxy1, 2 * N); A.w1 = S.in(hw1, N);
        A.pw2 = S.in(hp2, 3 * N); A.xy2 = (const float2*)S.in(hxy2, 2 * N); A.w2 = S.in(hw2, N);
        A.sim3 = S.io(hS, 13); A.stats = S.io(hstats, 16); A.inlier = S.out(hout, N);
        derr = S.dev<double>(4 * N); dlevel = S.dev<uint8_t>(N);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hp1, pos_w_1, 24 * N); memcpy(hxy1, obs_xy_1, 8 * N); memcpy(hw1, inv_sigma_sq_1, 4 * N);
    memcpy(hp2, pos_w_2, 24 * N); memcpy(hxy2, obs_xy_2, 8 * N); memcpy(hw2, inv_sigma_sq_2, 4 * N);
    memcpy(hS, sim3_12, 13 * 8);
    memset(hstats, 0, 128);
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    A.cam1 = to_cam(cam_1); A.cam2 = to_cam(cam_2);
    memcpy(A.pose1, pose_1w, 96); memcpy(A.pose2, pose_2w, 96);
    A.n = n;
    A.fix_scale = fix_scale ? 1 : 0; A.num_first_iter = num_first_iter; A.num_iter = num_iter;
    A.delta = (double)sqrtf(chi_sq); A.chi_sq = (double)chi_sq;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    k_sim3_optimize<<<kSim3Cluster, kSim3Threads, 0, st>>>(A, derr, dlevel);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(sim3_12, hS, 13 * 8);     // the device wrote it back only on success: otherwise these are the input bits
    memcpy(inlier_out, hout, N);
    *num_inliers = (int)hstats[4];
    if (stats) {
        stats->num_iterations = (int)hstats[0]; stats->num_trials = (int)hstats[1]; stats->num_rounds = (int)hstats[2];
        stats->final_chi2 = hstats[3];
        for (int r = 0; r < 2 && r < stats->num_rounds; ++r) {
            stats->lambda_init[r] = hstats[5 + r];
            stats->round_iterations[r] = (int)hstats[7 + r];
        }
        stats->last_lambda = hstats[9]; stats->last_chi2 = hstats[10];
        float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
        stats->device_us = ms * 1000.f;
    }
    return OVS_OK;
}

// ----------------------------------------------------------------------- Sim3 RANSAC solver
namespace {

constexpr int kRansacWarps = 4;                      // hypotheses per CTA, one warp each
constexpr int kRansacThreads = 32 * kRansacWarps;
constexpr int kRansacPrepThreads = 256;

struct RansacArgs {
    int B, N, fix_scale, min_num_inliers, max_num_iter;
    const int* off;                                  // B + 1 pair offsets
    const CameraD* cam1; const CameraD* cam2;        // B each
    const double* pose1; const double* pose2;        // B x 12, {R row-major, t}
    const double* pw1; const float* sig1; const double* pw2; const float* sig2;   // per pair
    const uint64_t* seed;                            // B
    unsigned long long* key;                         // B, zero on entry: max over hypotheses of (count << 32) | ~k
    unsigned* done;                                  // B, zero on entry: CTAs of the problem that have finished scoring
    double* pc1; double* pc2; double* rp1; double* rp2; float* bd1; float* bd2;   // per pair, written by k_sim3_ransac_prep
    double* sim3; int* num_inliers; int* best_iter; uint8_t* valid; uint8_t* inlier;  // out
};

// One thread per pair: the points in their keyframes' camera frames, their own reprojections and the two bounds
// (ransac_bound: -1 where the own reprojection does not exist).
__global__ void __launch_bounds__(kRansacPrepThreads) k_sim3_ransac_prep(RansacArgs A) {
    const int g = blockIdx.x * kRansacPrepThreads + threadIdx.x;
    if (g >= A.N) return;
    int lo = 0, hi = A.B;                            // the largest b with off[b] <= g (empty problems precede it)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (A.off[mid] <= g) lo = mid; else hi = mid;
    }
    const int b = lo;
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
#pragma unroll 1
    for (int side = 0; side < 2; ++side) {
        const double* pose = (side == 0 ? A.pose1 : A.pose2) + 12 * (size_t)b;
        const double* pwp = (side == 0 ? A.pw1 : A.pw2) + 3 * (size_t)g;
        const double pw[3] = {pwp[0], pwp[1], pwp[2]};
        double pc[3], uv[2] = {0.0, 0.0};
        ovs::mat3_vec(pose, pw, pc);
        pc[0] += pose[9]; pc[1] += pose[10]; pc[2] += pose[11];
        const bool ok = ovs::ransac_reproject(side == 0 ? A.cam1[b] : A.cam2[b], I, zero, pc, uv);
        double* pco = (side == 0 ? A.pc1 : A.pc2) + 3 * (size_t)g;
        double* rpo = (side == 0 ? A.rp1 : A.rp2) + 2 * (size_t)g;
        pco[0] = pc[0]; pco[1] = pc[1]; pco[2] = pc[2];
        rpo[0] = ok ? uv[0] : 0.0; rpo[1] = ok ? uv[1] : 0.0;
        (side == 0 ? A.bd1 : A.bd2)[g] = ovs::ransac_bound((side == 0 ? A.sig1 : A.sig2)[g], ok);
    }
}

// Hypothesis k of problem b (pairs o .. o + n - 1): its triple, S_12 and S_21.
__device__ void ransac_hypothesis(const RansacArgs& A, int b, int o, int n, int k, double* S12, double* S21) {
    int idx[3];
    ovs::sim3_ransac_triple(A.seed[b], k, n, idx);
    double p1[9], p2[9];
    for (int j = 0; j < 3; ++j)
        for (int c = 0; c < 3; ++c) {
            p1[3 * j + c] = A.pc1[3 * (size_t)(o + idx[j]) + c];
            p2[3 * j + c] = A.pc2[3 * (size_t)(o + idx[j]) + c];
        }
    ovs::sim3_horn(p1, p2, A.fix_scale != 0, S12, S21);
}

__device__ __forceinline__ bool ransac_pair(const RansacArgs& A, const CameraD& c1, const CameraD& c2, const double* sR12,
                                            const double* S12, const double* sR21, const double* S21, size_t i) {
    const double pc1[3] = {A.pc1[3 * i], A.pc1[3 * i + 1], A.pc1[3 * i + 2]};
    const double pc2[3] = {A.pc2[3 * i], A.pc2[3 * i + 1], A.pc2[3 * i + 2]};
    const double r1[2] = {A.rp1[2 * i], A.rp1[2 * i + 1]}, r2[2] = {A.rp2[2 * i], A.rp2[2 * i + 1]};
    return ovs::ransac_is_inlier(c1, c2, sR12, S12 + 9, sR21, S21 + 9, pc1, pc2, r1, r2, A.bd1[i], A.bd2[i]);
}

// find_via_ransac for every problem of the batch in one launch: grid (hypothesis blocks, problems), one warp per hypothesis
// (every lane forms the same S_12; the lanes then take the pairs with a stride of 32 and count by ballot).  The best hypothesis is
// the integer maximum of (count << 32) | ~k over the problem (atomicMax: order-independent), so the first of the hypotheses with
// the most inliers wins, as in the reference's sequential loop; a hypothesis with no inlier is never best.  The last CTA of a
// problem to finish writes S_12, the count, k, valid and the best hypothesis's inlier flags.
__global__ void __launch_bounds__(kRansacThreads) k_sim3_ransac(RansacArgs A) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const bool runs = n >= 3 && n >= A.min_num_inliers;
    const CameraD c1 = A.cam1[b], c2 = A.cam2[b];
    const int k = blockIdx.x * kRansacWarps + warp;
    if (runs && k < A.max_num_iter) {
        double S12[13], S21[13], sR12[9], sR21[9];
        ransac_hypothesis(A, b, o, n, k, S12, S21);
        ovs::sim3_scaled_rotation(S12, sR12);
        ovs::sim3_scaled_rotation(S21, sR21);
        const unsigned cnt = ovs::warp_count(n, lane, [&](int i) { return ransac_pair(A, c1, c2, sR12, S12, sR21, S21, (size_t)(o + i)); });
        if (lane == 0 && cnt > 0) {
            atomicMax(&A.key[b], ovs::best_key(cnt, k));
            __threadfence();
        }
    }
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(&A.done[b], 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    unsigned cnt;
    const int best = ovs::best_of_key(atomicOr(&A.key[b], 0ull), &cnt);
    double S12[13], S21[13];
    if (best >= 0) {
        double sR12[9], sR21[9];
        ransac_hypothesis(A, b, o, n, best, S12, S21);
        ovs::sim3_scaled_rotation(S12, sR12);
        ovs::sim3_scaled_rotation(S21, sR21);
        for (int i = threadIdx.x; i < n; i += kRansacThreads)
            A.inlier[o + i] = ransac_pair(A, c1, c2, sR12, S12, sR21, S21, (size_t)(o + i)) ? 1 : 0;
    } else {
        for (int m = 0; m < 13; ++m) S12[m] = (m == 0 || m == 4 || m == 8 || m == 12) ? 1.0 : 0.0;
        for (int i = threadIdx.x; i < n; i += kRansacThreads) A.inlier[o + i] = 0;
    }
    if (threadIdx.x < 13) A.sim3[13 * (size_t)b + threadIdx.x] = S12[threadIdx.x];
    if (threadIdx.x == 0) {
        A.num_inliers[b] = (int)cnt;
        A.best_iter[b] = best;
        A.valid[b] = (runs && (int)cnt >= A.min_num_inliers) ? 1 : 0;
    }
}

}  // namespace

extern "C" int ovs_sim3_solve_ransac_host(ovs_optimizer* h, int B, const int32_t* pair_offsets, const ovs_camera* cam_1,
                                          const double* pose_1w, const ovs_camera* cam_2, const double* pose_2w, const double* pos_w_1,
                                          const float* sigma_sq_1, const double* pos_w_2, const float* sigma_sq_2, int fix_scale,
                                          int min_num_inliers, int max_num_iter, const uint64_t* seeds, double* sim3_12, uint8_t* valid,
                                          int32_t* num_inliers, int32_t* best_iter, uint8_t* inlier_out) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(min_num_inliers >= 0 && max_num_iter >= 0, OVS_ERR_INVALID_ARG, "min_num_inliers and max_num_iter must not be negative");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(pair_offsets && cam_1 && pose_1w && cam_2 && pose_2w && seeds && sim3_12 && valid && num_inliers && best_iter,
                OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    for (int b = 0; b < B; ++b)
        if (!((cam_1[b].model == ovs::kCamPerspective || cam_1[b].model == ovs::kCamEquirectangular) &&
              (cam_2[b].model == ovs::kCamPerspective || cam_2[b].model == ovs::kCamEquirectangular))) {
            // problem by problem, the offsets up to problem b are checked before its cameras
            if ((rc = ovs::check_offsets(pair_offsets, b + 1, "pair_offsets")) != OVS_OK) return rc;
            OVS_REQUIRE(false, OVS_ERR_INVALID_ARG, "unknown camera model (problem %d)", b);
        }
    if ((rc = ovs::check_offsets(pair_offsets, B, "pair_offsets")) != OVS_OK) return rc;
    const int n_all = pair_offsets[B];
    OVS_REQUIRE(n_all == 0 || (pos_w_1 && sigma_sq_1 && pos_w_2 && sigma_sq_2 && inlier_out), OVS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n_all; ++i)
        OVS_REQUIRE(sigma_sq_1[i] > 0.0f && std::isfinite(sigma_sq_1[i]) && sigma_sq_2[i] > 0.0f && std::isfinite(sigma_sq_2[i]),
                    OVS_ERR_INVALID_ARG, "sigma_sq of pair %d must be positive and finite", i);
    if (n_all == 0) {   // every problem has fewer than 3 pairs: no hypothesis, invalid
        for (int b = 0; b < B; ++b) {
            for (int m = 0; m < 13; ++m) sim3_12[13 * (size_t)b + m] = (m == 0 || m == 4 || m == 8 || m == 12) ? 1.0 : 0.0;
            valid[b] = 0; num_inliers[b] = 0; best_iter[b] = -1;
        }
        return OVS_OK;
    }
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // carved from the same arenas as the pose optimiser: a prepared local-BA problem on this handle is gone
    invalidate_plan(h);
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(h->stream)); h->pending = false; }
    const size_t N = (size_t)n_all, NB = (size_t)B;
    RansacArgs A;
    A.B = B; A.N = n_all; A.fix_scale = fix_scale ? 1 : 0; A.min_num_inliers = min_num_inliers; A.max_num_iter = max_num_iter;
    int* hoff; CameraD *hc1, *hc2; double *hp1, *hp2, *hw1, *hw2; float *hs1, *hs2; uint64_t* hseed; unsigned long long* hkey; unsigned* hdone;
    double* hS; int *hnum, *hbest; uint8_t *hvalid, *hflags;
    ovs::Staging S;
    rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        A.off = S.in(hoff, NB + 1); A.cam1 = S.in(hc1, NB); A.cam2 = S.in(hc2, NB);
        A.pose1 = S.in(hp1, 12 * NB); A.pose2 = S.in(hp2, 12 * NB);
        A.pw1 = S.in(hw1, 3 * N); A.sig1 = S.in(hs1, N); A.pw2 = S.in(hw2, 3 * N); A.sig2 = S.in(hs2, N);
        A.seed = S.in(hseed, NB); A.key = S.in(hkey, NB); A.done = S.in(hdone, NB);
        A.sim3 = S.out(hS, 13 * NB); A.num_inliers = S.out(hnum, NB); A.best_iter = S.out(hbest, NB); A.valid = S.out(hvalid, NB);
        A.inlier = S.out(hflags, N);
        A.pc1 = S.dev<double>(3 * N); A.pc2 = S.dev<double>(3 * N); A.rp1 = S.dev<double>(2 * N); A.rp2 = S.dev<double>(2 * N);
        A.bd1 = S.dev<float>(N); A.bd2 = S.dev<float>(N);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hoff, pair_offsets, 4 * (NB + 1));
    for (int b = 0; b < B; ++b) { hc1[b] = to_cam(&cam_1[b]); hc2[b] = to_cam(&cam_2[b]); }
    memcpy(hp1, pose_1w, 96 * NB); memcpy(hp2, pose_2w, 96 * NB);
    memcpy(hw1, pos_w_1, 24 * N); memcpy(hs1, sigma_sq_1, 4 * N); memcpy(hw2, pos_w_2, 24 * N); memcpy(hs2, sigma_sq_2, 4 * N);
    memcpy(hseed, seeds, 8 * NB); memset(hkey, 0, 8 * NB); memset(hdone, 0, 4 * NB);
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    k_sim3_ransac_prep<<<(n_all + kRansacPrepThreads - 1) / kRansacPrepThreads, kRansacPrepThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    const int hyp_blocks = max_num_iter > 0 ? (max_num_iter + kRansacWarps - 1) / kRansacWarps : 1;
    k_sim3_ransac<<<dim3(hyp_blocks, B), kRansacThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(sim3_12, hS, 13 * 8 * NB);
    memcpy(num_inliers, hnum, 4 * NB); memcpy(best_iter, hbest, 4 * NB); memcpy(valid, hvalid, NB);
    memcpy(inlier_out, hflags, N);
    return OVS_OK;
}

// ----------------------------------------------------------------------- PnP RANSAC solver
namespace {

constexpr int kPnpHypThreads = 64;                   // k_pnp_hypotheses: one thread per hypothesis (and per correspondence)
constexpr int kPnpWarps = 4;                         // k_pnp_ransac: hypotheses per CTA, one warp each
constexpr int kPnpThreads = 32 * kPnpWarps;
constexpr int kPnpRefineThreads = ovs::kBlockSumThreads;   // k_pnp_refine: one CTA per problem, one thread per partial sum
constexpr int kPnpChunk = ovs::kBlockSumChunk;       // components reduced per pass of the CTA-wide sum

struct PnpArgs {
    int B, N, H, min_num_inliers, recompute;
    const int* off;                                  // B + 1 correspondence offsets
    const double* bear; const double* pw; const float* sf;   // per correspondence
    const uint64_t* seed;                            // B
    unsigned long long* key;                         // B, zero on entry: max over hypotheses of (count << 32) | ~k
    double* bound;                                   // per correspondence: max_cos_error, written by k_pnp_hypotheses
    double* hyp;                                     // B x H x 12: every hypothesis's pose
    int* cidx;                                       // per correspondence: the best hypothesis's inliers, compacted per problem
    double* pose; int* num_inliers; int* best_iter; uint8_t* valid; uint8_t* inlier;   // out
};

__device__ __forceinline__ bool pnp_runs(const PnpArgs& A, int n) { return n >= ovs::kPnpMinSet && n >= A.min_num_inliers; }

__device__ __forceinline__ bool pnp_corr(const PnpArgs& A, const double* pose, size_t i) {
    const double pw[3] = {A.pw[3 * i], A.pw[3 * i + 1], A.pw[3 * i + 2]};
    const double b[3] = {A.bear[3 * i], A.bear[3 * i + 1], A.bear[3 * i + 2]};
    return ovs::pnp_is_inlier(pose, pw, b, A.bound[i]);
}

// One thread per (problem, hypothesis): the minimal set of the counter-based sampler and its EPnP pose.  The first N threads
// also form the correspondences' bounds.
__global__ void __launch_bounds__(kPnpHypThreads) k_pnp_hypotheses(PnpArgs A) {
    const size_t g = (size_t)blockIdx.x * kPnpHypThreads + threadIdx.x;
    if (g < (size_t)A.N) A.bound[g] = ovs::pnp_max_cos(A.sf[g]);
    if (A.H == 0 || g >= (size_t)A.B * (size_t)A.H) return;
    const int b = (int)(g / (size_t)A.H), k = (int)(g % (size_t)A.H);
    const int o = A.off[b], n = A.off[b + 1] - o;
    if (!pnp_runs(A, n)) return;
    int idx[ovs::kPnpMinSet];
    ovs::ransac_sample<ovs::kPnpMinSet>(A.seed[b], k, n, idx);
    const ovs::PnpPoints P{A.pw + 3 * (size_t)o, A.bear + 3 * (size_t)o, idx, ovs::kPnpMinSet};
    ovs::epnp_pose(P, ovs::PnpSeqSum{ovs::kPnpMinSet}, A.hyp + 12 * g);
}

// check_inliers of every hypothesis: grid (hypothesis blocks, problems), one warp per hypothesis, the lanes take the
// correspondences with a stride of 32 and count by ballot.  The best hypothesis is the integer maximum of (count << 32) | ~k
// (atomicMax: order-independent), so the first of the hypotheses with the most inliers wins, as in the sequential loop; a
// hypothesis with no inlier is never best.
__global__ void __launch_bounds__(kPnpThreads) k_pnp_ransac(PnpArgs A) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const int k = blockIdx.x * kPnpWarps + warp;
    if (!pnp_runs(A, n) || k >= A.H) return;
    const double* hp = A.hyp + 12 * ((size_t)b * A.H + k);
    double pose[12];
    for (int m = 0; m < 12; ++m) pose[m] = hp[m];
    const unsigned cnt = ovs::warp_count(n, lane, [&](int i) { return pnp_corr(A, pose, (size_t)(o + i)); });
    if (lane == 0 && cnt > 0) atomicMax(&A.key[b], ovs::best_key(cnt, k));
}

// pnp_sum across the CTA (block_sum.cuh): same bits as PnpSeqSum.
using ovs::PnpBlockSum;

// One CTA per problem: the best hypothesis (or none), its inlier flags, `valid`, and with recompute (valid and at least
// kPnpMinSet inliers) EPnP on the compacted inliers with the CTA-wide sums and the flags re-checked at that pose.
__global__ void __launch_bounds__(kPnpRefineThreads) k_pnp_refine(PnpArgs A) {
    __shared__ double s_red[kPnpChunk * kPnpRefineThreads];
    __shared__ double s_res[78];
    __shared__ int s_warp[kPnpRefineThreads / 32];
    const int b = blockIdx.x, t = threadIdx.x;
    const int o = A.off[b], n = A.off[b + 1] - o;
    const bool runs = pnp_runs(A, n);
    unsigned cnt;
    const int best = ovs::best_of_key(A.key[b], &cnt);
    double pose[12];
    if (best >= 0) {
        const double* hp = A.hyp + 12 * ((size_t)b * A.H + best);
        for (int m = 0; m < 12; ++m) pose[m] = hp[m];
    } else {
        ovs::pnp_identity(pose);
    }
    for (int i = t; i < n; i += kPnpRefineThreads) A.inlier[o + i] = (best >= 0 && pnp_corr(A, pose, (size_t)(o + i))) ? 1 : 0;
    const bool valid = runs && (int)cnt >= A.min_num_inliers;
    int num = (int)cnt;
    if (valid && A.recompute && best >= 0 && (int)cnt >= ovs::kPnpMinSet) {
        ovs::cta_compact<kPnpRefineThreads>(n, A.cidx + o, s_warp, [&](int i) { return pnp_corr(A, pose, (size_t)(o + i)); });
        const ovs::PnpPoints P{A.pw + 3 * (size_t)o, A.bear + 3 * (size_t)o, A.cidx + o, (int)cnt};
        double np[12];
        ovs::epnp_pose(P, PnpBlockSum{(int)cnt, s_red, s_res}, np);
        for (int m = 0; m < 12; ++m) pose[m] = np[m];
        int c2 = 0;
        for (int base = 0; base < n; base += kPnpRefineThreads) {
            const int i = base + t;
            const bool f = i < n && pnp_corr(A, pose, (size_t)(o + i));
            if (i < n) A.inlier[o + i] = f ? 1 : 0;
            c2 += __syncthreads_count(f);
        }
        num = c2;
    }
    if (t < 12) A.pose[12 * (size_t)b + t] = pose[t];
    if (t == 0) {
        A.num_inliers[b] = num;
        A.best_iter[b] = best;
        A.valid[b] = valid ? 1 : 0;
    }
}

}  // namespace

extern "C" int ovs_pnp_solve_ransac_host(ovs_optimizer* h, int B, const int32_t* corr_offsets, const double* bearings,
                                         const double* pos_w, const float* scale_factor, int min_num_inliers, int max_num_iter,
                                         int recompute, const uint64_t* seeds, double* pose_cw, uint8_t* valid, int32_t* num_inliers,
                                         int32_t* best_iter, uint8_t* inlier_out) {
    OVS_REQUIRE(h && B >= 0 && B <= 65535, OVS_ERR_INVALID_ARG, "bad argument (B must be in 0 .. 65535)");
    OVS_REQUIRE(min_num_inliers >= 0 && max_num_iter >= 0, OVS_ERR_INVALID_ARG, "min_num_inliers and max_num_iter must not be negative");
    if (B == 0) return OVS_OK;
    OVS_REQUIRE(corr_offsets && seeds && pose_cw && valid && num_inliers && best_iter, OVS_ERR_INVALID_ARG, "null argument");
    int rc;
    if ((rc = ovs::check_offsets(corr_offsets, B, "corr_offsets")) != OVS_OK) return rc;
    const int n_all = corr_offsets[B];
    OVS_REQUIRE(n_all == 0 || (bearings && pos_w && scale_factor && inlier_out), OVS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n_all; ++i) {
        const double* p = pos_w + 3 * (size_t)i;
        const double* v = bearings + 3 * (size_t)i;
        OVS_REQUIRE(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]), OVS_ERR_INVALID_ARG,
                    "pos_w of correspondence %d is not finite", i);
        OVS_REQUIRE(std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]) &&
                    std::fabs(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] - 1.0) <= 1e-6,
                    OVS_ERR_INVALID_ARG, "bearing of correspondence %d is not a finite unit vector", i);
        OVS_REQUIRE(scale_factor[i] > 0.0f && scale_factor[i] <= 90.0f, OVS_ERR_INVALID_ARG,
                    "scale_factor of correspondence %d must be in (0, 90]", i);
    }
    if (n_all == 0) {   // no correspondence at all: no hypothesis, invalid
        for (int b = 0; b < B; ++b) {
            ovs::pnp_identity(pose_cw + 12 * (size_t)b);
            valid[b] = 0; num_inliers[b] = 0; best_iter[b] = -1;
        }
        return OVS_OK;
    }
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // carved from the same arenas as the pose optimiser: a prepared local-BA problem on this handle is gone
    invalidate_plan(h);
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(h->stream)); h->pending = false; }
    const size_t N = (size_t)n_all, NB = (size_t)B, H = (size_t)max_num_iter;
    PnpArgs A;
    A.B = B; A.N = n_all; A.H = max_num_iter; A.min_num_inliers = min_num_inliers; A.recompute = recompute ? 1 : 0;
    int* hoff; double *hbear, *hpw; float* hsf; uint64_t* hseed; unsigned long long* hkey;
    double* hpose; int *hnum, *hbest; uint8_t *hvalid, *hflags;
    ovs::Staging S;
    rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        A.off = S.in(hoff, NB + 1);
        A.bear = S.in(hbear, 3 * N); A.pw = S.in(hpw, 3 * N); A.sf = S.in(hsf, N);
        A.seed = S.in(hseed, NB); A.key = S.in(hkey, NB);
        A.pose = S.out(hpose, 12 * NB); A.num_inliers = S.out(hnum, NB); A.best_iter = S.out(hbest, NB); A.valid = S.out(hvalid, NB);
        A.inlier = S.out(hflags, N);
        A.bound = S.dev<double>(N); A.cidx = S.dev<int>(N); A.hyp = S.dev<double>(12 * NB * H);
    });
    if (rc != OVS_OK) return rc;
    memcpy(hoff, corr_offsets, 4 * (NB + 1));
    memcpy(hbear, bearings, 24 * N); memcpy(hpw, pos_w, 24 * N); memcpy(hsf, scale_factor, 4 * N);
    memcpy(hseed, seeds, 8 * NB); memset(hkey, 0, 8 * NB);
    cudaStream_t st = h->stream;
    OVS_CUDA_CHECK(S.upload(st));
    const size_t hyp_threads = std::max(N, NB * H);
    k_pnp_hypotheses<<<(unsigned)((hyp_threads + kPnpHypThreads - 1) / kPnpHypThreads), kPnpHypThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    if (max_num_iter > 0) {
        k_pnp_ransac<<<dim3((max_num_iter + kPnpWarps - 1) / kPnpWarps, B), kPnpThreads, 0, st>>>(A);
        OVS_LAUNCH_CHECK();
    }
    k_pnp_refine<<<B, kPnpRefineThreads, 0, st>>>(A);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(S.download(st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    memcpy(pose_cw, hpose, 12 * 8 * NB);
    memcpy(num_inliers, hnum, 4 * NB); memcpy(best_iter, hbest, 4 * NB); memcpy(valid, hvalid, NB);
    memcpy(inlier_out, hflags, N);
    return OVS_OK;
}

// ------------------------------------------------------------------- local bundle adjuster
// The call is split in three phases so that a prepared problem can be re-run with everything
// resident in HBM: prepare (graph bookkeeping + upload + co-observation lists), run (the two
// Levenberg rounds, device state), fetch (download).  ovs_local_ba_host = prepare + run + fetch.
// prepare enqueues and returns (one host->device copy, no synchronisation); run enqueues the whole static launch
// sequence of both rounds and waits once; fetch is one device->host copy.
struct ovs_ba_plan {
    bool valid = false;
    BaDev P{};
    int K = 0, L = 0, M = 0, nfree = 0, n = 0, npairs = 0, nb_obs = 0, nb_upd = 0;
    long long npair_entries = 0;
    size_t chol_smem = 0;
    int chol_dbuf = 0, chol_big = 0;
    // host (pinned) views
    double* hposes = nullptr; double* hpoints = nullptr; uint8_t* hout = nullptr;
    LmCtl* hctl = nullptr; int* hexec = nullptr; int exec_cap = 0;
    // device
    double *dposes_in = nullptr, *dpoints_in = nullptr;      // uploaded initial estimates
    double *dposes_ring = nullptr, *dpoints_ring = nullptr;   // kSpec + 1 buffers each: the current estimate + kSpec candidates
    uint8_t* dlevel = nullptr; double* derr = nullptr;        // derr: kSpec x M x 3 (edge errors of each speculative trial)
    uint8_t* dout = nullptr;
    LmCtl* dctl = nullptr; int* dexec = nullptr;
    size_t spart_stride = 0, S_stride = 0, invL_stride = 0;
    int rows = 2;                                               // rows of the edge records: 3 if any edge is stereo
    double* drec = nullptr;                                     // M edge records (EdgeRec<rows>)
    int4* dlblocks = nullptr; int* dnlblocks = nullptr; int nlseg = 0;   // landmark block table of the linearisation (per segment)
    double *dHll = nullptr, *dbl = nullptr, *dHpp = nullptr, *dbp = nullptr;
    double *dS = nullptr, *dbS = nullptr, *dx = nullptr, *dinvL = nullptr;
    int4* d_pair_rec = nullptr; int *dsegb = nullptr, *dsege = nullptr; int2* dpab = nullptr; int* ddiag = nullptr;
    int4 *dchunks = nullptr, *ddchunks = nullptr; int *dpair_chunk_begin = nullptr, *dkf_chunk_begin = nullptr;
    int* dnchunks = nullptr;                                    // [0] chunks of the Schur stage, [1] chunks of the Hpp stage
    double *dspart = nullptr, *dppart = nullptr; int max_chunks = 0, max_dchunks = 0;
    double *dpchi = nullptr, *dpscale = nullptr; int* dfail = nullptr; double* dmaxdiag = nullptr;
    int cur = 0;   // index of the buffer holding the current estimate after run
};

namespace {

// The dense FP64 solver of one trial batch: kSpec systems (n + 1) x n (lower triangle + rhs row, S_stride apart), factorised in
// place, solutions to x (n apart).  The cluster kernel up to the shared-memory panel limit, the multi-launch path above it.
struct DenseSolve {
    double* S; size_t S_stride; int n; double* x; double* invL; size_t invL_stride; int* fail;
    int chol_big, chol_dbuf; size_t chol_smem;
};

// chol_big / chol_dbuf / chol_smem for an n x n system
void dense_solve_config(int n, DenseSolve& ds) {
    // forward phase: the panel; backward phase: one or (if it fits) two (inverse block, row block) buffers
    const size_t fixed = chol_fixed_doubles(n), panel = chol_panel_doubles(n), back = chol_back_doubles(n) - 32 * 33;
    const size_t one = (fixed + std::max(panel, back)) * sizeof(double);
    const size_t two = (fixed + std::max(panel, back + chol_back_doubles(n))) * sizeof(double);
    ds.chol_big = one > (size_t)kCholMaxDynSmem ? 1 : 0;   // panel does not fit: multi-launch fallback (k_chol_big_*)
    ds.chol_dbuf = two <= (size_t)kCholMaxDynSmem ? 1 : 0;
    ds.chol_smem = ds.chol_big ? 0 : (ds.chol_dbuf ? two : one);
}

struct BaInputs {   // all host pointers, or all device pointers (obs_x_right may be null)
    const double* poses; const uint8_t* fixed; const double* points; const int32_t* obs_kf; const int32_t* obs_lm;
    const float* obs_xy; const float* obs_x_right; const float* inv_sigma_sq;
};

// prepare = upload (or device-to-device copy) of the graph, bookkeeping kernels, ONE small read-back (the counts that size
// the work buffers; it also carries the validation verdict), co-observation lists and chunk tables.  Returns with the
// remaining work enqueued.
int prepare_impl(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, int L, int M, const BaInputs& in, bool on_device) {
    OVS_REQUIRE(h && cam && K > 0 && L > 0 && M > 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(in.poses && in.fixed && in.points && in.obs_kf && in.obs_lm && in.obs_xy && in.inv_sigma_sq, OVS_ERR_INVALID_ARG, "null argument");
    OVS_REQUIRE(cam->model == ovs::kCamPerspective || cam->model == ovs::kCamEquirectangular, OVS_ERR_INVALID_ARG, "unknown camera model");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    ovs_ba_plan& pl = *h->plan;
    pl.valid = false;
    cudaStream_t st = h->stream;
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(st)); h->pending = false; }   // the arenas are about to be rewritten

    // ---- phase 1: everything whose size follows from K, L, M (inputs, index arrays, per-edge / per-landmark state)
    const size_t sM = (size_t)M, sL = (size_t)L, sK = (size_t)K;
    const int nb_obs = (M + 127) / 128, nb_upd = (L + K + 127) / 128;
    const int exec_cap = 1024;
    const int nlseg = M / kLbSegEdges + 1;           // k_ba_landmark_blocks: segments of the landmark block table
    double* hposes; double* hpoints; int *hkf, *hlm; float *hxy, *hxr, *hw; uint8_t* hfixed; uint8_t* hout; long long* hcounts;
    double* dposes_in; double* dpoints_in; int *dkf, *dlm; float *dxy, *dxr, *dw; uint8_t* dfixed;
    int *dfree, *dlmf, *dpoff; long long* dcounts;
    ovs::Staging S;
    int rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        dposes_in = S.in(hposes, 12 * sK); dpoints_in = S.in(hpoints, 3 * sL);
        dkf = S.in(hkf, sM); dlm = S.in(hlm, sM); dxy = S.in(hxy, 2 * sM); dxr = S.in(hxr, sM); dw = S.in(hw, sM);
        dfixed = S.in(hfixed, sK);
        // each read back by its own copy: the flags by fetch, the control block and solver slots by run, the counts below
        pl.dout = S.out(hout, sM); pl.dctl = S.out(pl.hctl, 1); pl.dexec = S.out(pl.hexec, exec_cap); dcounts = S.out(hcounts, 8);
        dfree = S.dev<int>(sK); dlmf = S.dev<int>(sL + 1); dpoff = S.dev<int>(sL + 1);
        pl.dposes_ring = S.dev<double>((kSpec + 1) * 12 * sK); pl.dpoints_ring = S.dev<double>((kSpec + 1) * 3 * sL);
        pl.dlevel = S.dev<uint8_t>(sM); pl.derr = S.dev<double>(kSpec * 3 * sM);
        pl.dlblocks = S.dev<int4>((size_t)nlseg * kLbSegCap); pl.dnlblocks = S.dev<int>(nlseg);
        pl.dHll = S.dev<double>(6 * sL); pl.dbl = S.dev<double>(3 * sL);
        pl.dpchi = S.dev<double>(kSpec * (size_t)nb_obs); pl.dpscale = S.dev<double>(kSpec * (size_t)nb_upd);
        pl.dfail = S.dev<int>(kSpec); pl.dmaxdiag = S.dev<double>(2); pl.dnchunks = S.dev<int>(2);
    });
    if (rc != OVS_OK) return rc;
    pl.exec_cap = exec_cap;
    h->pending = true;
    if (!on_device) {
        memcpy(hposes, in.poses, 96 * sK); memcpy(hpoints, in.points, 24 * sL);
        memcpy(hkf, in.obs_kf, 4 * sM); memcpy(hlm, in.obs_lm, 4 * sM); memcpy(hxy, in.obs_xy, 8 * sM); memcpy(hw, in.inv_sigma_sq, 4 * sM);
        if (in.obs_x_right) memcpy(hxr, in.obs_x_right, 4 * sM); else for (size_t i = 0; i < sM; ++i) hxr[i] = -1.0f;
        memcpy(hfixed, in.fixed, sK);
        OVS_CUDA_CHECK(S.upload(st));
    } else {
        const cudaMemcpyKind dd = cudaMemcpyDeviceToDevice;
        OVS_CUDA_CHECK(cudaMemcpyAsync(dposes_in, in.poses, 96 * sK, dd, st)); OVS_CUDA_CHECK(cudaMemcpyAsync(dpoints_in, in.points, 24 * sL, dd, st));
        OVS_CUDA_CHECK(cudaMemcpyAsync(dkf, in.obs_kf, 4 * sM, dd, st)); OVS_CUDA_CHECK(cudaMemcpyAsync(dlm, in.obs_lm, 4 * sM, dd, st));
        OVS_CUDA_CHECK(cudaMemcpyAsync(dxy, in.obs_xy, 8 * sM, dd, st)); OVS_CUDA_CHECK(cudaMemcpyAsync(dw, in.inv_sigma_sq, 4 * sM, dd, st));
        if (in.obs_x_right) OVS_CUDA_CHECK(cudaMemcpyAsync(dxr, in.obs_x_right, 4 * sM, dd, st));
        else { k_fill_f32<<<(unsigned)((sM + 255) / 256), 256, 0, st>>>(dxr, sM, -1.0f); OVS_LAUNCH_CHECK(); }
        OVS_CUDA_CHECK(cudaMemcpyAsync(dfixed, in.fixed, sK, dd, st));
    }
    // graph bookkeeping + validation on the device, then the one read-back of prepare
    hcounts[0] = 0; hcounts[1] = 0; hcounts[2] = 0; hcounts[3] = 0; hcounts[4] = 0x7fffffffffffffffll; hcounts[5] = 0;
    OVS_CUDA_CHECK(cudaMemcpyAsync(dcounts, hcounts, 6 * sizeof(long long), cudaMemcpyHostToDevice, st));
    k_ba_free_index<<<1, 1024, 0, st>>>(K, dfixed, dfree, dcounts);
    OVS_LAUNCH_CHECK();
    k_ba_landmark_index<<<(M + 255) / 256, 256, 0, st>>>(M, L, K, dkf, dlm, dxr, dlmf, dcounts);
    OVS_LAUNCH_CHECK();
    k_ba_pair_counts<<<(L + 255) / 256, 256, 0, st>>>(L, dlmf, dkf, dfree, dpoff, dcounts);
    OVS_LAUNCH_CHECK();
    k_ba_pair_offsets<<<1, 1024, 0, st>>>(L, dpoff, dcounts);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaMemcpyAsync(hcounts, dcounts, 6 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    if (hcounts[4] != 0x7fffffffffffffffll) {
        const long long i = hcounts[4] >> 2;
        const int code = (int)(hcounts[4] & 3);
        h->pending = false;
        if (code == 2) { ovs::set_error("observations must be grouped by landmark (obs_lm non-decreasing; first violation at observation %lld)", i); return OVS_ERR_INVALID_ARG; }
        if (!on_device) ovs::set_error("observation %lld references keyframe %d / landmark %d out of range", i, in.obs_kf[i], in.obs_lm[i]);
        else ovs::set_error("observation %lld references a keyframe / landmark out of range", i);
        return OVS_ERR_INVALID_ARG;
    }
    const int nfree = (int)hcounts[0];
    const long long npair_entries = hcounts[1], nfree_edges = hcounts[2];
    const int n = 6 * nfree;
    OVS_REQUIRE(nfree >= 1, OVS_ERR_INVALID_ARG, "no free keyframe");
    OVS_REQUIRE(n <= kMaxReducedDimBig, OVS_ERR_UNSUPPORTED, "more than %d free keyframes", kMaxReducedDimBig / 6);
    OVS_REQUIRE(npair_entries < (1ll << 30), OVS_ERR_UNSUPPORTED, "too many co-observations");
    const int npairs = nfree * (nfree + 1) / 2;
    const int rows = hcounts[5] ? 3 : 2;
    const size_t rec_doubles = (size_t)(rows == 3 ? EdgeRec<3>::kSize : EdgeRec<2>::kSize) * sM;

    // ---- phase 2: what depends on the number of free keyframes and of co-observations
    const size_t sE = (size_t)std::max<long long>(npair_entries, 1);
    const size_t max_chunks = sE / 128 + (size_t)npairs + 8;                     // ceil(len / 128) summed over the pairs
    const size_t max_dchunks = (size_t)nfree_edges / 128 + (size_t)nfree + 8;   // the same over the diagonal pairs
    unsigned *dkeys, *dkeys2; unsigned long long *dvals, *dvals2; int4* dprec; int* dsort;
    auto carve_work = [&](Arena& W) {
        pl.drec = W.take<double>(rec_doubles);
        pl.dpab = W.take<int2>(npairs); pl.ddiag = W.take<int>(nfree);
        pl.dHpp = W.take<double>(21 * (size_t)nfree); pl.dbp = W.take<double>(6 * (size_t)nfree);
        pl.S_stride = ((size_t)(n + 1) * n + 31) / 32 * 32; pl.invL_stride = (size_t)((n + kNB - 1) / kNB) * kNB * kNB;
        pl.dS = W.take<double>(kSpec * pl.S_stride); pl.dbS = pl.dS + (size_t)n * n; pl.dx = W.take<double>(kSpec * (size_t)n);   // b_S is row n of S
        pl.dinvL = W.take<double>(kSpec * pl.invL_stride);
        dkeys = W.take<unsigned>(sE); dkeys2 = W.take<unsigned>(sE);
        dvals = W.take<unsigned long long>(sE); dvals2 = W.take<unsigned long long>(sE); dprec = W.take<int4>(sE);
        dsort = W.take<int>(sort_scratch_ints((long long)sE));
        pl.dsegb = W.take<int>(npairs); pl.dsege = W.take<int>(npairs);
        pl.dchunks = W.take<int4>(max_chunks); pl.ddchunks = W.take<int4>(max_dchunks);
        pl.dpair_chunk_begin = W.take<int>(npairs + 1); pl.dkf_chunk_begin = W.take<int>(nfree + 1);
        pl.spart_stride = 42 * max_chunks;
        pl.dspart = W.take<double>(kSpec * pl.spart_stride); pl.dppart = W.take<double>(27 * max_dchunks);
    };
    Arena W{nullptr, 0};
    carve_work(W);
    if ((rc = ovs::grow_dev(&h->d_work, &h->w_cap, W.off)) != OVS_OK) return rc;
    W = Arena{h->d_work, 0};
    carve_work(W);
    pl.max_chunks = (int)max_chunks; pl.max_dchunks = (int)max_dchunks;
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.dsegb, 0, 4 * (size_t)npairs, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.dsege, 0, 4 * (size_t)npairs, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.dS, 0, 8 * kSpec * pl.S_stride, st));

    BaDev& P = pl.P;
    P.cam = to_cam(cam); P.K = K; P.L = L; P.M = M; P.nfree = nfree; P.n = n;
    P.poses = dposes_in; P.points = dpoints_in; P.poses_ring = pl.dposes_ring; P.points_ring = pl.dpoints_ring;
    P.obs_kf = dkf; P.obs_lm = dlm; P.obs_xy = (const float2*)dxy; P.obs_xr = dxr; P.inv_sigma_sq = dw;
    P.level = pl.dlevel; P.free_idx = dfree; P.lm_first = dlmf;
    const float chi_sq_2D = 5.99146f, chi_sq_3D = 7.81473f;
    P.use_huber = 1; P.delta = (double)(setup_is_mono ? sqrtf(chi_sq_2D) : sqrtf(chi_sq_3D));

    k_ba_landmark_blocks<<<nlseg, kLbThreads, 0, st>>>(L, dlmf, pl.dlblocks, pl.dnlblocks);
    OVS_LAUNCH_CHECK();

    // ---- co-observation lists, sorted by keyframe pair (stable: landmark order kept inside a pair), flattened to one
    //      16-byte record per co-observation; chunk tables (<= 128 co-observations per chunk) of the two-stage reductions
    k_ba_pair_table<<<nfree, 128, 0, st>>>(nfree, pl.dpab, pl.ddiag);
    OVS_LAUNCH_CHECK();
    pl.d_pair_rec = dprec;
    if (npair_entries > 0) {
        k_ba_emit_pairs<<<(L + 127) / 128, 128, 0, st>>>(P, dpoff, dkeys, dvals);
        OVS_LAUNCH_CHECK();
        int end_bit = 1;
        while ((1 << end_bit) < npairs) ++end_bit;
        unsigned* ksorted = nullptr; unsigned long long* vsorted = nullptr;
        const int src = sort_pairs(st, dkeys, dkeys2, dvals, dvals2, (int)npair_entries, end_bit, dsort, &ksorted, &vsorted);
        if (src != OVS_OK) return src;
        k_ba_segments<<<((int)npair_entries + 255) / 256, 256, 0, st>>>(ksorted, (int)npair_entries, pl.dsegb, pl.dsege);
        OVS_LAUNCH_CHECK();
        k_ba_pair_records<<<((int)npair_entries + 255) / 256, 256, 0, st>>>(vsorted, (int)npair_entries, dlm, dprec);
        OVS_LAUNCH_CHECK();
    }
    k_ba_chunk_scan<<<1, 1024, 0, st>>>(nullptr, npairs, pl.dsegb, pl.dsege, pl.dpair_chunk_begin, pl.dnchunks);
    OVS_LAUNCH_CHECK();
    k_ba_chunk_fill<<<(npairs + 127) / 128, 128, 0, st>>>(nullptr, npairs, pl.dsegb, pl.dsege, pl.dpair_chunk_begin, pl.dchunks);
    OVS_LAUNCH_CHECK();
    k_ba_chunk_scan<<<1, 1024, 0, st>>>(pl.ddiag, nfree, pl.dsegb, pl.dsege, pl.dkf_chunk_begin, pl.dnchunks + 1);
    OVS_LAUNCH_CHECK();
    k_ba_chunk_fill<<<(nfree + 127) / 128, 128, 0, st>>>(pl.ddiag, nfree, pl.dsegb, pl.dsege, pl.dkf_chunk_begin, pl.ddchunks);
    OVS_LAUNCH_CHECK();

    pl.K = K; pl.L = L; pl.M = M; pl.nfree = nfree; pl.n = n; pl.npairs = npairs; pl.nb_obs = nb_obs; pl.nb_upd = nb_upd;
    pl.rows = rows; pl.nlseg = nlseg;
    pl.npair_entries = npair_entries;
    {
        DenseSolve ds{};
        dense_solve_config(n, ds);
        pl.chol_big = ds.chol_big; pl.chol_dbuf = ds.chol_dbuf; pl.chol_smem = ds.chol_smem;
    }
    pl.hposes = hposes; pl.hpoints = hpoints; pl.hout = hout;
    pl.dposes_in = dposes_in; pl.dpoints_in = dpoints_in;
    pl.cur = 0;
    pl.valid = true;
    return OVS_OK;
}

}  // namespace

extern "C" int ovs_local_ba_prepare(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, const double* poses,
                                    const uint8_t* fixed, int L, const double* points, int M, const int32_t* obs_kf,
                                    const int32_t* obs_lm, const float* obs_xy, const float* obs_x_right, const float* inv_sigma_sq) {
    const BaInputs in{poses, fixed, points, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq};
    return prepare_impl(h, cam, setup_is_mono, K, L, M, in, false);
}

extern "C" int ovs_local_ba_prepare_device(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, const double* d_poses,
                                           const uint8_t* d_fixed, int L, const double* d_points, int M, const int32_t* d_obs_kf,
                                           const int32_t* d_obs_lm, const float* d_obs_xy, const float* d_obs_x_right, const float* d_inv_sigma_sq) {
    const BaInputs in{d_poses, d_fixed, d_points, d_obs_kf, d_obs_lm, d_obs_xy, d_obs_x_right, d_inv_sigma_sq};
    return prepare_impl(h, cam, setup_is_mono, K, L, M, in, true);
}

// results of the last run into device buffers of the caller (any may be null)
extern "C" int ovs_local_ba_fetch_device(ovs_optimizer* h, double* d_poses, double* d_points, uint8_t* d_outlier_out) {
    OVS_REQUIRE(h && h->plan->valid, OVS_ERR_INVALID_ARG, "no prepared bundle-adjustment problem");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    ovs_ba_plan& pl = *h->plan;
    cudaStream_t st = h->stream;
    const size_t sK = (size_t)pl.K, sL = (size_t)pl.L, sM = (size_t)pl.M;
    if (d_poses) OVS_CUDA_CHECK(cudaMemcpyAsync(d_poses, pl.dposes_ring + (size_t)pl.cur * 12 * sK, 96 * sK, cudaMemcpyDeviceToDevice, st));
    if (d_points) OVS_CUDA_CHECK(cudaMemcpyAsync(d_points, pl.dpoints_ring + (size_t)pl.cur * 3 * sL, 24 * sL, cudaMemcpyDeviceToDevice, st));
    if (d_outlier_out) OVS_CUDA_CHECK(cudaMemcpyAsync(d_outlier_out, pl.dout, sM, cudaMemcpyDeviceToDevice, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    h->pending = false;
    return OVS_OK;
}

static void invalidate_plan(ovs_optimizer* h) { h->plan->valid = false; }

namespace {

// Waits for the end of the enqueued run.  While waiting the host relays the caller's force_stop_flag to the device-
// visible stop word, which the device-side Levenberg loop polls between trials like g2o's terminate().
int wait_for_run(ovs_optimizer* h, cudaEvent_t done, const volatile uint8_t* force_stop_flag) {
    if (!force_stop_flag) { OVS_CUDA_CHECK(ovs::sync_event(done)); return OVS_OK; }
    const bool blocking = ovs::blocking_waits();
    for (;;) {
        const cudaError_t q = cudaEventQuery(done);
        if (q == cudaSuccess) break;
        if (q != cudaErrorNotReady) OVS_CUDA_CHECK(q);
        if (*force_stop_flag) *(volatile int*)(h->h_mirror + 2) = 1;
        if (blocking) { struct timespec ts = {0, 50000}; nanosleep(&ts, nullptr); } else sched_yield();
    }
    return OVS_OK;
}

int launch_dense_solve(ovs_optimizer* h, cudaStream_t st, LmCtl* ctl, const DenseSolve& ds) {
    const int n = ds.n;
    if (!ds.chol_big) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(h->chol_cluster * kSpec));
        cfg.blockDim = dim3(kCholThreads);
        cfg.dynamicSmemBytes = ds.chol_smem;
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)h->chol_cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        OVS_CUDA_CHECK(cudaLaunchKernelEx(&cfg, k_ba_cholesky_solve, (const LmCtl*)ctl, ds.S, ds.S_stride, n, ds.x, ds.invL, ds.invL_stride, ds.fail, ds.chol_dbuf));
        ovs::count_launch();
    } else {
        for (int kb = 0; kb < n; kb += kNB) {
            const int nb = std::min(kNB, n - kb), rem = n - kb - nb, prow = rem + 1;
            k_chol_big_diag<<<dim3(1, kSpec), 64, 0, st>>>(ctl, ds.S, ds.S_stride, n, kb, nb, ds.invL, ds.invL_stride, ds.fail);
            OVS_LAUNCH_CHECK();
            k_chol_big_panel<<<dim3((prow + 127) / 128, kSpec), 128, 0, st>>>(ctl, ds.S, ds.S_stride, n, kb, nb, ds.invL, ds.invL_stride);
            OVS_LAUNCH_CHECK();
            if (rem > 0) {
                int tiles = 0;
                for (int mi = 0; mi < (prow + 15) / 16; ++mi) tiles += std::min((rem + 31) / 32, (16 * mi + 15) / 32 + 1);
                k_chol_big_trailing<<<dim3((tiles + 3) / 4, kSpec), 128, 0, st>>>(ctl, ds.S, ds.S_stride, n, kb, nb);
                OVS_LAUNCH_CHECK();
            }
        }
        const size_t bsm = (size_t)(((n + 31) / 32) * 32 + 32 * 33 + 32) * sizeof(double);
        k_chol_big_backsolve<<<kSpec, 512, bsm, st>>>(ctl, ds.S, ds.S_stride, n, ds.invL, ds.invL_stride, ds.x, ds.fail);
        OVS_LAUNCH_CHECK();
    }
    return OVS_OK;
}

// The host side of one SparseOptimizer::optimize(iterations) call of the device-side Levenberg loop (LmCtl, k_ba_reduce):
// per iteration a static launch sequence (iteration_head: linearise, plan, the first trial batch), enqueued for all iterations
// at once (or replayed as a CUDA graph), one wait per round, and the rare path where a whole batch was rejected and the
// device halted.  The bundle adjusters (run_impl) and the pose graph (ovs_graph_optimize_host) differ only in the callbacks.
struct LmDriver {
    ovs_optimizer* h = nullptr; cudaStream_t st = nullptr; LmCtl* ctl = nullptr;
    const volatile int* stop_word = nullptr; double* maxdiag = nullptr; volatile int* mirror = nullptr; volatile int* hm = nullptr;
    bool host_sync = false, use_graph = false;
    std::function<int()> errors_at_current;                       // currentChi at the start of the round
    std::function<int(bool in_graph, bool halt_if_undecided)> iteration_head;
    std::function<int(bool in_graph, bool halt_if_undecided, int next_width_cap)> trial_batch;
    std::function<int()> wait_device;                             // waits for everything enqueued so far
};

int lm_round(LmDriver& D, int iterations, int use_huber) {
    ovs_optimizer* const h = D.h;
    const cudaStream_t st = D.st;
    LmCtl* const ctl = D.ctl;
    volatile int* const hm = D.hm;
    // the remaining trial batches of an iteration whose first batch was rejected entirely: enqueue one, look, repeat
    auto finish_iteration = [&]() -> int {
        for (;;) {
            int rc = D.wait_device();
            if (rc != OVS_OK) return rc;
            if (hm[0] == 0) return OVS_OK;       // decided (or the round is over)
            rc = D.trial_batch(false, false, 0);
            if (rc != OVS_OK) return rc;
        }
    };
    k_lm_round_begin<<<1, 1, 0, st>>>(ctl, iterations, use_huber, D.stop_word, D.maxdiag, D.mirror);
    OVS_LAUNCH_CHECK();
    if (iterations > 0) {
        const int rc = D.errors_at_current();
        if (rc != OVS_OK) return rc;
    }
    bool captured = false;
    int it0 = 0;
    while (it0 < iterations) {
        if (D.host_sync) {
            // one iteration at a time, the host deciding what to launch next
            int rc = D.iteration_head(false, false);
            if (rc != OVS_OK) return rc;
            rc = finish_iteration();
            if (rc != OVS_OK) return rc;
            if (hm[1] == 0) break;            // ok == false, stopped, or the budget is used up
            it0 = hm[4];
            continue;
        }
        // optimistic: all remaining iterations, one batch each, no host round trip
        for (int it = it0; it < iterations; ++it) {
            if (D.use_graph) {
                if (!captured) {
                    // the iteration's launch sequence does not depend on the iteration: capture it once per round
                    // (grids are those of the prepared problem), update-or-instantiate, then replay
                    OVS_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                    const int rc_body = D.iteration_head(true, true);
                    cudaGraph_t g = nullptr;
                    const cudaError_t ce = cudaStreamEndCapture(st, &g);
                    if (rc_body != OVS_OK) { if (g) cudaGraphDestroy(g); return rc_body; }
                    OVS_CUDA_CHECK(ce);
                    if (h->gx_iter) {
                        cudaGraphExecUpdateResultInfo info;
                        if (cudaGraphExecUpdate(h->gx_iter, g, &info) != cudaSuccess) { cudaGetLastError(); cudaGraphExecDestroy(h->gx_iter); h->gx_iter = nullptr; }
                    }
                    if (!h->gx_iter) {
                        const cudaError_t ie = cudaGraphInstantiate(&h->gx_iter, g, 0);
                        if (ie != cudaSuccess) { cudaGraphDestroy(g); OVS_CUDA_CHECK(ie); }
                    }
                    cudaGraphDestroy(g);
                    captured = true;
                }
                OVS_CUDA_CHECK(cudaGraphLaunch(h->gx_iter, st));
            } else {
                const int rc = D.iteration_head(false, true);
                if (rc != OVS_OK) return rc;
            }
        }
        int rc = D.wait_device();
        if (rc != OVS_OK) return rc;
        if (hm[3] == 0) break;                // every iteration was decided by its first batch: the round is complete
        // rare path: an iteration had its whole first batch rejected and the device halted there
        k_lm_resume<<<1, 1, 0, st>>>(ctl, D.mirror);
        OVS_LAUNCH_CHECK();
        rc = D.trial_batch(false, false, 0);
        if (rc != OVS_OK) return rc;
        rc = finish_iteration();
        if (rc != OVS_OK) return rc;
        if (hm[1] == 0) break;
        it0 = hm[4];
    }
    k_lm_round_end<<<1, 1, 0, st>>>(ctl, D.stop_word, D.mirror);
    OVS_LAUNCH_CHECK();
    return OVS_OK;
}

}  // namespace

namespace {
// rounds == 2: local_bundle_adjuster (Huber round, outlier cut, plain round, final classification);
// rounds == 1: global_bundle_adjuster (one round of num_first_iter iterations, Huber iff huber_first, no classification)
int run_impl(ovs_optimizer* h, int rounds, int huber_first, int num_first_iter, int num_second_iter, const volatile uint8_t* force_stop_flag,
             ovs_ba_stats* stats) {
    OVS_REQUIRE(h && h->plan->valid, OVS_ERR_INVALID_ARG, "no prepared bundle-adjustment problem");
    OVS_REQUIRE(num_first_iter >= 0 && num_second_iter >= 0, OVS_ERR_INVALID_ARG, "bad iteration counts");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    ovs_ba_plan& pl = *h->plan;
    cudaStream_t st = h->stream;
    const int L = pl.L, K = pl.K, M = pl.M, n = pl.n, nfree = pl.nfree, npairs = pl.npairs, nb_obs = pl.nb_obs, nb_upd = pl.nb_upd;
    const size_t sM = (size_t)M, pose_sz = 12 * (size_t)K, point_sz = 3 * (size_t)L;
    const BaDev P = pl.P;
    const float chi_sq_2D = 5.99146f, chi_sq_3D = 7.81473f;
    LmCtl* const ctl = pl.dctl;
    volatile int* const stop_word = h->d_mirror + 2;
    h->h_mirror[0] = 0; h->h_mirror[1] = 0; h->h_mirror[2] = 0;
    h->pending = true;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    // (re)start from the uploaded estimates: all edges active, errors cleared
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.dposes_ring, pl.dposes_in, 8 * pose_sz, cudaMemcpyDeviceToDevice, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.dpoints_ring, pl.dpoints_in, 8 * point_sz, cudaMemcpyDeviceToDevice, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.dlevel, 0, sM, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.derr, 0, 24 * sM, st));
    OVS_CUDA_CHECK(cudaMemsetAsync(pl.dout, 0, sM, st));
    if (pl.npair_entries > 0) {     // every edge is in the graph again: clear the "excluded" marks of the co-observation records
        k_ba_pair_flags<<<((int)pl.npair_entries + 255) / 256, 256, 0, st>>>(pl.dlevel, pl.d_pair_rec, (int)pl.npair_entries);
        OVS_LAUNCH_CHECK();
    }
    pl.cur = 0;
    if (force_stop_flag && *force_stop_flag) { OVS_CUDA_CHECK(ovs::sync_stream(st)); h->pending = false; return OVS_OK; }

    // The host looks at the device's state once per round (and after each batch on the rare path where a whole batch was
    // rejected).  host_sync mode: after EVERY batch, so that batches and iterations that are not needed are never
    // launched -- the default only where a batch is ~100 launches (the multi-launch solver of very large systems).
    const bool host_sync = h->lm_host_sync >= 0 ? h->lm_host_sync != 0 : pl.chol_big != 0;
    const bool use_graph = h->use_graphs && !host_sync;
    volatile int* const mirror = (volatile int*)h->d_mirror;
    volatile int* const hm = (volatile int*)h->h_mirror;
    const int sw = std::min(std::max(h->spec_width, 1), kSpec);
    const int sw2 = std::min(std::max(h->spec_width2, 0), kSpec);   // static follow-up batch (0 = none)
    const bool time_solver = stats != nullptr;
    int solver_slots = 0;   // trial batches enqueued outside graphs (events + exec_log slots)

    k_lm_init<<<1, 1, 0, st>>>(ctl, sw, pl.dfail, mirror);
    OVS_LAUNCH_CHECK();

    // waits for everything enqueued so far; meanwhile the caller's force_stop_flag is relayed to the device's stop word
    auto wait_device = [&]() -> int {
        if (!force_stop_flag) { OVS_CUDA_CHECK(ovs::sync_stream(st)); return OVS_OK; }
        OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
        return wait_for_run(h, h->ev[1], force_stop_flag);
    };

    // one trial batch: (Hll + lambda I)^-1, Schur complement, reduced solve, update, errors at the candidates, decision
    auto trial_batch = [&](bool in_graph, bool halt_if_undecided, int next_width_cap) -> int {
        const int slot = solver_slots;
        const bool ev = time_solver && !in_graph && slot < pl.exec_cap;
        if (ev) {
            // CUDA events on the launching stream: [4 slot] .. [4 slot + 1] Schur complement (chunk + final), [4 slot + 1] ..
            // [4 slot + 3] reduced-system solver (stats->schur_us / solver_us count the batches that ran)
            while (h->solver_ev.size() < 4 * (size_t)(slot + 1)) {
                cudaEvent_t e0;
                OVS_CUDA_CHECK(cudaEventCreateWithFlags(&e0, cudaEventDefault));
                h->solver_ev.push_back(e0);
            }
            OVS_CUDA_CHECK(cudaEventRecord(h->solver_ev[4 * slot], st));
        }
        if (pl.rows == 3) k_ba_schur_chunk<3><<<pl.max_chunks, 128, 0, st>>>(P, ctl, pl.dnchunks, pl.d_pair_rec, pl.dchunks, pl.dpab, pl.dHll, pl.drec, pl.dbl, pl.dspart, pl.spart_stride);
        else k_ba_schur_chunk<2><<<pl.max_chunks, 128, 0, st>>>(P, ctl, pl.dnchunks, pl.d_pair_rec, pl.dchunks, pl.dpab, pl.dHll, pl.drec, pl.dbl, pl.dspart, pl.spart_stride);
        OVS_LAUNCH_CHECK();
        k_ba_schur_final<<<dim3(npairs, kSpec), 64, 0, st>>>(n, ctl, pl.dpair_chunk_begin, pl.dpab, pl.dspart, pl.spart_stride, pl.dHpp, pl.dbp, pl.dS, pl.S_stride);
        OVS_LAUNCH_CHECK();
        if (ev) OVS_CUDA_CHECK(cudaEventRecord(h->solver_ev[4 * slot + 1], st));     // end of the Schur complement = start of the solver
        const DenseSolve ds{pl.dS, pl.S_stride, n, pl.dx, pl.dinvL, pl.invL_stride, pl.dfail, pl.chol_big, pl.chol_dbuf, pl.chol_smem};
        const int rc_solve = launch_dense_solve(h, st, ctl, ds);
        if (rc_solve != OVS_OK) return rc_solve;
        if (ev) OVS_CUDA_CHECK(cudaEventRecord(h->solver_ev[4 * slot + 3], st));
        if (pl.rows == 3) k_ba_update<3><<<nb_upd, 128, 0, st>>>(P, ctl, pl.drec, pl.dHll, pl.dbl, pl.dbp, pl.dx, pl.dposes_ring, pl.dpoints_ring, pl.dpscale, pl.dfail);
        else k_ba_update<2><<<nb_upd, 128, 0, st>>>(P, ctl, pl.drec, pl.dHll, pl.dbl, pl.dbp, pl.dx, pl.dposes_ring, pl.dpoints_ring, pl.dpscale, pl.dfail);
        OVS_LAUNCH_CHECK();
        k_ba_errors<<<dim3(nb_obs, kSpec), 128, 0, st>>>(P, ctl, 0, pl.derr, pl.dpchi);
        OVS_LAUNCH_CHECK();
        k_ba_reduce<<<1, kSpec * 256, 0, st>>>(ctl, 1, pl.dpchi, nb_obs, pl.dpscale, nb_upd, pl.dfail, stop_word, ev ? slot : -1, pl.dexec, mirror,
                                               halt_if_undecided ? 1 : 0, next_width_cap);
        OVS_LAUNCH_CHECK();
        if (!in_graph) ++solver_slots;
        return OVS_OK;
    };

    // the static part of one Levenberg iteration: buildSystem (linearise + accumulate), plan, the first trial batch
    auto iteration_head = [&](bool in_graph, bool halt_if_undecided) -> int {
        const unsigned nb_lin = (unsigned)(pl.nlseg * kLbSegCap);
        if (pl.rows == 3) k_ba_linearize<3><<<nb_lin, 128, 0, st>>>(P, ctl, pl.dnlblocks, pl.dlblocks, pl.drec, pl.dHll, pl.dbl, pl.dmaxdiag);
        else k_ba_linearize<2><<<nb_lin, 128, 0, st>>>(P, ctl, pl.dnlblocks, pl.dlblocks, pl.drec, pl.dHll, pl.dbl, pl.dmaxdiag);
        OVS_LAUNCH_CHECK();
        if (pl.rows == 3) k_ba_pose_accum_chunk<3><<<pl.max_dchunks, 128, 0, st>>>(P, ctl, pl.dnchunks + 1, pl.d_pair_rec, pl.ddchunks, pl.drec, pl.dppart);
        else k_ba_pose_accum_chunk<2><<<pl.max_dchunks, 128, 0, st>>>(P, ctl, pl.dnchunks + 1, pl.d_pair_rec, pl.ddchunks, pl.drec, pl.dppart);
        OVS_LAUNCH_CHECK();
        k_ba_pose_final_plan<<<1, 1024, 0, st>>>(ctl, nfree, pl.dkf_chunk_begin, pl.dppart, pl.dHpp, pl.dbp, pl.dmaxdiag, pl.dfail, stop_word, mirror);
        OVS_LAUNCH_CHECK();
        if (sw2 > 0 && halt_if_undecided) {
            // two static batches per iteration: sw trials, then (only if all of them were rejected: otherwise its kernels return
            // at their first instruction) sw2 more; the device halts only when both were rejected entirely
            const int rc = trial_batch(in_graph, false, sw2);
            if (rc != OVS_OK) return rc;
        }
        return trial_batch(in_graph, halt_if_undecided, 0);
    };

    LmDriver drv;
    drv.h = h; drv.st = st; drv.ctl = ctl; drv.stop_word = stop_word; drv.maxdiag = pl.dmaxdiag; drv.mirror = mirror; drv.hm = hm;
    drv.host_sync = host_sync; drv.use_graph = use_graph;
    drv.errors_at_current = [&]() -> int {
        // computeActiveErrors + activeRobustChi2 at the current estimate (errors go to slot 0)
        k_ba_errors<<<dim3(nb_obs, 1), 128, 0, st>>>(P, ctl, 1, pl.derr, pl.dpchi);
        OVS_LAUNCH_CHECK();
        k_ba_reduce<<<1, kSpec * 256, 0, st>>>(ctl, 0, pl.dpchi, nb_obs, pl.dpscale, 0, pl.dfail, stop_word, -1, nullptr, nullptr, 0, 0);
        OVS_LAUNCH_CHECK();
        return OVS_OK;
    };
    drv.iteration_head = iteration_head;
    drv.trial_batch = trial_batch;
    drv.wait_device = wait_device;
    // SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg
    auto lm_optimize = [&](int iterations, int use_huber) -> int { return lm_round(drv, iterations, use_huber); };

    int rc = lm_optimize(num_first_iter, huber_first);
    if (rc != OVS_OK) return rc;
    if (rounds == 2) {
        // between the rounds (skipped on the device when the call was stopped): outliers leave the graph, their errors are kept
        k_ba_classify<<<nb_obs, 128, 0, st>>>(P, ctl, pl.derr, (double)chi_sq_2D, (double)chi_sq_3D, 0, pl.dlevel, pl.dout);
        OVS_LAUNCH_CHECK();
        k_ba_replicate_err<<<(unsigned)((3 * sM + 255) / 256), 256, 0, st>>>(ctl, pl.derr, 3 * sM);
        OVS_LAUNCH_CHECK();
        if (pl.npair_entries > 0) {
            k_ba_pair_flags<<<((int)pl.npair_entries + 255) / 256, 256, 0, st>>>(pl.dlevel, pl.d_pair_rec, (int)pl.npair_entries);
            OVS_LAUNCH_CHECK();
        }
        rc = lm_optimize(num_second_iter, 0);
        if (rc != OVS_OK) return rc;
        k_ba_classify<<<nb_obs, 128, 0, st>>>(P, ctl, pl.derr, (double)chi_sq_2D, (double)chi_sq_3D, 1, pl.dlevel, pl.dout);
        OVS_LAUNCH_CHECK();
    }
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.hctl, ctl, sizeof(LmCtl), cudaMemcpyDeviceToHost, st));
    const int nslots = std::min(solver_slots, pl.exec_cap);
    if (time_solver && nslots > 0) OVS_CUDA_CHECK(cudaMemcpyAsync(pl.hexec, pl.dexec, sizeof(int) * (size_t)nslots, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    if (force_stop_flag) rc = wait_for_run(h, h->ev[1], force_stop_flag);
    else { OVS_CUDA_CHECK(ovs::sync_event(h->ev[1])); rc = OVS_OK; }
    if (rc != OVS_OK) return rc;
    h->pending = false;
    const LmCtl& c = *pl.hctl;
    pl.cur = c.cur;
    if (stats) {
        stats->num_rounds = c.num_rounds;    // a call stopped before its second optimize() reports one round, as the reference
        stats->num_iterations = c.num_iterations; stats->num_trials = c.num_trials;
        for (int r = 0; r < 8; ++r) { stats->round_iterations[r] = c.round_iterations[r]; stats->lambda_init[r] = c.lambda_init[r]; }
        stats->last_lambda = c.last_lambda; stats->last_chi2 = c.last_chi2; stats->final_chi2 = c.last_chi2;
        float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
        stats->device_us = ms * 1000.f;
        float sum = 0, sum_schur = 0;
        if (time_solver)
            for (int i = 0; i < nslots; ++i)
                if (pl.hexec[i] > 0) {
                    float m = 0;
                    cudaEventElapsedTime(&m, h->solver_ev[4 * i + 1], h->solver_ev[4 * i + 3]); sum += m;
                    cudaEventElapsedTime(&m, h->solver_ev[4 * i], h->solver_ev[4 * i + 1]); sum_schur += m;
                }
        stats->solver_us = sum * 1000.f;
        stats->schur_us = sum_schur * 1000.f;
        stats->co_observations = (int32_t)pl.npair_entries;
        stats->solver_launches = c.batches;
        stats->solver_trials = c.solver_trials;
        stats->reduced_dim = n;
    }
    return OVS_OK;
}
}  // namespace

extern "C" int ovs_local_ba_run(ovs_optimizer* h, int num_first_iter, int num_second_iter, const volatile uint8_t* force_stop_flag,
                                ovs_ba_stats* stats) {
    return run_impl(h, 2, 1, num_first_iter, num_second_iter, force_stop_flag, stats);
}

// optimize::global_bundle_adjuster::optimize (optimize/global_bundle_adjuster.cc): every keyframe and landmark of the map in
// one graph, the origin keyframe(s) fixed, ONE Levenberg round of num_iter iterations with the Huber kernel on every edge
// when use_huber_kernel, no outlier classification.  The caller writes the result back as the loop-BA poses / positions.
extern "C" int ovs_global_ba_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, double* poses, const uint8_t* fixed,
                                  int L, double* points, int M, const int32_t* obs_kf, const int32_t* obs_lm, const float* obs_xy,
                                  const float* obs_x_right, const float* inv_sigma_sq, int num_iter, int use_huber_kernel,
                                  const volatile uint8_t* force_stop_flag, ovs_ba_stats* stats) {
    OVS_REQUIRE(h && cam && K > 0 && L >= 0 && M >= 0 && num_iter >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(poses && fixed && (L == 0 || points) && (M == 0 || (obs_kf && obs_lm && obs_xy && inv_sigma_sq)), OVS_ERR_INVALID_ARG, "null argument");
    if (stats) memset(stats, 0, sizeof(*stats));
    if (force_stop_flag && *force_stop_flag) return OVS_OK;
    if (M == 0 || L == 0) return OVS_OK;
    int rc = ovs_local_ba_prepare(h, cam, setup_is_mono, K, poses, fixed, L, points, M, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq);
    if (rc != OVS_OK) return rc;
    rc = run_impl(h, 1, use_huber_kernel ? 1 : 0, num_iter, 0, force_stop_flag, stats);
    if (rc != OVS_OK) return rc;
    return ovs_local_ba_fetch(h, poses, points, nullptr);
}

// CTAs per thread-block cluster of the reduced-system solver: 8 (default) minimises the latency of one call; a process that
// runs several optimisers concurrently on one GPU gets more calls per second with 2 (the solver is latency bound: a wider
// cluster shortens it little but occupies 4x the SMs, which the other streams' kernels could use).  Same results for every width.
extern "C" int ovs_optimizer_set_cluster_width(ovs_optimizer* h, int width) {
    OVS_REQUIRE(h && (width == 1 || width == 2 || width == 4 || width == 8), OVS_ERR_INVALID_ARG, "cluster width must be 1, 2, 4 or 8");
    h->chol_cluster = width;
    return OVS_OK;
}

extern "C" int ovs_optimizer_set_speculation(ovs_optimizer* h, int width) {
    OVS_REQUIRE(h && width >= 1 && width <= kSpec, OVS_ERR_INVALID_ARG, "speculation width must be 1..%d", kSpec);
    h->spec_width = width;
    return OVS_OK;
}

extern "C" int ovs_optimizer_set_second_batch(ovs_optimizer* h, int width) {
    OVS_REQUIRE(h && width >= 0 && width <= kSpec, OVS_ERR_INVALID_ARG, "second-batch width must be 0..%d", kSpec);
    h->spec_width2 = width;
    return OVS_OK;
}

extern "C" int ovs_optimizer_set_graphs(ovs_optimizer* h, int enable) {
    OVS_REQUIRE(h, OVS_ERR_INVALID_ARG, "null handle");
    h->use_graphs = enable ? 1 : 0;
    return OVS_OK;
}

extern "C" int ovs_optimizer_set_host_sync(ovs_optimizer* h, int mode) {
    OVS_REQUIRE(h && mode >= -1 && mode <= 1, OVS_ERR_INVALID_ARG, "host-sync mode must be -1 (auto), 0 or 1");
    h->lm_host_sync = mode;
    return OVS_OK;
}

// Development aid / test hook: the co-observation sort of the graph preparation on host arrays (stable, by the low end_bit
// bits of the keys).  tests/test_optimize_gpu.py compares it with numpy's stable argsort.
extern "C" int ovs_debug_sort_pairs(int device, const uint32_t* keys, const uint64_t* vals, int n, int end_bit, uint32_t* keys_out, uint64_t* vals_out) {
    OVS_REQUIRE(keys && vals && keys_out && vals_out && n >= 0 && end_bit >= 1 && end_bit <= 32, OVS_ERR_INVALID_ARG, "bad argument");
    if (n == 0) return OVS_OK;
    OVS_CUDA_CHECK(cudaSetDevice(device));
    const size_t sn = (size_t)n;
    unsigned *k0 = nullptr, *k1 = nullptr; unsigned long long *v0 = nullptr, *v1 = nullptr; int* scratch = nullptr;
    auto release = [&]() { cudaFree(k0); cudaFree(k1); cudaFree(v0); cudaFree(v1); cudaFree(scratch); };
    int rc = OVS_OK;
    do {
        if (cudaMalloc(&k0, 4 * sn) != cudaSuccess || cudaMalloc(&k1, 4 * sn) != cudaSuccess || cudaMalloc(&v0, 8 * sn) != cudaSuccess ||
            cudaMalloc(&v1, 8 * sn) != cudaSuccess || cudaMalloc(&scratch, 4 * sort_scratch_ints(n)) != cudaSuccess) {
            cudaGetLastError(); ovs::set_error("ovs_debug_sort_pairs: out of device memory"); rc = OVS_ERR_CUDA; break;
        }
        if (cudaMemcpy(k0, keys, 4 * sn, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(v0, vals, 8 * sn, cudaMemcpyHostToDevice) != cudaSuccess) {
            ovs::set_error("ovs_debug_sort_pairs: upload failed"); rc = OVS_ERR_CUDA; break;
        }
        unsigned* ks = nullptr; unsigned long long* vs = nullptr;
        rc = sort_pairs(nullptr, k0, k1, v0, v1, n, end_bit, scratch, &ks, &vs);
        if (rc != OVS_OK) break;
        if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(keys_out, ks, 4 * sn, cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(vals_out, vs, 8 * sn, cudaMemcpyDeviceToHost) != cudaSuccess) {
            ovs::set_error("ovs_debug_sort_pairs: %s", cudaGetErrorString(cudaGetLastError())); rc = OVS_ERR_CUDA; break;
        }
    } while (0);
    release();
    return rc;
}

extern "C" int ovs_local_ba_fetch(ovs_optimizer* h, double* poses, double* points, uint8_t* outlier_out) {
    OVS_REQUIRE(h && h->plan->valid, OVS_ERR_INVALID_ARG, "no prepared bundle-adjustment problem");
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    ovs_ba_plan& pl = *h->plan;
    cudaStream_t st = h->stream;
    const size_t sK = (size_t)pl.K, sL = (size_t)pl.L, sM = (size_t)pl.M;
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.hposes, pl.dposes_ring + (size_t)pl.cur * 12 * sK, 96 * sK, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.hpoints, pl.dpoints_ring + (size_t)pl.cur * 3 * sL, 24 * sL, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(pl.hout, pl.dout, sM, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    h->pending = false;
    if (poses) memcpy(poses, pl.hposes, 96 * sK);
    if (points) memcpy(points, pl.hpoints, 24 * sL);
    if (outlier_out) memcpy(outlier_out, pl.hout, sM);
    return OVS_OK;
}

extern "C" int ovs_local_ba_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, double* poses, const uint8_t* fixed,
                                 int L, double* points, int M, const int32_t* obs_kf, const int32_t* obs_lm, const float* obs_xy,
                                 const float* obs_x_right, const float* inv_sigma_sq, int num_first_iter, int num_second_iter,
                                 const volatile uint8_t* force_stop_flag, uint8_t* outlier_out, ovs_ba_stats* stats) {
    OVS_REQUIRE(h && cam && K > 0 && L >= 0 && M >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(poses && fixed && (L == 0 || points) && (M == 0 || (obs_kf && obs_lm && obs_xy && inv_sigma_sq && outlier_out)),
                OVS_ERR_INVALID_ARG, "null argument");
    if (stats) memset(stats, 0, sizeof(*stats));
    for (int i = 0; i < M; ++i) outlier_out[i] = 0;
    if (force_stop_flag && *force_stop_flag) return OVS_OK;
    if (M == 0 || L == 0) return OVS_OK;
    int rc = ovs_local_ba_prepare(h, cam, setup_is_mono, K, poses, fixed, L, points, M, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq);
    if (rc != OVS_OK) return rc;
    rc = ovs_local_ba_run(h, num_first_iter, num_second_iter, force_stop_flag, stats);
    if (rc != OVS_OK) return rc;
    return ovs_local_ba_fetch(h, poses, points, outlier_out);
}

// ------------------------------------------------------------------------------ handle
extern "C" int ovs_optimizer_create(int device, ovs_optimizer** out) {
    OVS_REQUIRE(out, OVS_ERR_INVALID_ARG, "null argument");
    int rc = ovs::select_device(device);
    if (rc != OVS_OK) return rc;
    ovs_optimizer* h = new (std::nothrow) ovs_optimizer();
    OVS_REQUIRE(h, OVS_ERR_CUDA, "out of host memory");
    h->device = device;
    h->plan = new (std::nothrow) ovs_ba_plan();
    OVS_REQUIRE(h->plan, OVS_ERR_CUDA, "out of host memory");
    bool ok = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess
              && cudaEventCreateWithFlags(&h->ev[0], ovs::event_flags()) == cudaSuccess && cudaEventCreateWithFlags(&h->ev[1], ovs::event_flags()) == cudaSuccess
              && cudaHostAlloc(&h->h_mirror, 16 * sizeof(int), cudaHostAllocMapped) == cudaSuccess
              && cudaHostGetDevicePointer(&h->d_mirror, h->h_mirror, 0) == cudaSuccess
              && cudaFuncSetAttribute(k_ba_cholesky_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, kCholMaxDynSmem) == cudaSuccess
              && cudaFuncSetAttribute(k_chol_big_backsolve, cudaFuncAttributeMaxDynamicSharedMemorySize, 60 * 1024) == cudaSuccess;
    if (!ok) {
        ovs::set_error("optimizer handle setup failed: %s", cudaGetErrorString(cudaGetLastError()));
        ovs_optimizer_destroy(h);
        return OVS_ERR_CUDA;
    }
    *out = h;
    return OVS_OK;
}

extern "C" void ovs_optimizer_destroy(ovs_optimizer* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) ovs::sync_stream(h->stream);
    cudaFree(h->d_arena); cudaFree(h->d_work); cudaFreeHost(h->h_arena); cudaFreeHost(h->h_mirror);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    for (auto& e : h->solver_ev) cudaEventDestroy(e);
    if (h->gx_iter) cudaGraphExecDestroy(h->gx_iter);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h->plan;
    delete h;
}


// ================================================================================ pose graph
// optimize::graph_optimizer::optimize (loop closure): one Sim3 vertex per keyframe, relative Sim3 edges with identity
// information, g2o's Levenberg with the user lambda 1e-16, then the write-back of the poses and the landmark correction.
// Per Levenberg iteration (state in LmCtl, the same device-side controller as the bundle adjusters):
//   k_pg_linearize   per edge: e = log(S_ji S_i S_j^-1), J_i, J_j (sim3_math.cuh) -> H_ii, H_ij, H_jj, b_i, b_j
//   k_pg_plan        lambda_0 and the damping values of the first trial batch
//  per trial batch (up to 4 damping values):
//   k_pg_assemble    per block pair (r >= c) and trial: the whole lower triangle of H + lambda I and the rhs row, summed over the
//                    pair's edge list (edges sorted by block pair once per call, stable) in a fixed order -- no atomics
//   dense solver     the local BA's: k_ba_cholesky_solve (7 n_free <= 688) or k_chol_big_* above
//   k_pg_update      per vertex: S <- exp(x) S into the candidate slots, LM scale terms
//   k_pg_errors      per edge: chi2 at each candidate;  k_ba_reduce: the Levenberg decision
// Finish: k_pg_finish writes the optimised Sim3s, pose_cw = {R, t / s} and the corrected landmarks.
namespace {

constexpr int kPgBlk = 161;   // per-edge linearisation: H_ii, H_ij, H_jj (7 x 7 row-major each), b_i, b_j

struct PgDev {
    int K, E, nfree, n, fix_scale;      // n: pitch of a trial's solution in x (the system's row pitch)
    double* ring;                                       // (kSpec + 1) x K x 13: current estimate and candidates
    const int* free_idx;                                // K: block of a free vertex, -1 for fixed and isolated vertices
    const int* ei; const int* ej; const double* meas;   // E, E, E x 13 (S_ji)
};

__host__ __device__ __forceinline__ int pg_pair_id(int r, int c) { return r * (r + 1) / 2 + c; }   // block pair r >= c

// Edge list entries by block pair: per edge up to three (edge << 2 | role) -- role 0: H_ii on (a, a), 1: H_jj on (b, b),
// 2: H_ij on (a, b) with a > b, 3: H_ij' on (b, a) with b > a -- and the key `sentinel` for the slots an edge does not use.
__global__ void __launch_bounds__(256) k_pg_emit(PgDev P, unsigned sentinel, unsigned* __restrict__ keys, unsigned long long* __restrict__ vals) {
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= P.E) return;
    const int a = P.free_idx[P.ei[e]], b = P.free_idx[P.ej[e]];
    const unsigned long long v = (unsigned long long)e << 2;
    keys[3 * (size_t)e] = a >= 0 ? (unsigned)pg_pair_id(a, a) : sentinel;
    vals[3 * (size_t)e] = v;
    keys[3 * (size_t)e + 1] = b >= 0 ? (unsigned)pg_pair_id(b, b) : sentinel;
    vals[3 * (size_t)e + 1] = v | 1;
    unsigned k2 = sentinel;
    unsigned long long v2 = v | 2;
    if (a >= 0 && b >= 0) {
        if (a > b) k2 = (unsigned)pg_pair_id(a, b);
        else { k2 = (unsigned)pg_pair_id(b, a); v2 = v | 3; }
    }
    keys[3 * (size_t)e + 2] = k2;
    vals[3 * (size_t)e + 2] = v2;
}

__device__ __forceinline__ void pg_load13(const double* src, double* dst) {
#pragma unroll
    for (int k = 0; k < 13; ++k) dst[k] = src[k];
}

// one thread per edge with at least one free vertex
__global__ void __launch_bounds__(128) k_pg_linearize(PgDev P, const LmCtl* __restrict__ ctl, double* __restrict__ blk) {
    if (!ctl->active) return;
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= P.E) return;
    const int i = P.ei[e], j = P.ej[e];
    if (P.free_idx[i] < 0 && P.free_idx[j] < 0) return;
    const double* S = P.ring + (size_t)ctl->cur * 13 * P.K;
    double Sji[13], Si[13], Sj[13], err[7], J[98];
    pg_load13(P.meas + 13 * (size_t)e, Sji);
    pg_load13(S + 13 * (size_t)i, Si);
    pg_load13(S + 13 * (size_t)j, Sj);
    ovs::graph_edge(Sji, Si, Sj, err, J);
    double* o = blk + (size_t)kPgBlk * e;
    for (int r = 0; r < 7; ++r)
        for (int c = 0; c < 7; ++c) {
            double hii = 0.0, hij = 0.0, hjj = 0.0;
            for (int k = 0; k < 7; ++k) {
                hii += J[14 * k + r] * J[14 * k + c];
                hij += J[14 * k + r] * J[14 * k + 7 + c];
                hjj += J[14 * k + 7 + r] * J[14 * k + 7 + c];
            }
            o[7 * r + c] = hii; o[49 + 7 * r + c] = hij; o[98 + 7 * r + c] = hjj;
        }
    for (int r = 0; r < 7; ++r) {
        double gi = 0.0, gj = 0.0;
        for (int k = 0; k < 7; ++k) { gi += J[14 * k + r] * err[k]; gj += J[14 * k + 7 + r] * err[k]; }
        o[147 + r] = -gi; o[154 + r] = -gj;      // b = -J' e
    }
}

// One block per block pair (r >= c) and trial of the batch: element (7r + ri, 7c + ci) of H + lambda I, and on diagonal pairs
// the rhs row (row n).  Every element of the lower triangle is rewritten, zero blocks included: the factorisation works in
// place.  The pair's entries are summed in their sorted (edge) order.
// n is the system's row pitch: 7 x free vertices, plus one decoupled row (identity, rhs 0, solution 0) when that is odd, because
// the cluster Cholesky loads its rows 16 bytes at a time.  Block pid == npairs writes that row.
__global__ void __launch_bounds__(64) k_pg_assemble(int n, int npairs, const LmCtl* __restrict__ ctl, const int* __restrict__ seg_begin,
                                                    const int* __restrict__ seg_end, const unsigned long long* __restrict__ ent,
                                                    const double* __restrict__ blk, double* __restrict__ S, size_t S_stride,
                                                    double* __restrict__ bvec) {
    const int bt = blockIdx.y;
    if (bt >= ctl->nbatch) return;
    const double lambda = ctl->lam[bt];
    const int pid = blockIdx.x, t = threadIdx.x;
    if (pid >= npairs) {
        S += (size_t)bt * S_stride;
        for (int c = t; c < n; c += 64) S[(size_t)(n - 1) * n + c] = c == n - 1 ? 1.0 : 0.0;
        if (t == 0) S[(size_t)n * n + n - 1] = 0.0;
        return;
    }
    int r = (int)((sqrt(8.0 * pid + 1.0) - 1.0) * 0.5);
    while (pg_pair_id(r, 0) > pid) --r;
    while (pg_pair_id(r + 1, 0) <= pid) ++r;
    const int c = pid - pg_pair_id(r, 0);
    const bool diag = r == c;
    if (t >= 56 || (t >= 49 && !diag)) return;
    S += (size_t)bt * S_stride;
    const int s0 = seg_begin[pid], s1 = seg_end[pid];
    double v = 0.0;
    if (t < 49) {
        const int ri = t / 7, ci = t - 7 * ri;
        for (int s = s0; s < s1; ++s) {
            const unsigned long long x = ent[s];
            const double* o = blk + (size_t)kPgBlk * (size_t)(x >> 2);
            const int role = (int)(x & 3);
            v += role == 0 ? o[t] : role == 1 ? o[98 + t] : role == 2 ? o[49 + t] : o[49 + 7 * ci + ri];
        }
        if (diag && ri == ci) v += lambda;
        S[(size_t)(7 * r + ri) * n + 7 * c + ci] = v;
    } else {
        const int k = t - 49;
        for (int s = s0; s < s1; ++s) {
            const unsigned long long x = ent[s];
            const double* o = blk + (size_t)kPgBlk * (size_t)(x >> 2);
            v += (x & 3) == 0 ? o[147 + k] : o[154 + k];
        }
        S[(size_t)n * n + 7 * r + k] = v;
        if (bt == 0) bvec[7 * r + k] = v;
    }
}

// g2o's setUserLambdaInit(1e-16): the first iteration's damping is the user lambda, not 1e-5 max diag(H)
__global__ void k_pg_plan(LmCtl* ctl, int* fail, volatile int* mirror) {
    if (ctl->need_more) return;     // halted: the parked batch of the undecided iteration must survive
    lm_plan_iteration(ctl, 1e-16, nullptr, fail, mirror);
}

// one thread per vertex: the candidate of every trial of the batch (free vertices S <- exp(x) S, the others copied) and the
// LM scale terms x (lambda x + b) over all seven components, one partial per block and trial
__global__ void __launch_bounds__(128) k_pg_update(PgDev P, const LmCtl* __restrict__ ctl, const double* __restrict__ x,
                                                   const double* __restrict__ bvec, double* __restrict__ partial_scale) {
    __shared__ double sm[36];
    const int nbatch = ctl->nbatch;
    if (nbatch == 0) return;
    const int k = blockIdx.x * 128 + threadIdx.x;
    double sc[kSpec];
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) sc[bt] = 0.0;
    if (k < P.K) {
        const int fi = P.free_idx[k];
        double S[13];
        pg_load13(P.ring + (size_t)ctl->cur * 13 * P.K + 13 * (size_t)k, S);
        for (int bt = 0; bt < nbatch; ++bt) {
            const double lambda = ctl->lam[bt];
            double out[13];
            if (fi >= 0) {
                double u[7];
                for (int q = 0; q < 7; ++q) {
                    u[q] = x[(size_t)bt * P.n + 7 * fi + q];
                    sc[bt] += u[q] * (lambda * u[q] + bvec[7 * fi + q]);
                }
                ovs::sim3_oplus(S, u, P.fix_scale != 0, out);
            } else {
                for (int q = 0; q < 13; ++q) out[q] = S[q];
            }
            double* dst = P.ring + (size_t)ctl->buf[bt] * 13 * P.K + 13 * (size_t)k;
            for (int q = 0; q < 13; ++q) dst[q] = out[q];
        }
    }
#pragma unroll
    for (int bt = 0; bt < kSpec; ++bt) {
        if (bt < nbatch) {          // block-uniform
            const double tot = block_sum(sc[bt], sm);
            if (threadIdx.x == 0) partial_scale[(size_t)bt * gridDim.x + blockIdx.x] = tot;
        }
    }
}

// chi2 = e'e per edge (every edge, also those between fixed vertices), one partial per block; at_current: the current estimate
__global__ void __launch_bounds__(128) k_pg_errors(PgDev P, const LmCtl* __restrict__ ctl, int at_current, double* __restrict__ partial_chi) {
    __shared__ double sm[36];
    int slot;
    if (at_current) {
        if (!ctl->active) return;
        slot = ctl->cur;
    } else {
        if ((int)blockIdx.y >= ctl->nbatch) return;
        slot = ctl->buf[blockIdx.y];
    }
    partial_chi += (size_t)blockIdx.y * gridDim.x;
    const int e = blockIdx.x * 128 + threadIdx.x;
    double c = 0.0;
    if (e < P.E) {
        const double* S = P.ring + (size_t)slot * 13 * P.K;
        double Sji[13], Si[13], Sj[13], err[7];
        pg_load13(P.meas + 13 * (size_t)e, Sji);
        pg_load13(S + 13 * (size_t)P.ei[e], Si);
        pg_load13(S + 13 * (size_t)P.ej[e], Sj);
        ovs::graph_edge(Sji, Si, Sj, err, nullptr);
        for (int k = 0; k < 7; ++k) c += err[k] * err[k];
    }
    const double tot = block_sum(c, sm);
    if (threadIdx.x == 0) partial_chi[blockIdx.x] = tot;
}

// Write-back, one thread per vertex and per landmark: the optimised Sim3s, pose_cw = {R, t / s}, and
// p <- S_wr^opt (S_rw^init p) for a landmark with reference vertex r (ref = -1: the landmark's bits stay).
// ctl == null: no optimisation ran, the estimate is ring slot 0.
__global__ void __launch_bounds__(128) k_pg_finish(PgDev P, const LmCtl* __restrict__ ctl, const double* __restrict__ sim3_init,
                                                   double* __restrict__ sim3_out, double* __restrict__ pose_out, int L,
                                                   const double* __restrict__ lm_in, const int* __restrict__ lm_ref, double* __restrict__ lm_out) {
    const int t = blockIdx.x * 128 + threadIdx.x;
    const double* cur = P.ring + (size_t)(ctl ? ctl->cur : 0) * 13 * P.K;
    if (t < P.K) {
        double S[13];
        pg_load13(cur + 13 * (size_t)t, S);
        for (int q = 0; q < 13; ++q) sim3_out[13 * (size_t)t + q] = S[q];
        for (int q = 0; q < 9; ++q) pose_out[12 * (size_t)t + q] = S[q];
        for (int q = 0; q < 3; ++q) pose_out[12 * (size_t)t + 9 + q] = S[9 + q] / S[12];
    } else if (t < P.K + L) {
        const int l = t - P.K, r = lm_ref[l];
        const double p[3] = {lm_in[3 * (size_t)l], lm_in[3 * (size_t)l + 1], lm_in[3 * (size_t)l + 2]};
        if (r < 0) {
            for (int q = 0; q < 3; ++q) lm_out[3 * (size_t)l + q] = p[q];
            return;
        }
        double S0[13], S1[13], Si[13], q0[3], q1[3], pc[3];
        pg_load13(sim3_init + 13 * (size_t)r, S0);
        pg_load13(cur + 13 * (size_t)r, S1);
        ovs::sim3_inverse(S1, Si);
        ovs::mat3_vec(S0, p, q0);
        for (int q = 0; q < 3; ++q) pc[q] = S0[12] * q0[q] + S0[9 + q];      // S_rw^init p: camera frame of r
        ovs::mat3_vec(Si, pc, q1);
        for (int q = 0; q < 3; ++q) lm_out[3 * (size_t)l + q] = Si[12] * q1[q] + Si[9 + q];
    }
}

}  // namespace

extern "C" int ovs_graph_optimize_host(ovs_optimizer* h, int K, double* sim3_cw, const uint8_t* fixed, int E, const int32_t* edge_i,
                                       const int32_t* edge_j, const double* meas_ji, int fix_scale, int num_iter, int L, double* lm_pos_w,
                                       const int32_t* lm_ref, double* pose_cw_out, ovs_ba_stats* stats) {
    OVS_REQUIRE(h && K >= 1 && E >= 0 && L >= 0 && num_iter >= 0, OVS_ERR_INVALID_ARG, "bad argument");
    OVS_REQUIRE(sim3_cw && fixed && (E == 0 || (edge_i && edge_j && meas_ji)) && (L == 0 || (lm_pos_w && lm_ref)), OVS_ERR_INVALID_ARG,
                "null argument");
    auto scale_ok = [](double s) { return s > 0.0 && std::isfinite(s); };
    for (int k = 0; k < K; ++k)
        OVS_REQUIRE(scale_ok(sim3_cw[13 * (size_t)k + 12]), OVS_ERR_INVALID_ARG, "vertex %d: the Sim3 scale must be positive and finite", k);
    for (int e = 0; e < E; ++e) {
        const int i = edge_i[e], j = edge_j[e];
        OVS_REQUIRE(i >= 0 && i < K && j >= 0 && j < K, OVS_ERR_INVALID_ARG, "edge %d references a vertex out of range", e);
        OVS_REQUIRE(i != j, OVS_ERR_INVALID_ARG, "edge %d joins vertex %d to itself", e, i);
        OVS_REQUIRE(scale_ok(meas_ji[13 * (size_t)e + 12]), OVS_ERR_INVALID_ARG, "edge %d: the Sim3 scale must be positive and finite", e);
    }
    for (int l = 0; l < L; ++l)
        OVS_REQUIRE(lm_ref[l] >= -1 && lm_ref[l] < K, OVS_ERR_INVALID_ARG, "landmark %d references a vertex out of range", l);
    if (stats) memset(stats, 0, sizeof(*stats));
    // g2o optimises the vertices of its edges only: a free vertex without an edge is not part of the system
    std::vector<int> free_idx((size_t)K, -1);
    {
        std::vector<uint8_t> used((size_t)K, 0);
        for (int e = 0; e < E; ++e) { used[edge_i[e]] = 1; used[edge_j[e]] = 1; }
        int f = 0;
        for (int k = 0; k < K; ++k)
            if (used[k] && !fixed[k]) free_idx[k] = f++;
    }
    const int nfree = K > 0 ? *std::max_element(free_idx.begin(), free_idx.end()) + 1 : 0;
    const int n = 7 * nfree;
    const int nsys = n + (n & 1);      // row pitch of the dense system: even (see k_pg_assemble)
    OVS_REQUIRE(n <= kMaxReducedDimBig, OVS_ERR_UNSUPPORTED, "more than %d free vertices (dense 7n system)", kMaxReducedDimBig / 7);
    const bool run_lm = nfree > 0 && num_iter > 0;
    OVS_CUDA_CHECK(cudaSetDevice(h->device));
    // carved from the arenas a prepared local-BA problem lives in: that problem is gone
    invalidate_plan(h);
    if (h->pending) { OVS_CUDA_CHECK(ovs::sync_stream(h->stream)); h->pending = false; }

    const size_t sK = (size_t)K, sE = (size_t)E, sL = (size_t)L, nent = 3 * sE;
    const int npairs = nfree * (nfree + 1) / 2;
    const int nb_edge = (E + 127) / 128, nb_vert = (K + 127) / 128;
    const int exec_cap = 1024;
    DenseSolve ds{};
    dense_solve_config(std::max(nsys, 1), ds);
    ds.n = nsys;
    ds.S_stride = ((size_t)(nsys + 1) * nsys + 31) / 32 * 32;
    ds.invL_stride = (size_t)((nsys + kNB - 1) / kNB) * kNB * kNB;

    double *hS, *hmeas, *hlm, *hS_out, *hpose, *hlm_out; int *hfree, *hei, *hej, *href, *hexec; LmCtl* hctl;
    double *dS_in, *dmeas, *dlm, *dS_out, *dpose, *dlm_out, *dring, *dblk, *dbvec, *dpchi, *dpscale, *dmaxdiag;
    int *dfree, *dei, *dej, *dref, *dsegb, *dsege, *dsort, *dfail, *dexec; LmCtl* dctl;
    unsigned *dkeys, *dkeys2; unsigned long long *dvals, *dvals2;
    ovs::Staging S;
    int rc = ovs::stage(S, h->h_arena, h->h_cap, h->d_arena, h->d_cap, [&](ovs::Staging& S) {
        dS_in = S.in(hS, 13 * sK); dfree = S.in(hfree, sK); dei = S.in(hei, sE); dej = S.in(hej, sE); dmeas = S.in(hmeas, 13 * sE);
        dlm = S.in(hlm, 3 * sL); dref = S.in(href, sL);
        // each read back by its own copy
        dS_out = S.out(hS_out, 13 * sK); dpose = S.out(hpose, 12 * sK); dlm_out = S.out(hlm_out, 3 * sL);
        dctl = S.out(hctl, 1); dexec = S.out(hexec, exec_cap);
        dring = S.dev<double>((kSpec + 1) * 13 * sK);
        dblk = S.dev<double>(kPgBlk * sE);
        dkeys = S.dev<unsigned>(nent); dkeys2 = S.dev<unsigned>(nent);
        dvals = S.dev<unsigned long long>(nent); dvals2 = S.dev<unsigned long long>(nent);
        dsort = S.dev<int>(sort_scratch_ints((long long)std::max<size_t>(nent, 1)));
        dsegb = S.dev<int>((size_t)npairs + 1); dsege = S.dev<int>((size_t)npairs + 1);
        dbvec = S.dev<double>((size_t)std::max(n, 1));
        dpchi = S.dev<double>(kSpec * (size_t)std::max(nb_edge, 1)); dpscale = S.dev<double>(kSpec * (size_t)nb_vert);
        dfail = S.dev<int>(kSpec); dmaxdiag = S.dev<double>(2);
    });
    if (rc != OVS_OK) return rc;
    if (run_lm) {
        auto carve_work = [&](Arena& W) {
            ds.S = W.take<double>(kSpec * ds.S_stride); ds.x = W.take<double>(kSpec * (size_t)nsys); ds.invL = W.take<double>(kSpec * ds.invL_stride);
        };
        Arena W{nullptr, 0};
        carve_work(W);
        if ((rc = ovs::grow_dev(&h->d_work, &h->w_cap, W.off)) != OVS_OK) return rc;
        W = Arena{h->d_work, 0};
        carve_work(W);
        ds.fail = dfail;
    }
    memcpy(hS, sim3_cw, 104 * sK);
    memcpy(hfree, free_idx.data(), 4 * sK);
    if (E) { memcpy(hei, edge_i, 4 * sE); memcpy(hej, edge_j, 4 * sE); memcpy(hmeas, meas_ji, 104 * sE); }
    if (L) { memcpy(hlm, lm_pos_w, 24 * sL); memcpy(href, lm_ref, 4 * sL); }

    cudaStream_t st = h->stream;
    h->pending = true;
    h->h_mirror[0] = 0; h->h_mirror[1] = 0; h->h_mirror[2] = 0;
    volatile int* const mirror = (volatile int*)h->d_mirror;
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[0], st));
    OVS_CUDA_CHECK(S.upload(st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(dring, dS_in, 104 * sK, cudaMemcpyDeviceToDevice, st));
    PgDev P;
    P.K = K; P.E = E; P.nfree = nfree; P.n = nsys; P.fix_scale = fix_scale ? 1 : 0;
    P.ring = dring; P.free_idx = dfree; P.ei = dei; P.ej = dej; P.meas = dmeas;
    int solver_slots = 0;
    const bool time_solver = stats != nullptr;
    if (run_lm) {
        // the edge lists of the block pairs: (pair id, edge << 2 | role), stable sort by pair id, segments
        const unsigned sentinel = (unsigned)npairs;
        k_pg_emit<<<(E + 255) / 256, 256, 0, st>>>(P, sentinel, dkeys, dvals);
        OVS_LAUNCH_CHECK();
        int end_bit = 1;
        while ((1u << end_bit) <= sentinel) ++end_bit;
        unsigned* ksorted = nullptr; unsigned long long* vsorted = nullptr;
        rc = sort_pairs(st, dkeys, dkeys2, dvals, dvals2, (int)nent, end_bit, dsort, &ksorted, &vsorted);
        if (rc != OVS_OK) return rc;
        OVS_CUDA_CHECK(cudaMemsetAsync(dsegb, 0, 4 * ((size_t)npairs + 1), st));
        OVS_CUDA_CHECK(cudaMemsetAsync(dsege, 0, 4 * ((size_t)npairs + 1), st));
        k_ba_segments<<<(int)((nent + 255) / 256), 256, 0, st>>>(ksorted, (int)nent, dsegb, dsege);
        OVS_LAUNCH_CHECK();
        const int sw = std::min(std::max(h->spec_width, 1), kSpec);
        k_lm_init<<<1, 1, 0, st>>>(dctl, sw, dfail, mirror);
        OVS_LAUNCH_CHECK();

        LmDriver drv;
        drv.h = h; drv.st = st; drv.ctl = dctl; drv.stop_word = nullptr; drv.maxdiag = dmaxdiag; drv.mirror = mirror;
        drv.hm = (volatile int*)h->h_mirror;
        drv.host_sync = h->lm_host_sync >= 0 ? h->lm_host_sync != 0 : ds.chol_big != 0;   // as the local BA: skip the ~100-launch batches
        drv.use_graph = false;
        drv.errors_at_current = [&]() -> int {
            k_pg_errors<<<dim3(nb_edge, 1), 128, 0, st>>>(P, dctl, 1, dpchi);
            OVS_LAUNCH_CHECK();
            k_ba_reduce<<<1, kSpec * 256, 0, st>>>(dctl, 0, dpchi, nb_edge, dpscale, 0, dfail, nullptr, -1, nullptr, nullptr, 0, 0);
            OVS_LAUNCH_CHECK();
            return OVS_OK;
        };
        drv.trial_batch = [&](bool in_graph, bool halt_if_undecided, int next_width_cap) -> int {
            const int slot = solver_slots;
            const bool ev = time_solver && !in_graph && slot < exec_cap;
            if (ev) {
                while (h->solver_ev.size() < 4 * (size_t)(slot + 1)) {
                    cudaEvent_t e0;
                    OVS_CUDA_CHECK(cudaEventCreateWithFlags(&e0, cudaEventDefault));
                    h->solver_ev.push_back(e0);
                }
            }
            k_pg_assemble<<<dim3(npairs + (nsys - n), kSpec), 64, 0, st>>>(nsys, npairs, dctl, dsegb, dsege, vsorted, dblk, ds.S, ds.S_stride, dbvec);
            OVS_LAUNCH_CHECK();
            if (ev) OVS_CUDA_CHECK(cudaEventRecord(h->solver_ev[4 * slot + 1], st));
            const int rc_solve = launch_dense_solve(h, st, dctl, ds);
            if (rc_solve != OVS_OK) return rc_solve;
            if (ev) OVS_CUDA_CHECK(cudaEventRecord(h->solver_ev[4 * slot + 3], st));
            k_pg_update<<<nb_vert, 128, 0, st>>>(P, dctl, ds.x, dbvec, dpscale);
            OVS_LAUNCH_CHECK();
            k_pg_errors<<<dim3(nb_edge, kSpec), 128, 0, st>>>(P, dctl, 0, dpchi);
            OVS_LAUNCH_CHECK();
            k_ba_reduce<<<1, kSpec * 256, 0, st>>>(dctl, 1, dpchi, nb_edge, dpscale, nb_vert, dfail, nullptr, ev ? slot : -1, dexec, mirror,
                                                   halt_if_undecided ? 1 : 0, next_width_cap);
            OVS_LAUNCH_CHECK();
            if (!in_graph) ++solver_slots;
            return OVS_OK;
        };
        drv.iteration_head = [&](bool in_graph, bool halt_if_undecided) -> int {
            k_pg_linearize<<<nb_edge, 128, 0, st>>>(P, dctl, dblk);
            OVS_LAUNCH_CHECK();
            k_pg_plan<<<1, 1, 0, st>>>(dctl, dfail, mirror);
            OVS_LAUNCH_CHECK();
            return drv.trial_batch(in_graph, halt_if_undecided, 0);
        };
        drv.wait_device = [&]() -> int { OVS_CUDA_CHECK(ovs::sync_stream(st)); return OVS_OK; };
        rc = lm_round(drv, num_iter, 0);
        if (rc != OVS_OK) return rc;
        OVS_CUDA_CHECK(cudaMemcpyAsync(hctl, dctl, sizeof(LmCtl), cudaMemcpyDeviceToHost, st));
        const int nslots = std::min(solver_slots, exec_cap);
        if (time_solver && nslots > 0) OVS_CUDA_CHECK(cudaMemcpyAsync(hexec, dexec, sizeof(int) * (size_t)nslots, cudaMemcpyDeviceToHost, st));
    } else if (E > 0 && stats) {
        // nothing to optimise (no free vertex, or num_iter == 0): chi2 at the returned estimates, for the statistics
        k_lm_init<<<1, 1, 0, st>>>(dctl, 1, dfail, mirror);
        OVS_LAUNCH_CHECK();
        k_lm_round_begin<<<1, 1, 0, st>>>(dctl, 1, 0, nullptr, dmaxdiag, mirror);   // active, so that the errors are evaluated
        OVS_LAUNCH_CHECK();
        k_pg_errors<<<dim3(nb_edge, 1), 128, 0, st>>>(P, dctl, 1, dpchi);
        OVS_LAUNCH_CHECK();
        k_ba_reduce<<<1, kSpec * 256, 0, st>>>(dctl, 0, dpchi, nb_edge, dpscale, 0, dfail, nullptr, -1, nullptr, nullptr, 0, 0);
        OVS_LAUNCH_CHECK();
        OVS_CUDA_CHECK(cudaMemcpyAsync(hctl, dctl, sizeof(LmCtl), cudaMemcpyDeviceToHost, st));
    }
    k_pg_finish<<<(unsigned)((sK + sL + 127) / 128), 128, 0, st>>>(P, run_lm ? dctl : nullptr, dS_in, dS_out, dpose, L, dlm, dref, dlm_out);
    OVS_LAUNCH_CHECK();
    OVS_CUDA_CHECK(cudaEventRecord(h->ev[1], st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(hS_out, dS_out, 104 * sK, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(cudaMemcpyAsync(hpose, dpose, 96 * sK, cudaMemcpyDeviceToHost, st));
    if (L) OVS_CUDA_CHECK(cudaMemcpyAsync(hlm_out, dlm_out, 24 * sL, cudaMemcpyDeviceToHost, st));
    OVS_CUDA_CHECK(ovs::sync_stream(st));
    h->pending = false;
    memcpy(sim3_cw, hS_out, 104 * sK);
    if (pose_cw_out) memcpy(pose_cw_out, hpose, 96 * sK);
    if (L) memcpy(lm_pos_w, hlm_out, 24 * sL);
    if (stats) {
        if (run_lm) {
            const LmCtl& c = *hctl;
            stats->num_rounds = c.num_rounds; stats->num_iterations = c.num_iterations; stats->num_trials = c.num_trials;
            stats->round_iterations[0] = c.round_iterations[0]; stats->lambda_init[0] = c.lambda_init[0];
            stats->last_lambda = c.last_lambda; stats->last_chi2 = c.last_chi2; stats->final_chi2 = c.last_chi2;
            stats->solver_launches = c.batches; stats->solver_trials = c.solver_trials;
            float sum = 0;
            const int nslots = std::min(solver_slots, exec_cap);
            for (int i = 0; i < nslots; ++i)
                if (hexec[i] > 0) { float m = 0; cudaEventElapsedTime(&m, h->solver_ev[4 * i + 1], h->solver_ev[4 * i + 3]); sum += m; }
            stats->solver_us = sum * 1000.f;
        } else {
            // one optimize() call with no iteration; chi2 of an empty graph is 0
            stats->num_rounds = 1;
            stats->final_chi2 = stats->last_chi2 = E > 0 ? hctl->currentChi : 0.0;
        }
        stats->reduced_dim = n;
        float ms = 0; cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
        stats->device_us = ms * 1000.f;
    }
    return OVS_OK;
}
