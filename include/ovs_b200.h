/*
 * ovs_b200.h -- C ABI of the H100-native OpenVSLAM hot path (libovs_b200.so).
 *
 * This is the drop-in boundary of SURVEY.md section 8(b): plain pointers and sizes, int
 * return codes, no exceptions, no torch / OpenCV / Eigen types.  The reference has no
 * FFI for this path -- its boundary is the C++ class surface
 *   openvslam::feature::orb_extractor                       (src/openvslam/feature/orb_extractor.h)
 *   openvslam::match::{area,projection,robust,stereo}       (src/openvslam/match/*.h)
 *   openvslam::optimize::{pose_optimizer,local_bundle_adjuster} (src/openvslam/optimize/*.h)
 * [file names as recalled in SURVEY.md 8(a); /root/reference holds no source, so no line
 * numbers can be cited].  include/openvslam_b200/*.h re-declares those classes on top of the
 * entry points below; INTEGRATION.md shows the binding a maintainer adds.
 *
 * Conventions
 *  - every function returns OVS_OK (0) or a negative OVS_ERR_* code; ovs_last_error()
 *    returns a thread-local message for the last failure.
 *  - handles own their CUDA stream, device buffers and pinned staging; a handle must not be
 *    used from two threads at once (the reference uses one extractor per camera, and the
 *    stereo frame constructor runs two extractor instances on two threads).
 *  - *_host entry points take HOST buffers (copies are inside the call); *_device entry points
 *    take DEVICE buffers and leave results on the device.
 *  - there is no CPU fallback: if no sm_90 (H100) device is present, *_create fails.
 */
#ifndef OVS_B200_H
#define OVS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVS_OK 0
#define OVS_ERR_INVALID_ARG (-1)
#define OVS_ERR_CUDA (-2)
#define OVS_ERR_NO_DEVICE (-3)
#define OVS_ERR_CAPACITY (-4)      /* caller-provided output capacity too small */
#define OVS_ERR_OVERFLOW (-5)      /* an internal buffer overflowed: the extractor sizes its candidate and selection buffers
                                      from bounds that hold for every image, so this reports a library defect */
#define OVS_ERR_UNSUPPORTED (-6)
#define OVS_ERR_NUMERIC (-7)       /* linear solve failed (not positive definite) */

const char* ovs_last_error(void);
/* Library / build identification: "ovs_b200 <version> sm_90a". */
const char* ovs_version(void);
/* Number of CUDA kernels launched by this library in the calling process so far. */
uint64_t ovs_kernel_launch_count(void);
/* How host threads wait for the device inside the calls below.  0 (default): spin -- lowest latency, right for one
 * camera stream per GPU.  1: sleep on a blocking CUDA event (frees the core; ~100 us per wake-up).  2: poll with
 * sched_yield() -- near-spin latency while cores are free, fair sharing once host threads outnumber cores.
 * Process-wide; call it before creating the handles it should apply to. */
int ovs_set_wait_mode(int mode);
/* Number of times the calling process's threads have waited inside this library for the device to finish (stream or event
 * synchronisations), so far. */
uint64_t ovs_host_wait_count(void);

/* ------------------------------------------------------------------ feature::orb_extractor */

/* openvslam::feature::orb_params (feature/orb_params.h): same field names. */
typedef struct {
    uint32_t max_num_keypts;   /* Feature.max_num_keypoints */
    float scale_factor;        /* Feature.scale_factor */
    uint32_t num_levels;       /* Feature.num_levels (1..16) */
    uint32_t ini_fast_thr;     /* Feature.ini_fast_threshold */
    uint32_t min_fast_thr;     /* Feature.min_fast_threshold */
} ovs_orb_params;

/* Binary-compatible with cv::KeyPoint (28 bytes): pt.x, pt.y, size, angle, response, octave,
 * class_id -- so a std::vector<cv::KeyPoint>::data() can be passed directly. */
typedef struct {
    float x, y;
    float size;
    float angle;
    float response;
    int32_t octave;
    int32_t class_id;
} ovs_keypoint;

typedef struct ovs_extractor ovs_extractor;

/* orb_extractor::orb_extractor(const orb_params&) + mask_rects_ ({x_min,x_max,y_min,y_max} in
 * [0,1] each, num_mask_rects*4 floats, may be NULL).  `device` is the CUDA ordinal. */
int ovs_extractor_create(const ovs_orb_params* params, const float* mask_rects, int num_mask_rects,
                         int device, ovs_extractor** out);
void ovs_extractor_destroy(ovs_extractor* h);

/* Upper bound on the number of keypoints one extract() can return for this handle
 * (max_num_keypts + 3 per level: the tree distribution may overshoot by < 4 per level). */
int ovs_extractor_max_keypoints(const ovs_extractor* h);

/* orb_extractor::extract(in_image, in_image_mask, keypts, out_descriptors), HOST buffers.
 *  image: CV_8UC1, `pitch` bytes per row.  mask: CV_8UC1 same size or NULL (0 = masked out).
 *  keypts_out[capacity], descriptors_out[capacity*32]; *num_out receives the count. */
int ovs_extract_host(ovs_extractor* h, const uint8_t* image, int width, int height, size_t pitch,
                     const uint8_t* mask, size_t mask_pitch,
                     ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out);

/* util::convert_to_grayscale(img, color_order) + extract() in one call (SURVEY 8f rank 3): `image` is CV_8UC3 or CV_8UC4
 * (`channels`), `pitch` bytes per row, channel order OVS_COLOR_ORDER_BGR (BGR / BGRA) or OVS_COLOR_ORDER_RGB (RGB / RGBA);
 * the gray conversion is cv::cvtColor's 15-bit fixed point (OpenCV 4), bit-exact, done on the device. */
#define OVS_COLOR_ORDER_BGR 0
#define OVS_COLOR_ORDER_RGB 1
int ovs_extract_host_color(ovs_extractor* h, const uint8_t* image, int width, int height, size_t pitch, int channels, int color_order,
                           const uint8_t* mask, size_t mask_pitch,
                           ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out);

/* Same, DEVICE image in / DEVICE keypoints + descriptors out (they stay resident for the
 * matchers).  The mask, if any, is still a HOST buffer (it only drives host-side cell and
 * keypoint filtering, as in the reference). */
int ovs_extract_device(ovs_extractor* h, const uint8_t* d_image, int width, int height, size_t pitch,
                       const uint8_t* mask, size_t mask_pitch,
                       ovs_keypoint* d_keypts_out, uint8_t* d_descriptors_out, int capacity, int* num_out);

/* orb_extractor::image_pyramid_ (public member read by match::stereo): geometry and device
 * pointer of level `level` of the last extract(); and a host copy. */
int ovs_extractor_pyramid_level(const ovs_extractor* h, int level, const uint8_t** d_ptr, size_t* pitch,
                                int* width, int* height);
int ovs_extractor_copy_pyramid_level(ovs_extractor* h, int level, uint8_t* out, size_t out_pitch);
/* orb_extractor::scale_factors_ etc. (filled by orb_params::calc_scale_factors). */
int ovs_extractor_scale_factors(const ovs_extractor* h, float* scale_factors, float* inv_scale_factors,
                                float* level_sigma_sq, float* inv_level_sigma_sq);

/* Stage taps for the parity tests (device -> host copies of intermediate results of the last
 * extract()): FAST score map of a level (0 where score < min_fast_thr), and the candidate list
 * (x, y relative to the 19 px border, score) that went into the tree distribution. */
int ovs_extractor_debug_score_map(ovs_extractor* h, int level, uint8_t* out, size_t out_pitch);
int ovs_extractor_debug_candidates(ovs_extractor* h, int level, int32_t* xys_out /* [cap*3] */, int cap, int* n_out);
/* Per-stage device time of the last extract() in microseconds (CUDA events):
 * [0] upload [1] pyramid [2] fast score [3] cell nms+compact [4] host tree distribution (wall)
 * [5] orientation+descriptor [6] download [7] total wall. */
int ovs_extractor_last_timings(const ovs_extractor* h, float* out_us /* [8] */);

/* ------------------------------------------------------------------------- util::stereo_rectifier */

typedef struct ovs_stereo_rectifier ovs_stereo_rectifier;

/* util::stereo_rectifier(camera, StereoRectifier params): the rectification maps of both cameras of a stereo rig, as
 * cv::initUndistortRectifyMap (model OVS_CAMERA_PERSPECTIVE, dist = k1, k2, p1, p2, k3) or cv::fisheye::initUndistortRectifyMap
 * (OVS_CAMERA_FISHEYE, dist = k1..k4) build them with CV_32FC1 maps, for cols x rows images (1 .. 32767 each).  K_*, R_* and
 * K_rect are row-major 3 x 3; K_rect is the rectified camera matrix (the camera's own K).  The maps are built on `device`
 * (float64, evaluated as OpenCV writes it; the fisheye model's atan is within an ulp of the host's) and the handle is
 * immutable once create returns, so any number of threads may read it at once.  A singular K_rect R, an unknown model or
 * a null array return OVS_ERR_INVALID_ARG. */
int ovs_stereo_rectifier_create(int device, int model, int cols, int rows, const double* K_l, const double* D_l, const double* R_l,
                                const double* K_r, const double* D_r, const double* R_r, const double* K_rect,
                                ovs_stereo_rectifier** out);
void ovs_stereo_rectifier_destroy(ovs_stereo_rectifier* h);
/* The float maps of side 0 (left) or 1 (right): map_x[rows * cols], map_y[rows * cols], host buffers. */
int ovs_stereo_rectifier_maps(const ovs_stereo_rectifier* h, int side, float* map_x, float* map_y);
/* util::stereo_rectifier::rectify(in_l, in_r, out_l, out_r): cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of both u8 images
 * (1, 3 or 4 interleaved channels, `pitch` bytes per row) through their maps, bit-exact with OpenCV 4; the outputs have the
 * input's channels, `out_pitch` bytes per row.  Calls on one handle from several threads run one after the other. */
int ovs_stereo_rectify_host(ovs_stereo_rectifier* h, const uint8_t* left, const uint8_t* right, int width, int height, size_t pitch,
                            int channels, uint8_t* out_left, uint8_t* out_right, size_t out_pitch);
/* rectify one side, util::convert_to_grayscale (color_order as ovs_extract_host_color; ignored for 1 channel) and
 * orb_extractor::extract in one call: the raw image is uploaded and remapped straight into level 0 of the pyramid, with one
 * host synchronisation.  The mask is in rectified coordinates.  Call it per side on the stereo frame's two extractors, from
 * two threads if wanted: both may read one rectifier at once.  An image whose size differs from the rectifier's, channels
 * other than 1 / 3 / 4, side outside {0, 1}, a null pointer, or a rectifier on another device than the extractor return
 * OVS_ERR_INVALID_ARG before any launch. */
int ovs_extract_host_rectified(ovs_extractor* h, const ovs_stereo_rectifier* rectifier, int side, const uint8_t* image, int width,
                               int height, size_t pitch, int channels, int color_order, const uint8_t* mask, size_t mask_pitch,
                               ovs_keypoint* keypts_out, uint8_t* descriptors_out, int capacity, int* num_out);

/* ------------------------------------------------------------------------------- match::* */

/* match::base constants (match/base.h). */
#define OVS_HAMMING_DIST_THR_LOW 50
#define OVS_HAMMING_DIST_THR_HIGH 100
#define OVS_MAX_HAMMING_DIST 256

/* Length of the per-query candidate lists of the brute-force search. */
#define OVS_MATCH_TOPK 8

typedef struct ovs_matcher ovs_matcher;
int ovs_matcher_create(int device, ovs_matcher** out);
void ovs_matcher_destroy(ovs_matcher* h);

/* Hamming brute force (the inner double loop of match::robust::brute_force_match, match/robust.cc,
 * with match::compute_descriptor_distance_32, match/base.h): for each of the nq query descriptors
 * the OVS_MATCH_TOPK (8) smallest keys (distance << 16 | train index) over the nt train descriptors, ascending, i.e.
 * exactly the order a sequential `<` scan ranks them (lowest index wins ties).  Missing entries
 * (nt < 8) are 0xFFFFFFFF.  nt must be < 65536.  keys_out[nq * 8].  Descriptors are 32 bytes each,
 * device pointers 16-byte aligned. */
int ovs_match_bruteforce_topk_host(ovs_matcher* h, const uint8_t* query, int nq, const uint8_t* train, int nt,
                                   uint32_t* keys_out);
int ovs_match_bruteforce_topk_device(ovs_matcher* h, const uint8_t* d_query, int nq, const uint8_t* d_train, int nt,
                                     uint32_t* d_keys_out);
/* match::robust::match_for_triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs) (match/robust.cc) on plain arrays.
 * The BoW feature vectors are inputs: bow_node_k[i] = vocabulary node of keypoint i of keyframe k (keyfrm->bow_feat_vec_
 * inverted; < 0 = none).  bearing_k[n*3] = keyfrm->bearings_ (f64), octave_1 / angle_k = undist_keypts_, has_lm_k[i] =
 * keyfrm->get_landmark(i) != nullptr, is_stereo_k[i] = stereo_x_right_[i] >= 0 (NULL = monocular), E_12[9] row-major,
 * epipole_in_2[3] = camera centre of keyframe 1 reprojected to a bearing of keyframe 2, scale_factors_1 = keyfrm_1->
 * scale_factors_.  Candidates are the keyframe-2 keypoints of the same node without a landmark, distance <=
 * HAMMING_DIST_THR_LOW, not within cos 0.998 of the epipole (monocular pairs), inside 0.2 deg x scale of the epipolar
 * plane (check_epipolar_constraint); first taker keeps a keyframe-2 keypoint; orientation histogram if requested.
 * matched_idx_2_of_1[n1] = keypoint of keyframe 2 or -1; *num_matches = the reference's return value. */
int ovs_robust_match_for_triangulation_host(ovs_matcher* m, int n1, const uint8_t* desc_1, const double* bearing_1, const int32_t* octave_1,
                                            const float* angle_1, const uint8_t* has_lm_1, const uint8_t* is_stereo_1, const int32_t* bow_node_1,
                                            int n2, const uint8_t* desc_2, const double* bearing_2, const float* angle_2, const uint8_t* has_lm_2,
                                            const uint8_t* is_stereo_2, const int32_t* bow_node_2, const double* E_12, const double* epipole_in_2,
                                            const float* scale_factors_1, int num_scale_levels, int check_orientation,
                                            int32_t* matched_idx_2_of_1, int* num_matches);

/* Convenience view of the same search: best index (-1 if none), best and second-best distance
 * (OVS_MAX_HAMMING_DIST when absent) of desc1[i] over desc2. */
int ovs_match_bruteforce_host(ovs_matcher* h, const uint8_t* desc1, int n1, const uint8_t* desc2, int n2,
                              int32_t* best_idx, int32_t* best_dist, int32_t* second_dist);

/* match::robust::brute_force_match(frm, keyfrm, matches) (match/robust.cc) on plain arrays:
 *  desc_frm[n1*32]: frm.descriptors_;  desc_keyfrm[n2*32]: keyfrm->descriptors_;
 *  lm_valid_2[n2]: 1 where keyfrm->get_landmarks()[idx_2] is non-null and not will_be_erased()
 *  (NULL = all valid);  lowe_ratio: robust::lowe_ratio_.
 * Output pairs (idx_1 in frame, idx_2 in keyframe) in the reference's emission order (ascending
 * idx_2), with its greedy "a frame keypoint is matched at most once" rule.  Returns the count in
 * *num_matches (the reference's return value). */
int ovs_robust_brute_force_match_host(ovs_matcher* h, const uint8_t* desc_frm, int n1, const uint8_t* desc_keyfrm, int n2,
                                      const uint8_t* lm_valid_2, float lowe_ratio,
                                      int32_t* pairs_out, int capacity, int* num_matches);
/* The same with both descriptor sets resident in device memory (16-byte aligned; e.g. the output of ovs_extract_device):
 * only the per-keypoint candidate lists travel to the host for the sequential replay.  lm_valid_2 / pairs_out: host. */
int ovs_robust_brute_force_match_device(ovs_matcher* h, const uint8_t* d_desc_frm, int n1, const uint8_t* d_desc_keyfrm, int n2,
                                        const uint8_t* lm_valid_2, float lowe_ratio,
                                        int32_t* pairs_out, int capacity, int* num_matches);
/* solve::essential_solver(bearings_1, bearings_2, matches_12).find_via_ransac(max_num_iter, recompute) (solve/essential_solver.cc)
 * for B independent problems in one call.  Problem b owns the matches match_offsets[b] .. match_offsets[b + 1] - 1
 * (match_offsets[0] = 0, non-decreasing); the bearings are gathered per match: bearings_1[i*3] = bearings_1_[matches_12_[i].first],
 * bearings_2[i*3] = bearings_2_[matches_12_[i].second] (unit; any camera model: ovs_undistort_keypoints_* produces them).
 * seeds[B]: the sampler's seed per problem (a problem gives the same result alone or inside a batch).
 * Per problem: E_21[b*9] = get_best_E_21() row-major (b2^T E_21 b1 = 0; zero when no hypothesis scored above 0), valid[b] =
 * solution_is_valid() (best score > 0 and at least 8 inliers), num_inliers[b] = the number of inlier flags set, best_iter[b] = the best
 * hypothesis (-1: none), best_score[b] = its score (after the recompute, when one ran), inlier_out[n] = get_inlier_matches().
 * Fewer than 8 matches: no hypothesis runs and the problem is invalid.  With recompute, a valid problem is solved again by the
 * eight-point algorithm on all inliers and its flags, count and score are re-checked at that E_21 (valid keeps its value).  The
 * sampler, the rank-2 projection, the inlier test, the score and their fixed summation orders are described in DESIGN.md section 5.
 * B outside 0 .. 65535, invalid offsets, a bearing that is not finite or not unit (|b.b - 1| > 1e-6) or a negative max_num_iter
 * return OVS_ERR_INVALID_ARG; B == 0 or no match at all returns without a launch.  Otherwise the call is three launches (one with
 * max_num_iter == 0), one copy each way and one wait.  The solve has its own buffers on the handle: the brute-force entry points
 * above are unaffected by it. */
int ovs_essential_solve_ransac_host(ovs_matcher* h, int B, const int32_t* match_offsets, const double* bearings_1, const double* bearings_2,
                                    int max_num_iter, int recompute, const uint64_t* seeds, double* E_21, uint8_t* valid,
                                    int32_t* num_inliers, int32_t* best_iter, double* best_score, uint8_t* inlier_out);
/* solve::homography_solver(undist_keypts_1, undist_keypts_2, matches_12, sigma).find_via_ransac(max_num_iter, recompute) and
 * solve::fundamental_solver(...) the same way (solve/{homography,fundamental}_solver.cc): the two solvers perspective map
 * initialisation runs on each frame (it passes sigma = 1.0 and recompute = true), for B independent problems in one call.
 * Problem b owns the keypoints keypt_offsets_1[b] .. keypt_offsets_1[b + 1] - 1 of keypts_1 (ALL of view 1's undistorted
 * keypoints: undist_keypts_.data() can be passed; only pt is read), the same of keypts_2 through keypt_offsets_2, and the matches
 * match_offsets[b] .. match_offsets[b + 1] - 1 of matches_12 (2 per match: idx_1, idx_2, indices into the problem's own keypoints).
 * Every offset array starts at 0 and is non-decreasing.  seeds[B]: the sampler's seed per problem (a problem gives the same
 * result alone or inside a batch).  Each view is normalised over all of its keypoints; hypotheses are solved on 8 matches.
 * Per problem: H_21[b*9] / F_21[b*9] row-major (p2 ~ H_21 p1, p2^T F_21 p1 = 0, pixel coordinates; the entry of largest magnitude
 * positive; zero when no hypothesis scored above 0), valid[b] = solution_is_valid() (best score > 0 and at least 8 inliers),
 * num_inliers[b] = the number of inlier flags set, best_iter[b] = the best hypothesis (-1: none), best_score[b] = get_best_score()
 * (after the recompute, when one ran), inlier_out[m] = get_inlier_matches().  Fewer than 8 matches: no hypothesis runs and the
 * problem is invalid.  With recompute, a valid problem is solved again on all inliers and its flags, count and score are re-checked
 * (valid keeps its value).  The conventions (normalisation, minimal solves, the inlier tests and score, their summation orders) are
 * in DESIGN.md section 5.  B outside 0 .. 65535, invalid offsets, a match index outside its problem's keypoints, a keypoint
 * coordinate that is not finite, sigma <= 0 (or not finite) or a negative max_num_iter return OVS_ERR_INVALID_ARG before any
 * launch; B == 0 or no match at all returns without a launch.  Otherwise the call is four launches (one with max_num_iter == 0),
 * one copy each way and one wait.  The solve has its own buffers on the handle: the brute-force and essential entry points are
 * unaffected by it. */
int ovs_homography_solve_ransac_host(ovs_matcher* h, int B, const int32_t* keypt_offsets_1, const ovs_keypoint* keypts_1,
                                     const int32_t* keypt_offsets_2, const ovs_keypoint* keypts_2, const int32_t* match_offsets,
                                     const int32_t* matches_12, float sigma, int max_num_iter, int recompute, const uint64_t* seeds,
                                     double* H_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                     uint8_t* inlier_out);
int ovs_fundamental_solve_ransac_host(ovs_matcher* h, int B, const int32_t* keypt_offsets_1, const ovs_keypoint* keypts_1,
                                      const int32_t* keypt_offsets_2, const ovs_keypoint* keypts_2, const int32_t* match_offsets,
                                      const int32_t* matches_12, float sigma, int max_num_iter, int recompute, const uint64_t* seeds,
                                      double* F_21, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, double* best_score,
                                      uint8_t* inlier_out);
/* match::robust::match_frame_and_keyframe(frm, keyfrm, matched_lms_in_frm) (match/robust.cc), the tracker's robust-match fallback:
 * ovs_robust_brute_force_match_host (the same pairs, bit for bit), then the essential solver on them with recompute off
 * (the reference calls find_via_ransac(50, false); pass max_num_iter = 50).  bearings_frm[n1*3] = frm.bearings_,
 * bearings_keyfrm[n2*3] = keyfrm->bearings_ (unit), gathered by pair index on the device; seed: the sampler's seed.
 * matched_keyfrm_idx_of_frm[n1] = idx_2 of the inlier pair of frame keypoint idx_1 (the keypoint whose landmark
 * matched_lms_in_frm[idx_1] receives) or -1; *num_inlier_matches = the reference's return value (0 when the solution is invalid,
 * e.g. with fewer than 8 pairs). */
int ovs_robust_match_frame_and_keyframe_host(ovs_matcher* h, const uint8_t* desc_frm, const double* bearings_frm, int n1,
                                             const uint8_t* desc_keyfrm, const double* bearings_keyfrm, int n2, const uint8_t* lm_valid_2,
                                             float lowe_ratio, int max_num_iter, uint64_t seed, int32_t* matched_keyfrm_idx_of_frm,
                                             int* num_inlier_matches);
/* The same with descriptors and bearings resident in device memory (the outputs of ovs_extract_device and
 * ovs_undistort_keypoints_device; descriptors 16-byte aligned): only the pair list goes to the device and the flags come back.
 * lm_valid_2 / matched_keyfrm_idx_of_frm: host. */
int ovs_robust_match_frame_and_keyframe_device(ovs_matcher* h, const uint8_t* d_desc_frm, const double* d_bearings_frm, int n1,
                                               const uint8_t* d_desc_keyfrm, const double* d_bearings_keyfrm, int n2, const uint8_t* lm_valid_2,
                                               float lowe_ratio, int max_num_iter, uint64_t seed, int32_t* matched_keyfrm_idx_of_frm,
                                               int* num_inlier_matches);
/* Diagnostic: how many single-query GPU re-searches the greedy replays of this handle have needed. */
int ovs_matcher_num_requeries(const ovs_matcher* h, int* out);
/* Device time (CUDA events, microseconds) of the Hamming kernels of the last call. */
int ovs_matcher_last_kernel_us(const ovs_matcher* h, float* out_us);
/* Development aids / test hooks: the kernels behind the greedy replays' GPU re-queries, on host arrays, with the launch geometry
 * and the handle buffers of the entry points that use them; keys as in their candidate lists (8 per query, ascending,
 * 0xFFFFFFFF past the end).
 *  ovs_debug_hamming_one: the brute-force re-query of one 32-byte query over nt (1 .. 65535) train descriptors, train
 *    descriptor j skipped where bit j & 31 of exclude_mask[j >> 5] is set; keys (distance << 16 | j) in keys_out[8].
 *  ovs_debug_node_topk: the bow_tree lists; query k's candidates are ranks qseg[2k] .. qseg[2k + 1] - 1 of tdesc[R * 32],
 *    keys (distance << 16 | rank).  q0 < 0: the list launch over all nq queries, a candidate r with taken[r] != 0 skipped
 *    (taken may be NULL), keys_out[nq * 8].  q0 >= 0: the list launch without taken, then the re-query of query q0 alone with
 *    taken, its list in the spare row nq, keys_out[(nq + 1) * 8].
 *  ovs_debug_triangulation_topk: the match_for_triangulation lists (batched == 0: one problem, nprob == 1 and
 *    queries_per_prob == nq) or create_new_landmarks' batched lists (nq == nprob * queries_per_prob; query q of problem
 *    p = q / queries_per_prob reads keypoint entry q - p * queries_per_prob, E_12 prob_E[9 p], epipole prob_epipole[3 p] and
 *    the candidates and taken flags from prob_tbase[p] on, qseg relative to that base); the distance, epipole and epipolar tests
 *    of ovs_robust_match_for_triangulation_host, keys (distance << 16 | 0xFFFF - rank).  q0 and taken as ovs_debug_node_topk. */
int ovs_debug_hamming_one(ovs_matcher* h, const uint8_t* query, const uint8_t* train, int nt, const uint32_t* exclude_mask, uint32_t* keys_out);
int ovs_debug_node_topk(ovs_matcher* h, int nq, const uint8_t* qdesc, const int32_t* qseg, int R, const uint8_t* tdesc, const uint8_t* taken,
                        int q0, uint32_t* keys_out);
int ovs_debug_triangulation_topk(ovs_matcher* h, int batched, int nq, int queries_per_prob, const uint8_t* qdesc, const double* qbearing,
                                 const float* qscale, const uint8_t* qstereo, const int32_t* qseg, int R, const uint8_t* tdesc,
                                 const double* tbearing, const uint8_t* tstereo, int nprob, const double* prob_E, const double* prob_epipole,
                                 const int32_t* prob_tbase, const uint8_t* taken, int q0, uint32_t* keys_out);

/* ---- windowed search: match::projection / match::area (match/projection.cc, match/area.cc) ---- */

/* The part of camera::base that data::frame::get_keypoints_in_cell reads (camera/base.h):
 * img_bounds_.min_x_/min_y_, inv_cell_width_, inv_cell_height_, num_grid_cols_ (64), num_grid_rows_ (48). */
typedef struct {
    float min_x, min_y;
    float inv_cell_width, inv_cell_height;
    int32_t num_grid_cols, num_grid_rows;
} ovs_grid;

/* A frame's keypoints uploaded once and indexed by grid cell (data::assign_keypoints_to_grid,
 * data/common.cc): x/y/octave/angle = undist_keypts_[i].{pt, octave, angle}, x_right =
 * stereo_x_right_ (NULL: monocular), desc = descriptors_.  Owned by the matcher `m` (its stream). */
typedef struct ovs_frame_index ovs_frame_index;
int ovs_frame_index_create(ovs_matcher* m, int n, const float* x, const float* y, const int32_t* octave, const float* angle,
                           const float* x_right, const uint8_t* desc, const ovs_grid* grid, ovs_frame_index** out);
/* The same index built from the DEVICE output of ovs_extract_device (keypoint records + descriptors, optionally the
 * stereo x_right array, all device pointers; descriptors 16-byte aligned): the descriptors are never copied to the host
 * (SURVEY 8f rank 1: data::frame grid + device-resident descriptors).  The matcher's stream must be ordered after the
 * extraction that produced the arrays (ovs_extract_device returns with its stream drained). */
int ovs_frame_index_create_device(ovs_matcher* m, int n, const ovs_keypoint* d_keypts, const uint8_t* d_desc, const float* d_x_right,
                                  const ovs_grid* grid, ovs_frame_index** out);
void ovs_frame_index_destroy(ovs_frame_index* f);

/* frame::get_keypoints_in_cell(ref_x, ref_y, margin, min_level, max_level) followed by the nearest
 * descriptor search every projection matcher performs, for nq queries at once: the 4 best candidates
 * of each query (index into the frame's keypoints and Hamming distance; -1 / 256 where absent) in
 * the reference's candidate order (ties: first visited wins).  x_right_q may be NULL. */
int ovs_match_window_topk_host(ovs_frame_index* f, int nq, const float* ref_xy, const float* margin, const int32_t* min_level,
                               const int32_t* max_level, const float* x_right_q, const uint8_t* qdesc,
                               int32_t* idx_out, int32_t* dist_out);

/* match::projection::match_frame_and_landmarks(frm, local_landmarks, margin):
 *  lm_usable[l] = is_observable_in_tracking_ && !will_be_erased();  reproj_xy / x_right_in_tracking /
 *  pred_scale_level = the landmark's reproj_in_tracking_, x_right_in_tracking_, scale_level_in_tracking_;
 *  lm_desc = get_descriptor();  kp_has_observed_lm[i] = frm.landmarks_[i] && has_observation().
 * matched_lm_of_kp[i] receives the landmark index assigned to frm.landmarks_[i] by this call (-1: none). */
int ovs_projection_match_frame_and_landmarks_host(ovs_frame_index* f, const float* scale_factors, int num_scale_levels, int nlm, const uint8_t* lm_usable,
                                                  const float* reproj_xy, const float* x_right_in_tracking,
                                                  const int32_t* pred_scale_level, const uint8_t* lm_desc,
                                                  const uint8_t* kp_has_observed_lm, float margin, float lowe_ratio,
                                                  int32_t* matched_lm_of_kp, int* num_matches);

/* match::projection::match_current_and_last_frames(curr_frm, last_frm, margin): one entry per keypoint
 * of the last frame.  last_usable[i] = it has a landmark, is not an outlier and reprojects into the
 * current image (camera->reproject_to_image, evaluated by the caller as in the reference);
 * reproj_xy / reproj_x_right = that reprojection; last_scale_level / last_angle = last_frm keypoint
 * octave / undistorted angle; lm_desc = landmark descriptors.  assume_forward / assume_backward as
 * computed from trans_lc.  matched_last_of_kp[i] = index in the last frame or -1. */
int ovs_projection_match_current_and_last_host(ovs_frame_index* curr, const float* scale_factors, int num_scale_levels, int n_last,
                                               const uint8_t* last_usable, const float* reproj_xy, const float* reproj_x_right,
                                               const int32_t* last_scale_level, const float* last_angle, const uint8_t* lm_desc,
                                               const uint8_t* kp_has_observed_lm, float margin, int assume_forward, int assume_backward,
                                               int check_orientation, int32_t* matched_last_of_kp, int* num_matches);

/* The search loop shared by projection::match_current_and_last_frames, match_frame_and_keyframe,
 * match_by_Sim3_transform and each direction of match_keyframes_mutually (match/projection.cc): one
 * query per reprojected landmark -- usable[i] (NULL = all), reprojection ref_xy, optional reprojected
 * x_right (NULL: the x_right test is not part of the matcher), search margin (already multiplied by
 * the scale factor of the predicted level), level range [min_level, max_level] (max < 0: unbounded),
 * descriptor, keypoint/landmark angle (for the orientation check).  kp_unavailable[i] marks frame
 * keypoints that must not be matched (already associated).  A query takes its nearest available
 * keypoint when the distance is <= hamm_dist_thr; queries are served in index order and a keypoint is
 * given to the first taker, as in the reference loops.  matched_query_of_kp[i] = query index or -1. */
int ovs_projection_match_best_host(ovs_frame_index* f, int nq, const uint8_t* usable, const float* ref_xy, const float* ref_x_right,
                                   const float* margin, const int32_t* min_level, const int32_t* max_level, const float* q_angle,
                                   const uint8_t* q_desc, const uint8_t* kp_unavailable, unsigned hamm_dist_thr, int check_orientation,
                                   int32_t* matched_query_of_kp, int* num_matches);

/* match::projection::match_keyframes_mutually(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, Sim3_12, Sim3_21, margin)
 * (match/projection.cc, loop closure).  Landmark arrays are indexed by the keypoint of the keyframe they belong to
 * (keyfrm->landmarks_): usable_k[i] = landmark present, not bad, not already matched, reprojection inside the other
 * image; reproj_a_in_b / pred_level_a_in_b = its reprojection with the Sim3 and predict_scale_level(); lm_desc = the
 * landmark's representative descriptor.  Each landmark takes its nearest keypoint of the other keyframe in the window
 * margin * scale_factors[level], levels [level - 1, level], distance <= HAMMING_DIST_THR_HIGH; pairs on which both
 * directions agree are returned: matched_idx_2_of_kp_1[i1] = keypoint of keyframe 2 or -1 (f1->n entries). */
int ovs_projection_match_keyframes_mutually_host(ovs_frame_index* f1, ovs_frame_index* f2, const float* scale_factors,
                                                 const uint8_t* usable_1, const float* reproj_1_in_2, const int32_t* pred_level_1_in_2,
                                                 const uint8_t* lm_desc_1, const uint8_t* usable_2, const float* reproj_2_in_1,
                                                 const int32_t* pred_level_2_in_1, const uint8_t* lm_desc_2, float margin,
                                                 int32_t* matched_idx_2_of_kp_1, int* num_matches);

/* match::area::match_in_consistent_area(frm_1, frm_2, prev_matched_pts, matched_indices_2_in_frm_1, margin):
 * f2 indexes frm_2; octave_1 / angle_1 / desc_1 describe frm_1's keypoints; prev_matched_xy[n1*2] is
 * updated in place. */
int ovs_area_match_in_consistent_area_host(ovs_frame_index* f2, int n1, const int32_t* octave_1, const float* angle_1, const uint8_t* desc_1,
                                           float* prev_matched_xy, int32_t* matched_idx_2_in_1, int margin, float lowe_ratio,
                                           int check_orientation, int* num_matches);

/* match::stereo(left_image_pyramid, right_image_pyramid, keypts_left, keypts_right, descs_left,
 * descs_right, scale_factors, inv_scale_factors, focal_x_baseline, true_baseline)
 *   .compute(stereo_x_right, depths)  (match/stereo.cc).
 * The pyramids are read from the two extractors (device resident, after their extract() of the pair). */
int ovs_stereo_compute_host(ovs_matcher* m, const ovs_extractor* left, const ovs_extractor* right,
                            int n_left, const float* lx, const float* ly, const int32_t* loct, const uint8_t* ldesc,
                            int n_right, const float* rx, const float* ry, const int32_t* roct, const uint8_t* rdesc,
                            float focal_x_baseline, float true_baseline, float* stereo_x_right, float* depths, int* num_matched);

/* ------------------------------------------------------------------------------ optimize::* */

#define OVS_CAMERA_PERSPECTIVE 0       /* camera::perspective (and fisheye: same edges on undistorted keypoints) */
#define OVS_CAMERA_EQUIRECTANGULAR 1   /* camera::equirectangular */
#define OVS_CAMERA_FISHEYE 2           /* camera::fisheye -- ovs_undistort_keypoints_* only (matchers / optimisers see it as perspective) */
#define OVS_CAMERA_RADIAL_DIVISION 3   /* camera::radial_division -- ovs_undistort_keypoints_* only */

/* The camera parameters the reprojection edges read (optimize/g2o/se3/ *_edge.h): fx_, fy_, cx_, cy_,
 * focal_x_baseline_ (stereo / RGBD), cols_, rows_ (equirectangular). */
typedef struct {
    int32_t model;
    double fx, fy, cx, cy, focal_x_baseline;
    double cols, rows;
} ovs_camera;

/* ---- tracking: frame::can_observe and the reprojections of the two projection searches (data/frame.cc, data/landmark.cc,
 * camera/perspective.cc, camera/equirectangular.cc,
 * module/tracking_module.cc search_local_landmarks, module/frame_tracker.cc motion_based_track) ---- */

/* What the tracker's geometry reads of the current frame: camera_ (OVS_CAMERA_PERSPECTIVE, FISHEYE and RADIAL_DIVISION all
 * reproject with the pinhole formula on undistorted keypoints; EQUIRECTANGULAR), camera_->img_bounds_ (min/max x/y; not read
 * for equirectangular), rot_cw_ / trans_cw_ (row-major), cam_center_ (as the frame holds it: the library does not derive it),
 * num_scale_levels_ (1 .. 16) and log_scale_factor_. */
typedef struct {
    ovs_camera camera;
    float min_x, max_x, min_y, max_y;
    double rot_cw[9], trans_cw[3], cam_center[3];
    int32_t num_scale_levels;
    float log_scale_factor;
} ovs_frame_geometry;

/* frame::can_observe(lm, ray_cos_thr, reproj, x_right, pred_scale_level) for nlm landmarks in one launch (one copy each way, one
 * wait).  usable[l] (NULL: all) = the tracker's skip rule: the landmark is present, not will_be_erased() and not already
 * observed in the frame.  pos_w[nlm*3] = get_pos_in_world(); mean_normal[nlm*3] = get_obs_mean_normal(); min_valid_dist /
 * max_valid_dist = the landmark's raw min_valid_dist_ / max_valid_dist_ (the 0.7 / 1.3 factors are applied inside).  Outputs:
 * observable[l]; where observable, reproj_xy[l*2] (the double reprojection rounded to float), x_right[l] (-1 equirectangular)
 * and pred_scale_level[l] (landmark::predict_scale_level); elsewhere 0, 0, 0 and 0.  The conventions (summation orders, the
 * float scale range, the double ray test, the level's log) are in DESIGN.md section 5.
 * OVS_ERR_INVALID_ARG before any launch: nlm < 0, a null array with nlm > 0, an unknown camera model, num_scale_levels outside
 * 1 .. 16, a log_scale_factor <= 0 or not finite, a non-finite pose or camera centre.  nlm == 0 returns without a launch. */
int ovs_frame_can_observe_host(ovs_matcher* m, const ovs_frame_geometry* geometry, int nlm, const uint8_t* usable, const double* pos_w,
                               const double* mean_normal, const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr,
                               uint8_t* observable, float* reproj_xy, float* x_right, int32_t* pred_scale_level);

/* The compute of tracking_module::search_local_landmarks: ovs_frame_can_observe_host on the matcher of f, then
 * ovs_projection_match_frame_and_landmarks_host(f, scale_factors, num_scale_levels, nlm, observable, reproj_xy, x_right,
 * pred_scale_level, lm_desc, kp_has_observed_lm, margin, lowe_ratio, ...) on those outputs: the same matcher and first-taker
 * replay, so one launch more than that call.  scale_factors[num_scale_levels] = scale_factors_; lm_desc[nlm*32] =
 * get_descriptor().  The per-landmark outputs are returned so that the caller can set reproj_in_tracking_,
 * x_right_in_tracking_, scale_level_in_tracking_ and is_observable_in_tracking_ and call increase_num_observable().  Checks of
 * ovs_frame_can_observe_host plus a null scale table, descriptor or output array. */
int ovs_projection_search_local_landmarks_host(ovs_frame_index* f, const ovs_frame_geometry* geometry, const float* scale_factors, int nlm,
                                               const uint8_t* usable, const double* pos_w, const double* mean_normal,
                                               const float* min_valid_dist, const float* max_valid_dist, const uint8_t* lm_desc,
                                               const uint8_t* kp_has_observed_lm, float ray_cos_thr, float margin, float lowe_ratio,
                                               uint8_t* observable, float* reproj_xy, float* x_right, int32_t* pred_scale_level,
                                               int32_t* matched_lm_of_kp, int* num_matches);

/* match::projection::match_current_and_last_frames(curr_frm, last_frm, margin) with the reprojections made on the device: every
 * landmark of the last frame is reprojected into the current frame (camera->reproject_to_image with the current pose, one
 * launch), the direction comes from the two poses (trans_lc = R_lw (-R_cw^T t_cw) + t_lw against +-true_baseline, neither for
 * is_monocular), and ovs_projection_match_current_and_last_host runs on the in-image ones: one launch more than that call.
 * last_usable[i] (NULL: all) = last_frm.landmarks_[i] present and not an outlier; pos_w[n_last*3] = its position;
 * last_pose_cw[12] = last_frm's cam_pose_cw_ {R row-major, t}; last_octave / last_angle = last_frm.undist_keypts_[i].octave /
 * .angle; lm_desc[n_last*32] = landmark descriptors.  in_image_out[n_last] / reproj_xy_out[n_last*2] (both NULL or both given):
 * the in-image flag and the reprojection (0, 0 where not in the image).  Checks of ovs_frame_can_observe_host plus a non-finite
 * last pose or true_baseline, a null scale table, descriptor or octave array, an octave of a usable keypoint outside the scale
 * table. */
int ovs_projection_match_current_and_last_reproject_host(ovs_frame_index* curr, const ovs_frame_geometry* geometry, int is_monocular,
                                                         double true_baseline, const double* last_pose_cw, const float* scale_factors,
                                                         int n_last, const uint8_t* last_usable, const double* pos_w,
                                                         const int32_t* last_octave, const float* last_angle, const uint8_t* lm_desc,
                                                         const uint8_t* kp_has_observed_lm, float margin, int check_orientation,
                                                         int32_t* matched_last_of_kp, int* num_matches, uint8_t* in_image_out,
                                                         float* reproj_xy_out);

/* ---- local mapping: module::two_view_triangulator (module/two_view_triangulator.cc) and the compute step of
 * mapping_module::create_new_landmarks (module/mapping_module.cc) ---- */

/* What the triangulator (and, for ovs_create_new_landmarks_host, the triangulation matcher) reads of one keyframe.  The arrays
 * are the keyframe's own vectors, so `.data()` can be passed:
 *  pose_cw[12]: get_cam_pose() as {R row-major (9), t (3)};  camera: camera_ (perspective, or fisheye on undistorted
 *  keypoints passed as perspective; equirectangular); true_baseline: camera_->true_baseline_ (read for stereo keypoints only);
 *  scale_factor: scale_factor_;  scale_factors / level_sigma_sq [num_scale_levels]: scale_factors_, level_sigma_sq_;
 *  undist_keypts[num_keypts]: undist_keypts_ (pt, octave and, for the matcher, angle are read);  bearings[num_keypts*3]: bearings_
 *  (unit);  stereo_x_right / depths [num_keypts]: stereo_x_right_, depths_ (NULL, both: monocular; an equirectangular keyframe
 *  has no stereo keypoint);
 *  descriptors[num_keypts*32], has_landmark[num_keypts] (get_landmark(i) != nullptr), bow_node[num_keypts] (bow_feat_vec_
 *  inverted, < 0 = none): read by ovs_create_new_landmarks_host only (NULL elsewhere). */
typedef struct {
    double pose_cw[12];
    ovs_camera camera;
    double true_baseline;
    float scale_factor;
    int32_t num_scale_levels;
    const float* scale_factors;
    const float* level_sigma_sq;
    int32_t num_keypts;
    const ovs_keypoint* undist_keypts;
    const double* bearings;
    const float* stereo_x_right;
    const float* depths;
    const uint8_t* descriptors;
    const uint8_t* has_landmark;
    const int32_t* bow_node;
} ovs_keyframe_view;

/* module::two_view_triangulator(keyfrm_1, keyfrm_2, rays_parallax_deg_thr).triangulate(idx_1, idx_2, pos_w) for every pair of a
 * list, for B independent keyframe pairs in one call (create_new_landmarks passes 1.0 degree).  Problem b triangulates the pairs
 * pair_offsets[b] .. pair_offsets[b + 1] - 1 of pairs (2 per pair: idx_1 into keyfrms_1[b], idx_2 into keyfrms_2[b]);
 * pair_offsets[0] = 0, non-decreasing.  valid[m] = the reference's return value, pos_w[m*3] = the point (zero where invalid).
 * The conventions (world-frame rays, the closed-form stereo parallax, the branch rule, the two-camera solve by a 4x4 Jacobi
 * on A^T A, the stereo back-projection, the cheirality, reprojection and scale tests) are in DESIGN.md section 5.
 * B outside 0 .. 65535, invalid offsets, an index outside its keyframe, an octave outside the scale table, a bearing that is not a
 * finite unit vector, a stereo keypoint with a non-finite depth, an unknown camera model (or a stereo keypoint on an
 * equirectangular camera), a non-finite pose or rays_parallax_deg_thr return OVS_ERR_INVALID_ARG, and more than 2^30 - 1 pairs in
 * all OVS_ERR_UNSUPPORTED, before any launch; B == 0 or
 * no pair at all returns without a launch.  Otherwise the call is one launch, one copy each way and one wait, on buffers of its
 * own: the other entry points of the handle are unaffected. */
int ovs_two_view_triangulate_host(ovs_matcher* h, int B, const ovs_keyframe_view* keyfrms_1, const ovs_keyframe_view* keyfrms_2,
                                  const int32_t* pair_offsets, const int32_t* pairs, double rays_parallax_deg_thr, uint8_t* valid,
                                  double* pos_w);

/* ---- monocular map initialisation: initialize::perspective and initialize::bearing_vector (initialize/perspective.cc, bearing_vector.cc) ---- */

/* What an initialiser reads of one frame: camera_ (perspective -- fisheye passed as perspective on its undistorted keypoints --
 * for ovs_initialize_perspective_host, equirectangular for ovs_initialize_bearing_vector_host; fx, fy, cx, cy or cols, rows are
 * read), undist_keypts[num_keypts] = undist_keypts_.data() (pt is read), bearings[num_keypts*3] = bearings_ (unit). */
typedef struct {
    ovs_camera camera;
    int32_t num_keypts;
    const ovs_keypoint* undist_keypts;
    const double* bearings;
} ovs_init_view;

#define OVS_INIT_OK 0                  /* initialize() returned true */
#define OVS_INIT_NO_VALID_MODEL 1      /* no valid solution to decompose (e.g. fewer than 8 matches) */
#define OVS_INIT_DECOMPOSITION_REFUSED 2  /* the homography's singular values are too close (d1/d2 or d2/d3 < 1.00001) */
#define OVS_INIT_TOO_FEW 3             /* the best hypothesis has fewer than min_num_triangulated valid points */
#define OVS_INIT_AMBIGUOUS 4           /* more than one hypothesis has more than 0.8 x the best count */
#define OVS_INIT_SMALL_PARALLAX 5      /* the best hypothesis's parallax is below parallax_deg_thr */

#define OVS_INIT_MODEL_NONE 0
#define OVS_INIT_MODEL_H 1
#define OVS_INIT_MODEL_F 2
#define OVS_INIT_MODEL_E 3

/* The outcome of one initialisation problem. */
typedef struct {
    int32_t status;                    /* OVS_INIT_* */
    int32_t model;                     /* OVS_INIT_MODEL_*: the decomposed solution */
    int32_t chosen;                    /* the hypothesis with the most valid points (first on ties), -1 with none */
    int32_t num_hypotheses;            /* 8 (H), 4 (F, E), 0 */
    int32_t num_valid[8];              /* per hypothesis: check_pose's count of valid points */
    float cos_parallax[8];             /* per hypothesis: the min(50, n - 1)-th smallest cos_parallax of its n valid points (1: n = 0) */
    double rot_ref_to_cur[9];          /* get_rotation_ref_to_cur(), row-major (p_cur = R p_ref + t), when status is OVS_INIT_OK */
    double trans_ref_to_cur[3];        /* get_translation_ref_to_cur() (unit norm), when status is OVS_INIT_OK */
    double solver_M[2][9];             /* perspective: H_21, F_21; bearing_vector: E_21, zero */
    double solver_score[2];            /* the solvers' best scores, in the same order */
    int32_t solver_num_inliers[2];
    uint8_t solver_valid[2];
    uint8_t reserved[6];
} ovs_init_result;

/* initialize::perspective(ref_frm, num_ransac_iters, min_num_triangulated, parallax_deg_thr, reproj_err_thr).initialize(cur_frm,
 * ref_matches_with_cur) for B independent problems in one call.  Problem b has the reference view ref_views[b] and the current
 * view cur_views[b]; its ref_matches_with_cur (one entry per reference keypoint: the matched current keypoint, or -1) and its
 * outputs is_triangulated / triangulated_pts[*3] (get_triangulated_flags() / get_triangulated_pts(), in the reference camera's
 * frame; zero where not triangulated and for a failed problem) are concatenated over the problems in order, ref_views[b].num_keypts
 * entries each.  seeds[B]: one sampler seed per problem, used by both the homography and the fundamental-matrix solver (a
 * problem gives the same result alone or inside a batch).  The steps (both solvers on the matches in reference-index order with
 * sigma = 1 and recompute, the model choice S_H / (S_H + S_F) > 0.40, the decompositions into 8 or 4 hypotheses, check_pose with
 * reproj_err_thr_sq (the reference passes 4.0) and depth_is_positive, find_most_plausible_pose) and their conventions are in
 * DESIGN.md section 5; solver_M / solver_score / solver_num_inliers / solver_valid equal ovs_homography_solve_ransac_host and
 * ovs_fundamental_solve_ransac_host on the same matches and seeds.
 * Checked before any launch -- OVS_ERR_INVALID_ARG: B outside 0 .. 65535, a negative num_ransac_iters or min_num_triangulated,
 * a parallax_deg_thr outside 0 .. 180, a reproj_err_thr_sq that is negative or not finite, a camera of another model or with
 * fx, fy not positive and finite, a keypoint that is not finite, a bearing that is not a finite unit vector, an entry of
 * ref_matches_with_cur outside -1 .. cur_views[b].num_keypts - 1, a missing array; OVS_ERR_UNSUPPORTED: 2^28 or more keypoints of
 * one side or matches in all, or B x num_ransac_iters above 2^31 - 1.  B == 0 or no match at all returns without a launch.
 * Otherwise the call is 13 launches (7 with num_ransac_iters == 0): the homography solve's 4, the fundamental solve's 4 and the 5
 * initialiser kernels, one copy each way and one wait, whatever B and whichever model each problem takes.  The call has its own
 * buffers on the handle: the matcher and solver entry points are unaffected by it. */
int ovs_initialize_perspective_host(ovs_matcher* h, int B, const ovs_init_view* ref_views, const ovs_init_view* cur_views,
                                    const int32_t* ref_matches_with_cur, int num_ransac_iters, int min_num_triangulated,
                                    float parallax_deg_thr, float reproj_err_thr_sq, const uint64_t* seeds, ovs_init_result* results,
                                    uint8_t* is_triangulated, double* triangulated_pts);
/* initialize::bearing_vector(...).initialize(cur_frm, ref_matches_with_cur): the same for equirectangular cameras, with the
 * essential solver on the matches' bearings (recompute on), 4 hypotheses and no depth test.  solver_M[0] / solver_score[0] /
 * solver_num_inliers[0] / solver_valid[0] equal ovs_essential_solve_ransac_host on the gathered bearings and the same seeds.
 * 8 launches (6 with num_ransac_iters == 0): the essential solve's 3 and the 5 initialiser kernels, one copy each way, one wait. */
int ovs_initialize_bearing_vector_host(ovs_matcher* h, int B, const ovs_init_view* ref_views, const ovs_init_view* cur_views,
                                       const int32_t* ref_matches_with_cur, int num_ransac_iters, int min_num_triangulated,
                                       float parallax_deg_thr, float reproj_err_thr_sq, const uint64_t* seeds, ovs_init_result* results,
                                       uint8_t* is_triangulated, double* triangulated_pts);

/* A landmark create_new_landmarks makes: keyfrms_2[neighbour], keypoint idx_1 of keyframe 1, idx_2 of the neighbour, pos_w. */
typedef struct {
    int32_t neighbour, idx_1, idx_2, reserved;
    double pos_w[3];
} ovs_new_landmark;

/* The compute step of mapping_module::create_new_landmarks: for b = 0 .. B - 1 (the neighbours in the reference's order, after
 * the caller's baseline and depth gates), robust::match_for_triangulation(keyfrm_1, keyfrms_2[b], E_12[b*9], ...) exactly as
 * ovs_robust_match_for_triangulation_host with the landmark flags of keyframe 1 as they stand at that neighbour, then
 * two_view_triangulator(keyfrm_1, keyfrms_2[b], rays_parallax_deg_thr) on its pairs in idx_1 order; every valid pair becomes a
 * record and its keyframe-1 keypoint counts as having a landmark for the neighbours after b.  epipole_in_2[b*3]: as for the
 * matcher.  out[capacity >= keyfrm_1->num_keypts] receives the records in creation order, *num_out their count.
 * Neighbour b's records depend on neighbours 0 .. b only: the records of the first k + 1 neighbours of a call are the records of a
 * call with those k + 1 neighbours, so a caller that stops at the reference's keyframe_is_queued() check keeps the prefix that
 * ends before the neighbour it stops at.
 * Device work: ONE launch of the matcher's candidate-list kernel for every (neighbour, query) pair, ONE launch of the
 * triangulation kernel over every listed candidate, one copy each way and one wait; then, when a record comes from a list, one
 * gather launch, one copy each way and one wait.  A list exhausted by earlier takers costs a re-query: two launches (its list, its
 * pair's triangulation), one copy each way and one wait.  Nothing else depends on B.  Checked before any launch:
 *  OVS_ERR_INVALID_ARG: the keyframe checks of ovs_two_view_triangulate_host (on every keypoint of every keyframe), a missing
 *    descriptor, landmark-flag or node array, B outside 0 .. 65535, a non-finite E_12 or epipole;
 *  OVS_ERR_CAPACITY: capacity < keyfrm_1->num_keypts;
 *  OVS_ERR_UNSUPPORTED: a neighbour with 65536 or more keypoints, or (B x queries + 1) x 8 candidate slots above 2^31 - 1 (queries:
 *    the keyframe-1 keypoints without a landmark that have a node).
 * Uses the buffers of ovs_two_view_triangulate_host. */
int ovs_create_new_landmarks_host(ovs_matcher* h, const ovs_keyframe_view* keyfrm_1, int B, const ovs_keyframe_view* keyfrms_2,
                                  const double* E_12, const double* epipole_in_2, int check_orientation, double rays_parallax_deg_thr,
                                  ovs_new_landmark* out, int capacity, int* num_out);

/* data::frame's constructor right after extract(): camera->undistort_keypoints(keypts_, undist_keypts_) +
 * camera->convert_keypoints_to_bearings(undist_keypts_, bearings_) (camera/perspective.cc, camera/equirectangular.cc; SURVEY 8f
 * rank 3).  Perspective: cv::undistortPoints(pts, K, dist, R = I, P = K, MAX_ITER num_iterations) -- OpenVSLAM uses 20 --
 * with dist = {k1, k2, p1, p2, k3} (NULL = no distortion), bit-exact with OpenCV in the float keypoints; bearings[n*3] f64.
 * Equirectangular: keypoints unchanged, bearings from longitude / latitude.  Only pt changes in the keypoint records.
 * Fisheye (camera/fisheye.cc): cv::fisheye::undistortPoints(pts, K, D, R = I, P = K) with its default criteria -- the `dist`
 * argument then holds D = (k1, k2, k3, k4) and num_iterations the Newton step limit (OpenCV: 10); points that do not converge
 * become (-1e6, -1e6) as in OpenCV >= 4.5.  Radial division (camera/radial_division.cc): p_u = p_d / (1 + dist[0] |p_d|^2) on
 * normalised coordinates.  Both take perspective bearings of the undistorted keypoints.
 * The _device variant works on the extractor's device output (d_undist_out may alias d_keypts_in; outputs may be NULL). */
int ovs_undistort_keypoints_device(ovs_extractor* h, const ovs_camera* cam, const double* dist_k1k2p1p2k3, int num_iterations, int n,
                                   const ovs_keypoint* d_keypts_in, ovs_keypoint* d_undist_out, double* d_bearings_out);
int ovs_undistort_keypoints_host(ovs_extractor* h, const ovs_camera* cam, const double* dist_k1k2p1p2k3, int num_iterations, int n,
                                 const ovs_keypoint* keypts_in, ovs_keypoint* undist_out, double* bearings_out);

typedef struct {
    int32_t num_rounds;            /* optimizer.optimize() calls made */
    int32_t num_iterations;        /* Levenberg iterations executed in total */
    int32_t num_trials;            /* linear solves (LM trials) in total */
    int32_t round_iterations[8];
    double lambda_init[8];         /* computeLambdaInit() of each round */
    double last_lambda, last_chi2; /* of the last round */
    double final_chi2;             /* robust chi2 of the active edges at the returned state */
    float device_us;               /* CUDA-event time of the call's device work */
    float solver_us;               /* local BA: CUDA-event time (launching stream) of the reduced-system solver launches, summed */
    int32_t solver_launches;       /* local BA: launches of the reduced-system solver (one per Levenberg iteration) */
    int32_t solver_trials;         /* local BA: systems factorised (speculative damping trials, <= 4 per launch) */
    int32_t reduced_dim;           /* local BA: dimension of the reduced camera system (6 x free keyframes) */
    float schur_us;                /* local BA: CUDA-event time of the Schur-complement launches (chunk + final) of the batches that ran, summed */
    int32_t co_observations;       /* local BA: (landmark, keyframe pair a <= b) records the Schur complement sums over */
} ovs_ba_stats;

typedef struct ovs_optimizer ovs_optimizer;
int ovs_optimizer_create(int device, ovs_optimizer** out);
void ovs_optimizer_destroy(ovs_optimizer* h);

/* pose_optimizer::optimize(data::frame& frm) (optimize/pose_optimizer.cc) on plain arrays: one SE3
 * vertex, one unary reprojection edge per matched landmark (frm.landmarks_[idx] valid).
 *  setup_is_mono: camera->setup_type_ == Monocular (selects the Huber delta sqrt(5.991) / sqrt(7.815));
 *  pts_w[n*3]: lm->get_pos_in_world();  obs_xy[n*2]: frm.undist_keypts_[idx].pt;
 *  obs_x_right[n]: frm.stereo_x_right_[idx] (< 0 = monocular edge; NULL = all monocular);
 *  inv_sigma_sq[n]: frm.inv_level_sigma_sq_[octave];
 *  pose_cw[12]: frm.cam_pose_cw_ as {R row-major (9), t (3)}, updated in place (frm.set_cam_pose);
 *  outlier_flags[n]: frm.outlier_flags_;  *num_inliers: the return value (num_init_obs - num_bad_obs).
 * num_trials / num_each_iter: the constructor arguments (4, 10).
 * A handle holds ONE problem at a time: this call reuses the handle's device buffers, so a local-BA problem prepared on
 * the same handle (ovs_local_ba_prepare) is invalidated by it -- ovs_local_ba_run / _fetch then fail with
 * OVS_ERR_INVALID_ARG until the problem is prepared again.  Use separate handles to keep both resident. */
int ovs_pose_optimize_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int n, const double* pts_w,
                           const float* obs_xy, const float* obs_x_right, const float* inv_sigma_sq,
                           double* pose_cw, uint8_t* outlier_flags, int num_trials, int num_each_iter,
                           int* num_inliers, ovs_ba_stats* stats);

/* transform_optimizer::optimize(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, g2o_Sim3_12, chi_sq)
 * (optimize/transform_optimizer.cc, loop closure) on plain arrays: one Sim3 vertex S_12 (camera 2 -> camera 1,
 * S p = s R p + t) and, per correspondence i, a forward edge (lm_2 through S_12 into keyframe 1) and a backward edge
 * (lm_1 through S_12^-1 into keyframe 2), Huber delta (double)sqrtf(chi_sq).  The caller keeps the pairs the reference keeps
 * (both landmarks valid, lm_2 observed in keyframe 2):
 *  cam_1 / cam_2: keyfrm_x->camera_;  pose_1w[12] / pose_2w[12]: keyfrm_x->get_cam_pose() as {R row-major, t};
 *  pos_w_1[n*3]: lm_1->get_pos_in_world(), lm_1 = keyframe 1's landmark at keypoint idx_i;
 *  obs_xy_1[n*2]: keyfrm_1->undist_keypts_[idx_i].pt;  inv_sigma_sq_1[n]: keyfrm_1->inv_level_sigma_sq_[its octave];
 *  pos_w_2 / obs_xy_2 / inv_sigma_sq_2: the same for lm_2 = matched_lms_in_keyfrm_2[idx_i] and its keypoint in keyframe 2;
 *  fix_scale: the constructor's fix_scale (camera not monocular): update[6] = 0 inside the update, the damped system stays 7x7;
 *  chi_sq: the reference passes 10;  num_first_iter / num_iter: the two rounds (5, and the constructor's num_iter, 10);
 *  sim3_12[13]: g2o_Sim3_12 as {R row-major (9), t (3), s > 0}, overwritten only when the call succeeds;
 *  inlier_out[n]: 1 while matched_lms_in_keyfrm_2[idx_i] stays set, 0 where the reference nulls it;
 *  *num_inliers: the return value (0 when fewer than 10 pairs survive the first round).
 * stats: num_rounds, iterations, trials, round_iterations, lambda_init per round, last_lambda, last_chi2, final_chi2 (plain
 * chi2 of the surviving pairs' stored errors) and device_us.  n == 0 returns at once without a launch.
 * Like ovs_pose_optimize_host this call reuses the handle's device buffers: a local-BA problem prepared on the same handle is
 * invalidated (ovs_local_ba_run / _fetch then fail with OVS_ERR_INVALID_ARG until it is prepared again). */
int ovs_transform_optimize_host(ovs_optimizer* h, const ovs_camera* cam_1, const ovs_camera* cam_2, const double* pose_1w,
                                const double* pose_2w, int n, const double* pos_w_1, const float* obs_xy_1, const float* inv_sigma_sq_1,
                                const double* pos_w_2, const float* obs_xy_2, const float* inv_sigma_sq_2, int fix_scale, float chi_sq,
                                int num_first_iter, int num_iter, double* sim3_12, uint8_t* inlier_out, int* num_inliers,
                                ovs_ba_stats* stats);

/* solve::sim3_solver(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, fix_scale, min_num_inliers).find_via_ransac(max_num_iter)
 * (solve/sim3_solver.cc, loop detection) for B independent problems (loop candidates) in one call.  Problem b owns the pairs
 * pair_offsets[b] .. pair_offsets[b + 1] - 1 (pair_offsets[0] = 0, non-decreasing); the caller keeps the pairs the reference keeps
 * (both landmarks valid and not to be erased, lm_2 observed in keyframe 2), in keyframe 1's keypoint order:
 *  cam_1[b] / cam_2[b]: keyfrm_x->camera_;  pose_1w / pose_2w [B*12]: keyfrm_x->get_cam_pose() as {R row-major, t};
 *  pos_w_1[n*3]: lm_1->get_pos_in_world();  sigma_sq_1[n]: keyfrm_1->level_sigma_sq_[octave of lm_1's keypoint];
 *  pos_w_2 / sigma_sq_2: the same for lm_2 = matched_lms_in_keyfrm_2[idx_1] and its keypoint in keyframe 2;
 *  fix_scale, min_num_inliers (the reference passes 20), max_num_iter (200): as in the reference;
 *  seeds[B]: the sampler's seed per problem (a problem gives the same result alone or inside a batch).
 * Per problem: sim3_12[b*13] = the best S_12 {R row-major (9), t (3), s} (identity when no hypothesis has an inlier);
 * valid[b] = solution_is_valid(); num_inliers[b] = the best count; best_iter[b] = the hypothesis it came from (-1: none);
 * inlier_out[n] = the best hypothesis's inlier flags.  With fewer than 3 or fewer than min_num_inliers pairs no hypothesis runs
 * and the problem is invalid.  The sampler, Horn's solution, the inlier test and the conventions fixed here are described in
 * DESIGN.md section 5.  B > 65535, invalid offsets, camera models, sigma_sq that is not positive and finite, or negative counts return
 * OVS_ERR_INVALID_ARG; B == 0 or no pair at all returns without a launch.  Otherwise the call is two launches, one copy each
 * way and one wait.  Like ovs_pose_optimize_host this call reuses the handle's device buffers: a local-BA problem prepared on
 * the same handle is invalidated (ovs_local_ba_run / _fetch then fail with OVS_ERR_INVALID_ARG until it is prepared again). */
int ovs_sim3_solve_ransac_host(ovs_optimizer* h, int B, const int32_t* pair_offsets, const ovs_camera* cam_1, const double* pose_1w,
                               const ovs_camera* cam_2, const double* pose_2w, const double* pos_w_1, const float* sigma_sq_1,
                               const double* pos_w_2, const float* sigma_sq_2, int fix_scale, int min_num_inliers, int max_num_iter,
                               const uint64_t* seeds, double* sim3_12, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter,
                               uint8_t* inlier_out);

/* solve::pnp_solver(valid_bearings, valid_keypts, valid_points, scale_factors, min_num_inliers).find_via_ransac(max_num_iter,
 * recompute) (solve/pnp_solver.cc, relocalisation) for B independent problems (relocalisation candidates) in one call.  Problem b
 * owns the correspondences corr_offsets[b] .. corr_offsets[b + 1] - 1 (corr_offsets[0] = 0, non-decreasing), in the order the
 * reference's constructor receives them:
 *  bearings[n*3]: frm.bearings_[idx] (unit; any camera model: ovs_undistort_keypoints_* produces them);
 *  pos_w[n*3]: the matched landmark's get_pos_in_world();
 *  scale_factor[n]: scale_factors_[octave of the keypoint], in (0, 90]: the bound is cos(pi / 180 * scale_factor), in double;
 *  min_num_inliers (the reference's default 10), max_num_iter (the relocaliser's 30), recompute (default true): as in the
 *  reference; seeds[B]: the sampler's seed per problem (a problem gives the same result alone or inside a batch).
 * Per problem: pose_cw[b*12] = get_best_cam_pose() as {R row-major (9), t (3)} (identity when no hypothesis has an inlier);
 * valid[b] = solution_is_valid(); num_inliers[b] = the number of inlier flags set; best_iter[b] = the best hypothesis (-1: none);
 * inlier_out[n] = get_inlier_flags().  With fewer than 6 (the minimal set) or fewer than min_num_inliers correspondences no
 * hypothesis runs and the problem is invalid.  With recompute, a valid problem whose best hypothesis has at least 6 inliers is
 * solved again by EPnP on all of them and its flags are re-checked at that pose.  The sampler, EPnP, the fixed order of the
 * recompute's sums and the conventions fixed here are described in DESIGN.md section 5.  B outside 0 .. 65535, invalid offsets,
 * a non-finite position, a bearing that is not finite or not unit (|b.b - 1| > 1e-6), a scale factor outside (0, 90] or negative
 * counts return OVS_ERR_INVALID_ARG; B == 0 or no correspondence at all returns without a launch.  Otherwise the call is three
 * launches (two with max_num_iter == 0), one copy each way and one wait.  Like ovs_pose_optimize_host this call reuses the
 * handle's device buffers: a local-BA problem prepared on the same handle is invalidated (ovs_local_ba_run / _fetch then fail
 * with OVS_ERR_INVALID_ARG until it is prepared again). */
int ovs_pnp_solve_ransac_host(ovs_optimizer* h, int B, const int32_t* corr_offsets, const double* bearings, const double* pos_w,
                              const float* scale_factor, int min_num_inliers, int max_num_iter, int recompute, const uint64_t* seeds,
                              double* pose_cw, uint8_t* valid, int32_t* num_inliers, int32_t* best_iter, uint8_t* inlier_out);

/* graph_optimizer::optimize(loop_keyfrm, curr_keyfrm, non_corrected_Sim3s, pre_corrected_Sim3s, loop_connections)
 * (optimize/graph_optimizer.cc, loop closure) on plain arrays: one Sim3 vertex per keyframe, one relative Sim3 edge per keyframe
 * pair, e = log(S_ji S_i S_j^-1) with identity information and no robust kernel, g2o's Levenberg with the user lambda 1e-16.
 * The caller flattens the graph as the reference builds it (INTEGRATION.md):
 *  sim3_cw[K*13]: S_iw as {R row-major (9), t (3), s > 0} -- the pre-corrected Sim3 where the keyframe has one, otherwise
 *    {R, t, 1} of cam_pose_cw; overwritten with the optimised estimates;
 *  fixed[K]: 1 for the loop keyframe (a free vertex without an edge is left out of the system and keeps its bits);
 *  edge_i[E] / edge_j[E] / meas_ji[E*13]: vertex 0, vertex 1 and the measurement S_ji of each edge (i != j);
 *  fix_scale: the constructor's fix_scale (stereo / RGB-D): update[6] = 0 inside the update, the system stays 7 per vertex;
 *  num_iter: the reference's 50;
 *  lm_pos_w[L*3] / lm_ref[L]: landmark positions, corrected in place as p <- S_wr^opt (S_rw^init p) through the reference
 *    vertex r (the landmark's reference keyframe, or ref_keyfrm_id_in_loop_fusion_); lm_ref = -1 leaves a landmark's bits;
 *  pose_cw_out[K*12] (may be NULL): cam_pose_cw = {R, t / s} of the optimised S_iw.
 * stats: num_rounds (1), iterations, trials, lambda_init[0] (1e-16), last_lambda, last_chi2, final_chi2 (chi2 at the returned
 * estimates, also when nothing is optimised; 0 for E == 0), device_us, solver_us, solver_launches, solver_trials,
 * reduced_dim = 7 x free vertices.
 * An index out of range, i == j, or a scale that is not positive and finite returns OVS_ERR_INVALID_ARG; more than 857 free
 * vertices (7 x 857 = 5999 <= 6000, the dense solver's limit) returns OVS_ERR_UNSUPPORTED.  With no free vertex in the system
 * (E == 0 included) nothing is optimised: the estimates come back unchanged and only the write-back runs.
 * Like ovs_pose_optimize_host this call reuses the handle's device buffers: a local-BA problem prepared on the same handle is
 * invalidated (ovs_local_ba_run / _fetch then fail with OVS_ERR_INVALID_ARG until it is prepared again). */
int ovs_graph_optimize_host(ovs_optimizer* h, int K, double* sim3_cw, const uint8_t* fixed, int E, const int32_t* edge_i,
                            const int32_t* edge_j, const double* meas_ji, int fix_scale, int num_iter, int L, double* lm_pos_w,
                            const int32_t* lm_ref, double* pose_cw_out, ovs_ba_stats* stats);

/* local_bundle_adjuster::optimize(curr_keyfrm, force_stop_flag) (optimize/local_bundle_adjuster.cc) on
 * the graph the reference builds: K keyframe vertices (local keyframes free, "fixed" keyframes and
 * keyframe id 0 fixed), L landmark vertices (marginalised), M reprojection edges.
 *  poses[K*12] ({R row-major, t} of cam_pose_cw), points[L*3]: updated in place;
 *  observations grouped by landmark (obs_lm non-decreasing), the order the reference adds them;
 *  outlier_out[M]: 1 where the reference would erase the observation (chi2 over the 5% bound or
 *  non-positive depth after the second round).  force_stop_flag (the reference's `bool* const`, read as
 *  one byte) may be NULL; it is polled between LM trials like g2o's terminate().  num_first_iter / num_second_iter: constructor arguments (5, 10).
 * Up to 114 free keyframes the reduced camera system is factorised by one cluster kernel out of shared memory; larger
 * local maps (up to 1000 free keyframes) take a multi-launch path with the panel in global memory. */
int ovs_local_ba_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, double* poses, const uint8_t* fixed,
                      int L, double* points, int M, const int32_t* obs_kf, const int32_t* obs_lm, const float* obs_xy,
                      const float* obs_x_right, const float* inv_sigma_sq, int num_first_iter, int num_second_iter,
                      const volatile uint8_t* force_stop_flag, uint8_t* outlier_out, ovs_ba_stats* stats);

/* The same call in three phases, for callers that keep the problem resident on the device:
 * prepare = graph bookkeeping + upload + co-observation lists (enqueued, returns without waiting; the input arrays
 * are copied before it returns); run = the two Levenberg rounds, restarting from the uploaded estimates each time
 * (state stays in HBM; the whole Levenberg loop, accept / reject decisions included, runs on the device: the host enqueues
 * a static launch sequence and waits once); fetch = download of the poses, points and outlier flags of the last run (any
 * output pointer may be NULL). */
int ovs_local_ba_prepare(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, const double* poses,
                         const uint8_t* fixed, int L, const double* points, int M, const int32_t* obs_kf,
                         const int32_t* obs_lm, const float* obs_xy, const float* obs_x_right, const float* inv_sigma_sq);
int ovs_local_ba_run(ovs_optimizer* h, int num_first_iter, int num_second_iter, const volatile uint8_t* force_stop_flag,
                     ovs_ba_stats* stats);
int ovs_local_ba_fetch(ovs_optimizer* h, double* poses, double* points, uint8_t* outlier_out);
/* The same with the graph already resident in device memory (all array arguments are device pointers, d_obs_x_right may be
 * NULL): what a caller that keeps its map on the GPU uses -- no host loop touches the observations, the graph bookkeeping
 * (free-keyframe ids, per-landmark edge ranges, validation) runs on the device.  The arrays are copied before return. */
int ovs_local_ba_prepare_device(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, const double* d_poses,
                                const uint8_t* d_fixed, int L, const double* d_points, int M, const int32_t* d_obs_kf,
                                const int32_t* d_obs_lm, const float* d_obs_xy, const float* d_obs_x_right, const float* d_inv_sigma_sq);
int ovs_local_ba_fetch_device(ovs_optimizer* h, double* d_poses, double* d_points, uint8_t* d_outlier_out);
/* optimize::global_bundle_adjuster::optimize(lead_keyfrm_id_in_global_BA, force_stop_flag) (optimize/global_bundle_adjuster.cc)
 * on the graph the reference builds: every keyframe (the origin keyframe fixed: fixed[k] != 0) and every landmark of the map,
 * one reprojection edge per observation, ONE Levenberg round of num_iter (constructor argument, 10) iterations, Huber kernel
 * on every edge when use_huber_kernel (constructor argument, true); no outlier classification.  poses / points are updated in
 * place (the reference stores them as pose_cw_after_loop_BA_ / pos_w_after_global_BA_).  Same array conventions as
 * ovs_local_ba_host; up to 1000 free keyframes (beyond 114 the reduced system takes the multi-launch solver). */
int ovs_global_ba_host(ovs_optimizer* h, const ovs_camera* cam, int setup_is_mono, int K, double* poses, const uint8_t* fixed,
                       int L, double* points, int M, const int32_t* obs_kf, const int32_t* obs_lm, const float* obs_xy,
                       const float* obs_x_right, const float* inv_sigma_sq, int num_iter, int use_huber_kernel,
                       const volatile uint8_t* force_stop_flag, ovs_ba_stats* stats);
/* Test hook: the stable radix sort of the BA graph preparation (co-observations by keyframe pair: k_sort_hist /
 * k_sort_tile_prefix / k_sort_scatter) on host arrays, by the low end_bit bits of the keys. */
int ovs_debug_sort_pairs(int device, const uint32_t* keys, const uint64_t* vals, int n, int end_bit, uint32_t* keys_out, uint64_t* vals_out);
/* Local / global BA: CTAs per cluster of the reduced-system solver (1, 2, 4 or 8; default 8).  8 gives the lowest latency of a
 * single call; 2 is meant for several optimisers sharing the GPU: each call occupies fewer SMs, so more calls run at once.
 * The result does not depend on the width. */
int ovs_optimizer_set_cluster_width(ovs_optimizer* h, int width);
/* Local BA: the launch sequence of one Levenberg iteration is static (damping values, ring slots and the accept / reject
 * walk live in device memory), so it can be captured once per run and replayed as ONE CUDA graph per iteration.  Trims
 * the inter-kernel gaps of a single stream; off by default. */
int ovs_optimizer_set_graphs(ovs_optimizer* h, int enable);
/* Local BA: the Levenberg loop runs on the device without host round trips.  mode 1 makes the host read the device's
 * decision after every trial batch and skip the launches that are not needed (default only for reduced systems beyond
 * the cluster solver, whose batches are ~100 launches each); mode 0 never synchronises; -1 = automatic.  Same results. */
int ovs_optimizer_set_host_sync(ovs_optimizer* h, int mode);
/* Local BA: number of Levenberg damping trials evaluated speculatively per launch sequence (1..4, default 4).  The
 * result is the sequential algorithm's for every width; 4 minimises the latency of one session (a rejected trial costs
 * no extra round trip); smaller widths trade latency for less speculative GPU work. */
int ovs_optimizer_set_speculation(ovs_optimizer* h, int width);
/* Local BA: a second trial batch of `width` (1..4) damping values enqueued statically behind the first batch of every
 * iteration (0 = off, the default).  Its kernels return at their first instruction when the first batch decided the
 * iteration, so e.g. speculation 2 + second batch 2 evaluates 2 trials where g2o's loop needs <= 2 and 4 where it needs
 * 3 or 4, still without a host round trip: less speculative GPU work per call (throughput when several sessions share the
 * GPU) for one more dependent launch sequence on the iterations that reject their first trials (latency).  Same results. */
int ovs_optimizer_set_second_batch(ovs_optimizer* h, int width);

/* match::bow_tree::match_frame_and_keyframe(keyfrm, frm, matched_lms_in_frm) (match/bow_tree.cc) on plain arrays.  The BoW
 * feature vectors are inputs: bow_node_x[i] = vocabulary node of keypoint i (< 0 = none).  Nodes ascending, keypoints of a
 * node in index order (the reference's lock-step walk over the two feature vectors): every keyframe keypoint with a valid
 * landmark (lm_valid_kf) takes its nearest still-unmatched frame keypoint of the same node when the distance is <=
 * HAMMING_DIST_THR_LOW and lowe_ratio * second_best >= best; orientation histogram if requested.
 * matched_keyfrm_idx_of_frm[n_frm] = keyframe keypoint whose landmark frame keypoint i receives, or -1. */
int ovs_bow_tree_match_frame_and_keyframe_host(ovs_matcher* m, int n_kf, const uint8_t* desc_kf, const float* angle_kf, const uint8_t* lm_valid_kf,
                                               const int32_t* bow_node_kf, int n_frm, const uint8_t* desc_frm, const float* angle_frm,
                                               const int32_t* bow_node_frm, float lowe_ratio, int check_orientation,
                                               int32_t* matched_keyfrm_idx_of_frm, int* num_matches);
/* match::bow_tree::match_keyframes(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_1): both keypoints need a valid landmark, a
 * keyframe-2 keypoint is matched at most once.  matched_idx_2_of_1[n1] = keypoint of keyframe 2 or -1. */
int ovs_bow_tree_match_keyframes_host(ovs_matcher* m, int n1, const uint8_t* desc_1, const float* angle_1, const uint8_t* lm_valid_1,
                                      const int32_t* bow_node_1, int n2, const uint8_t* desc_2, const float* angle_2, const uint8_t* lm_valid_2,
                                      const int32_t* bow_node_2, float lowe_ratio, int check_orientation,
                                      int32_t* matched_idx_2_of_1, int* num_matches);
/* match::fuse (match/fuse.cc): the matching core of replace_duplication / detect_duplication.  Every usable landmark
 * (reprojected into the keyframe `f` by the caller: reproj_xy[nq*2], reproj_x_right[nq] or NULL, pred_level[nq] from
 * predict_scale_level, lm_desc[nq*32]) searches the window margin * scale_factors[level], levels [level - 1, level];
 * candidates whose reprojection error times inv_level_sigma_sq[own octave] exceeds 5.99 (7.8 with the x_right term) are
 * skipped; nearest descriptor, first in visiting order on ties, accepted at <= HAMMING_DIST_THR_LOW.  best_idx_of_lm[nq] =
 * keypoint index or -1 (what happens to a keypoint that already holds a landmark is the caller's data-model decision). */
int ovs_fuse_best_keypoints_host(ovs_frame_index* f, int nq, const uint8_t* usable, const float* reproj_xy, const float* reproj_x_right,
                                 const int32_t* pred_level, const uint8_t* lm_desc, const float* scale_factors,
                                 const float* inv_level_sigma_sq, int num_scale_levels, float margin,
                                 int32_t* best_idx_of_lm, int* num_matches);

/* ---- local mapping: match::fuse::replace_duplication with its reprojection (match/fuse.cc), for the forward and backward passes of
 * mapping_module::fuse_landmark_duplication (module/mapping_module.cc) ---- */

/* What replace_duplication reads of one target keyframe, from the keyframe's own vectors: the geometry (camera_, img_bounds_,
 * rot_cw / trans_cw, get_cam_center() as the keyframe holds it, num_scale_levels_, log_scale_factor_), scale_factors_ and
 * inv_level_sigma_sq_ (num_scale_levels entries each), num_keypts undist_keypts_ (x, y, octave), stereo_x_right_ (NULL:
 * monocular), descriptors_ (32 B each) and the camera's grid. */
typedef struct {
    ovs_frame_geometry geometry;
    const float* scale_factors;
    const float* inv_level_sigma_sq;
    int32_t num_keypts;
    const float* x;
    const float* y;
    const int32_t* octave;
    const float* x_right;
    const uint8_t* descriptors;
    ovs_grid grid;
} ovs_fuse_target;

/* Each of the number of targets, of landmarks, of queries, of all targets' keypoints and of all targets' grid cells is at most this
 * (OVS_ERR_UNSUPPORTED beyond): the staged buffers stay far inside size_t and their offsets inside int. */
#define OVS_FUSE_MAX_ITEMS (1 << 26)

/* The compute of match::fuse::replace_duplication(keyfrm, landmarks_to_check, margin) for B targets at once, without its data-model
 * updates: for every query, the keypoint best_idx of its target that the reference would fuse the landmark with, or -1.
 * Landmarks (nlm rows): pos_w[nlm*3] = get_pos_in_world(), mean_normal[nlm*3] = get_obs_mean_normal(), min_valid_dist /
 * max_valid_dist = the raw min_valid_dist_ / max_valid_dist_, lm_desc[nlm*32] = get_descriptor().  Queries: those of target t are
 * q_lm[q_off[t] .. q_off[t+1]) (q_off[0] = 0, non-decreasing, Q = q_off[B]); q_lm[q] is a landmark row, or -1 for a query to
 * skip (the caller's skip rule: no landmark, will_be_erased(), is_observed_in_keyframe()).  A query is answered from its own
 * landmark row and its target only: reproject_to_image, the valid-distance and ray gates in double, predict_scale_level (DESIGN.md
 * section 5), then the window margin * scale_factors[level] over the levels [level - 1, level], the chi-square gate of
 * ovs_fuse_best_keypoints_host, the nearest descriptor (first in get_keypoints_in_cell order on ties) at <= HAMMING_DIST_THR_LOW.
 * A query whose position or reprojection is not finite gets -1.  num_fused = the number of queries with a best_idx.  Optional
 * per-query outputs (each may be NULL): passed (the geometry's gates), reproj_xy[Q*2] (rounded to float), x_right, pred_level;
 * 0 where not passed.  At most 2 launches, one copy each way and one wait, whatever B is; Q = 0 or no query with q_lm >= 0 makes
 * no launch.  Refused before any launch and any allocation: OVS_ERR_INVALID_ARG for B < 0, a null array that is needed, a target
 * geometry that ovs_frame_can_observe_host refuses, a null scale table, a keypoint octave outside its target's scale table, a
 * grid with no cell or more than 2^20 cells, a malformed q_off, a q_lm entry outside [-1, nlm), a margin that is not finite and
 * positive; OVS_ERR_UNSUPPORTED for a target with 65536 keypoints or more, or a count above OVS_FUSE_MAX_ITEMS. */
int ovs_fuse_replace_duplication_host(ovs_matcher* m, int B, const ovs_fuse_target* targets, int nlm, const double* pos_w,
                                      const double* mean_normal, const float* min_valid_dist, const float* max_valid_dist,
                                      const uint8_t* lm_desc, const int32_t* q_off, const int32_t* q_lm, float margin, int32_t* best_idx,
                                      int* num_fused, uint8_t* passed, float* reproj_xy, float* x_right, int32_t* pred_level);

/* Measured FP64 peaks of `device` (whole chip, TFLOP/s counting 2 per FMA): independent mma.sync.m8n8k4.f64 (DMMA) and
 * independent DFMA.  bench.py quotes the Cholesky roofline against the DMMA figure measured in the same run. */
int ovs_probe_fp64_peaks(int device, double* dmma_tflops, double* dfma_tflops);

#ifdef __cplusplus
}
#endif
#endif /* OVS_B200_H */
