// openvslam_b200.hpp -- the reference's hot-path class surfaces, re-declared over the C ABI of
// libovs_b200.so (include/ovs_b200.h).  Header only.
//
//   openvslam::feature::orb_params / orb_extractor        (src/openvslam/feature/orb_params.h, orb_extractor.h)
//   openvslam::util::stereo_rectifier                     (src/openvslam/util/stereo_rectifier.h)
//   openvslam::match::robust / projection / area / stereo (src/openvslam/match/*.h)
//   openvslam::optimize::pose_optimizer / local_bundle_adjuster / transform_optimizer / graph_optimizer (src/openvslam/optimize/*.h)
//   openvslam::solve::sim3_solver                         (src/openvslam/solve/sim3_solver.h)
//   openvslam::solve::pnp_solver                          (src/openvslam/solve/pnp_solver.h)
//   openvslam::solve::essential_solver                    (src/openvslam/solve/essential_solver.h)
//   openvslam::solve::homography_solver / fundamental_solver (src/openvslam/solve/{homography,fundamental}_solver.h)
// [file names as recalled in SURVEY.md 8(a); /root/reference holds no source, so no line numbers].
//
// The reference's methods take cv::Mat / cv::KeyPoint / Eigen / data::frame / data::keyframe.  None of
// those headers exist in this build environment, so every method is declared on plain views
// (pointers + sizes, `ovs_keypoint` which is layout-compatible with cv::KeyPoint).  When
// OVS_B200_WITH_OPENCV is defined (a tree that has OpenCV), the cv::_InputArray overloads with the
// reference's exact signatures are compiled as well and forward to the same code.
// The data::frame / data::keyframe flattening the matchers and optimisers need is the job of the
// adapter shown in INTEGRATION.md; the classes here keep the reference's constructor arguments,
// member names and return values.
#pragma once

#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../ovs_b200.h"

#ifdef OVS_B200_WITH_OPENCV
#include <opencv2/core.hpp>
#endif

namespace openvslam {

// The reference's data model (data/frame.h, data/keyframe.h, data/landmark.h).  With OVS_B200_WITH_REFERENCE_TYPES the classes
// below also declare the reference's own method signatures on these types; their bodies -- the flattening of the data model
// into the array views -- are in adapters.hpp, which a tree that has those headers includes instead of this file.
namespace data { class frame; class keyframe; class landmark; }

namespace detail {
inline void check(int rc) {
    if (rc != OVS_OK) throw std::runtime_error(std::string("ovs_b200: ") + ovs_last_error());
}
}  // namespace detail

namespace util {

//! util::stereo_rectifier: the rectification maps of both cameras of a stereo rig, built once on the device from the
//! StereoRectifier block (K_left, D_left, R_left, K_right, D_right, R_right, model) and the camera's cols, rows and K, the
//! rectified camera matrix.  Matrices are row-major 3 x 3; D is {k1, k2, p1, p2, k3} (perspective) or {k1..k4} (fisheye).
//! Immutable after construction: extractors on several threads may read one rectifier at once.
class stereo_rectifier {
public:
    //! The parsed StereoRectifier block of the config.
    struct params {
        int model = OVS_CAMERA_PERSPECTIVE;   // OVS_CAMERA_PERSPECTIVE or OVS_CAMERA_FISHEYE
        std::array<double, 9> K_left{}, R_left{}, K_right{}, R_right{};
        std::vector<double> D_left, D_right;
    };

    stereo_rectifier(const int cols, const int rows, const std::array<double, 9>& K_rect, const params& p, const int device = 0) {
        const std::size_t nd = p.model == OVS_CAMERA_FISHEYE ? 4 : 5;
        if (p.D_left.size() != nd || p.D_right.size() != nd) throw std::runtime_error("stereo_rectifier: wrong number of distortion parameters");
        detail::check(ovs_stereo_rectifier_create(device, p.model, cols, rows, p.K_left.data(), p.D_left.data(), p.R_left.data(), p.K_right.data(),
                                                  p.D_right.data(), p.R_right.data(), K_rect.data(), &h_));
        cols_ = cols; rows_ = rows;
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! util::stereo_rectifier(camera, StereoRectifier block): K_rect is the camera's K (body in adapters.hpp)
    template <class Camera>
    stereo_rectifier(const Camera* camera, const params& p, const int device = 0);
#endif
    ~stereo_rectifier() { ovs_stereo_rectifier_destroy(h_); }
    stereo_rectifier(const stereo_rectifier&) = delete;
    stereo_rectifier& operator=(const stereo_rectifier&) = delete;

    //! rectify(in_l, in_r, out_l, out_r) on u8 images with `channels` (1, 3, 4) interleaved channels; outputs keep them
    void rectify(const std::uint8_t* in_l, const std::uint8_t* in_r, const int rows, const int cols, const std::size_t step, const int channels,
                 std::uint8_t* out_l, std::uint8_t* out_r, const std::size_t out_step) const {
        detail::check(ovs_stereo_rectify_host(h_, in_l, in_r, cols, rows, step, channels, out_l, out_r, out_step));
    }
#ifdef OVS_B200_WITH_OPENCV
    //! The reference's signature.
    void rectify(const cv::Mat& in_img_l, const cv::Mat& in_img_r, cv::Mat& out_img_l, cv::Mat& out_img_r) const;
#endif

    //! The float maps of side 0 (left) or 1 (right), rows x cols each, as cv::initUndistortRectifyMap returns them
    void maps(const int side, std::vector<float>& map_x, std::vector<float>& map_y) const {
        map_x.resize(static_cast<std::size_t>(rows_) * cols_); map_y.resize(map_x.size());
        detail::check(ovs_stereo_rectifier_maps(h_, side, map_x.data(), map_y.data()));
    }

    int cols() const { return cols_; }
    int rows() const { return rows_; }
    ovs_stereo_rectifier* handle() const { return h_; }

private:
    ovs_stereo_rectifier* h_ = nullptr;
    int cols_ = 0, rows_ = 0;
};

}  // namespace util

namespace feature {

struct orb_params {
    orb_params() = default;
    orb_params(const unsigned int max_num_keypts, const float scale_factor, const unsigned int num_levels,
               const unsigned int ini_fast_thr, const unsigned int min_fast_thr,
               const std::vector<std::vector<float>>& mask_rects = {})
        : max_num_keypts_(max_num_keypts), scale_factor_(scale_factor), num_levels_(num_levels),
          ini_fast_thr_(ini_fast_thr), min_fast_thr(min_fast_thr), mask_rects_(mask_rects) {
        for (const auto& v : mask_rects_) {
            if (v.size() != 4) throw std::runtime_error("Each of mask rectangles must contain four parameters");
            if (v.at(0) >= v.at(1)) throw std::runtime_error("x_max must be greater than x_min");
            if (v.at(2) >= v.at(3)) throw std::runtime_error("y_max must be greater than x_min");
        }
    }
    unsigned int max_num_keypts_ = 2000;
    float scale_factor_ = 1.2f;
    unsigned int num_levels_ = 8;
    unsigned int ini_fast_thr_ = 20;
    unsigned int min_fast_thr = 7;
    //! A vector of keypoint area represents mask area: {x_min / cols, x_max / cols, y_min / rows, y_max / rows}
    std::vector<std::vector<float>> mask_rects_;
};

class orb_extractor {
public:
    orb_extractor() = delete;
    explicit orb_extractor(const orb_params& orb_params, const int device = 0) : orb_params_(orb_params) {
        ovs_orb_params p{orb_params.max_num_keypts_, orb_params.scale_factor_, orb_params.num_levels_, orb_params.ini_fast_thr_,
                         orb_params.min_fast_thr};
        std::vector<float> rects;
        for (const auto& r : orb_params.mask_rects_) rects.insert(rects.end(), r.begin(), r.end());
        detail::check(ovs_extractor_create(&p, rects.empty() ? nullptr : rects.data(), static_cast<int>(rects.size() / 4), device, &h_));
        const unsigned int L = orb_params.num_levels_;
        scale_factors_.resize(L); inv_scale_factors_.resize(L); level_sigma_sq_.resize(L); inv_level_sigma_sq_.resize(L);
        detail::check(ovs_extractor_scale_factors(h_, scale_factors_.data(), inv_scale_factors_.data(), level_sigma_sq_.data(),
                                                  inv_level_sigma_sq_.data()));
    }
    orb_extractor(const unsigned int max_num_keypts, const float scale_factor, const unsigned int num_levels,
                  const unsigned int ini_fast_thr, const unsigned int min_fast_thr,
                  const std::vector<std::vector<float>>& mask_rects = {})
        : orb_extractor(orb_params{max_num_keypts, scale_factor, num_levels, ini_fast_thr, min_fast_thr, mask_rects}) {}
    ~orb_extractor() { ovs_extractor_destroy(h_); }
    orb_extractor(const orb_extractor&) = delete;
    orb_extractor& operator=(const orb_extractor&) = delete;

    //! Extract keypoints and each descriptor of them (image: CV_8UC1 rows x cols, `step` bytes per row;
    //! mask: same size or nullptr).  descriptors: keypts.size() x 32 bytes.
    void extract(const std::uint8_t* image, const int rows, const int cols, const std::size_t step, const std::uint8_t* mask,
                 const std::size_t mask_step, std::vector<ovs_keypoint>& keypts, std::vector<std::uint8_t>& descriptors) {
        keypts.clear(); descriptors.clear();
        if (!image || rows <= 0 || cols <= 0) return;
        const int cap = ovs_extractor_max_keypoints(h_);
        keypts.resize(cap); descriptors.resize(static_cast<std::size_t>(cap) * 32);
        int n = 0;
        detail::check(ovs_extract_host(h_, image, cols, rows, step, mask, mask_step, keypts.data(), descriptors.data(), cap, &n));
        keypts.resize(n); descriptors.resize(static_cast<std::size_t>(n) * 32);
    }

    //! util::convert_to_grayscale(img, color_order) + extract() in one call: image is CV_8UC3 / CV_8UC4 (`channels`),
    //! color_order = OVS_COLOR_ORDER_BGR or OVS_COLOR_ORDER_RGB (camera::color_order_t)
    void extract_color(const std::uint8_t* image, const int rows, const int cols, const std::size_t step, const int channels, const int color_order,
                       const std::uint8_t* mask, const std::size_t mask_step, std::vector<ovs_keypoint>& keypts,
                       std::vector<std::uint8_t>& descriptors) {
        keypts.clear(); descriptors.clear();
        if (!image || rows <= 0 || cols <= 0) return;
        const int cap = ovs_extractor_max_keypoints(h_);
        keypts.resize(cap); descriptors.resize(static_cast<std::size_t>(cap) * 32);
        int n = 0;
        detail::check(ovs_extract_host_color(h_, image, cols, rows, step, channels, color_order, mask, mask_step, keypts.data(), descriptors.data(),
                                             cap, &n));
        keypts.resize(n); descriptors.resize(static_cast<std::size_t>(n) * 32);
    }

    //! rectifier.rectify() of one side (0 left, 1 right), util::convert_to_grayscale and extract() in one call: the raw image
    //! (1, 3 or 4 channels; color_order as extract_color) is rectified on the device straight into the pyramid.  The mask is in
    //! rectified coordinates.  The stereo frame's two extractors may run this on two threads with one rectifier.
    void extract(const util::stereo_rectifier& rectifier, const int side, const std::uint8_t* image, const int rows, const int cols,
                 const std::size_t step, const int channels, const int color_order, const std::uint8_t* mask, const std::size_t mask_step,
                 std::vector<ovs_keypoint>& keypts, std::vector<std::uint8_t>& descriptors) {
        keypts.clear(); descriptors.clear();
        const int cap = ovs_extractor_max_keypoints(h_);
        keypts.resize(cap); descriptors.resize(static_cast<std::size_t>(cap) * 32);
        int n = 0;
        detail::check(ovs_extract_host_rectified(h_, rectifier.handle(), side, image, cols, rows, step, channels, color_order, mask, mask_step,
                                                 keypts.data(), descriptors.data(), cap, &n));
        keypts.resize(n); descriptors.resize(static_cast<std::size_t>(n) * 32);
    }

    //! camera->undistort_keypoints(keypts, undist_keypts) + camera->convert_keypoints_to_bearings(undist_keypts, bearings):
    //! dist = {k1, k2, p1, p2, k3} or nullptr; bearings = 3 doubles per keypoint
    void undistort_keypoints(const ovs_camera& camera, const double* dist, const std::vector<ovs_keypoint>& keypts,
                             std::vector<ovs_keypoint>& undist_keypts, std::vector<double>& bearings, const int num_iterations = 20) const {
        undist_keypts.resize(keypts.size()); bearings.resize(keypts.size() * 3);
        detail::check(ovs_undistort_keypoints_host(h_, &camera, dist, num_iterations, static_cast<int>(keypts.size()), keypts.data(),
                                                   undist_keypts.data(), bearings.data()));
    }

#ifdef OVS_B200_WITH_OPENCV
    //! The reference's signature.
    void extract(const cv::_InputArray& in_image, const cv::_InputArray& in_image_mask, std::vector<cv::KeyPoint>& keypts,
                 const cv::_OutputArray& out_descriptors) {
        static_assert(sizeof(cv::KeyPoint) == sizeof(ovs_keypoint), "cv::KeyPoint layout changed");
        if (in_image.empty()) return;
        const cv::Mat image = in_image.getMat();
        CV_Assert(image.type() == CV_8UC1);
        const cv::Mat mask = in_image_mask.empty() ? cv::Mat() : in_image_mask.getMat();
        const int cap = ovs_extractor_max_keypoints(h_);
        keypts.resize(cap);
        cv::Mat desc(cap, 32, CV_8U);
        int n = 0;
        detail::check(ovs_extract_host(h_, image.data, image.cols, image.rows, image.step, mask.empty() ? nullptr : mask.data,
                                       mask.empty() ? 0 : mask.step, reinterpret_cast<ovs_keypoint*>(keypts.data()), desc.data, cap, &n));
        keypts.resize(n);
        if (n == 0) out_descriptors.release(); else desc.rowRange(0, n).copyTo(out_descriptors);
    }
#endif

    unsigned int get_max_num_keypoints() const { return orb_params_.max_num_keypts_; }
    float get_scale_factor() const { return orb_params_.scale_factor_; }
    unsigned int get_num_scale_levels() const { return orb_params_.num_levels_; }
    unsigned int get_initial_fast_threshold() const { return orb_params_.ini_fast_thr_; }
    unsigned int get_minimum_fast_threshold() const { return orb_params_.min_fast_thr; }
    std::vector<float> get_scale_factors() const { return scale_factors_; }
    std::vector<float> get_inv_scale_factors() const { return inv_scale_factors_; }
    std::vector<float> get_level_sigma_sq() const { return level_sigma_sq_; }
    std::vector<float> get_inv_level_sigma_sq() const { return inv_level_sigma_sq_; }

    //! image_pyramid_ (read by match::stereo): host copy of one level of the last extract()
    std::vector<std::uint8_t> image_pyramid(const int level, int& rows, int& cols) const {
        detail::check(ovs_extractor_pyramid_level(h_, level, nullptr, nullptr, &cols, &rows));
        std::vector<std::uint8_t> out(static_cast<std::size_t>(rows) * cols);
        detail::check(ovs_extractor_copy_pyramid_level(h_, level, out.data(), static_cast<std::size_t>(cols)));
        return out;
    }

    ovs_extractor* handle() const { return h_; }

private:
    orb_params orb_params_;
    ovs_extractor* h_ = nullptr;
    std::vector<float> scale_factors_, inv_scale_factors_, level_sigma_sq_, inv_level_sigma_sq_;
};

}  // namespace feature

namespace match {

static constexpr unsigned int HAMMING_DIST_THR_LOW = OVS_HAMMING_DIST_THR_LOW;
static constexpr unsigned int HAMMING_DIST_THR_HIGH = OVS_HAMMING_DIST_THR_HIGH;
static constexpr unsigned int MAX_HAMMING_DIST = OVS_MAX_HAMMING_DIST;

class base {
public:
    base(const float lowe_ratio, const bool check_orientation, const int device = 0)
        : lowe_ratio_(lowe_ratio), check_orientation_(check_orientation) {
        detail::check(ovs_matcher_create(device, &h_));
    }
    virtual ~base() { ovs_matcher_destroy(h_); }
    base(const base&) = delete;
    base& operator=(const base&) = delete;
    ovs_matcher* handle() const { return h_; }

protected:
    const float lowe_ratio_;
    const bool check_orientation_;
    ovs_matcher* h_ = nullptr;
};

//! A data::frame as the matchers see it: undist_keypts_, stereo_x_right_, descriptors_ and the grid.
struct frame_view {
    int num_keypts = 0;
    const float* x = nullptr; const float* y = nullptr; const std::int32_t* octave = nullptr; const float* angle = nullptr;
    const float* stereo_x_right = nullptr;   // nullptr: monocular
    const std::uint8_t* descriptors = nullptr;
    ovs_grid grid{};
};

class frame_index {
public:
    frame_index(const base& m, const frame_view& f) : n_(f.num_keypts) {
        detail::check(ovs_frame_index_create(m.handle(), f.num_keypts, f.x, f.y, f.octave, f.angle, f.stereo_x_right, f.descriptors, &f.grid, &h_));
    }
    //! over the device output of orb_extractor::extract_device: keypoint records and descriptors stay on the GPU
    frame_index(const base& m, const int num_keypts, const ovs_keypoint* d_keypts, const std::uint8_t* d_descriptors, const float* d_stereo_x_right,
                const ovs_grid& grid) : n_(num_keypts) {
        detail::check(ovs_frame_index_create_device(m.handle(), num_keypts, d_keypts, d_descriptors, d_stereo_x_right, &grid, &h_));
    }
    ~frame_index() { ovs_frame_index_destroy(h_); }
    frame_index(const frame_index&) = delete;
    frame_index& operator=(const frame_index&) = delete;
    ovs_frame_index* handle() const { return h_; }
    int num_keypts() const { return n_; }
private:
    ovs_frame_index* h_ = nullptr;
    int n_ = 0;
};

class robust final : public base {
public:
    explicit robust(const float lowe_ratio = 0.6, const bool check_orientation = true, const int device = 0)
        : base(lowe_ratio, check_orientation, device) {}
    //! brute_force_match(frm, keyfrm, matches): matches = (idx in frame, idx in keyframe)
    unsigned int brute_force_match(const std::uint8_t* descs_frm, const int num_keypts_frm, const std::uint8_t* descs_keyfrm,
                                   const int num_keypts_keyfrm, const std::uint8_t* keyfrm_lm_valid,
                                   std::vector<std::pair<int, int>>& matches) const {
        std::vector<std::int32_t> pairs(2 * static_cast<std::size_t>(std::max(1, std::min(num_keypts_frm, num_keypts_keyfrm))));
        int n = 0;
        detail::check(ovs_robust_brute_force_match_host(h_, descs_frm, num_keypts_frm, descs_keyfrm, num_keypts_keyfrm, keyfrm_lm_valid,
                                                        lowe_ratio_, pairs.data(), static_cast<int>(pairs.size() / 2), &n));
        matches.clear();
        for (int i = 0; i < n; ++i) matches.emplace_back(pairs[2 * i], pairs[2 * i + 1]);
        return static_cast<unsigned int>(n);
    }
    //! match_frame_and_keyframe(frm, keyfrm, matched_lms_in_frm) on arrays: brute_force_match, then the essential-matrix RANSAC on
    //! the pairs (find_via_ransac(max_num_iter, false)); matched_keyfrm_idx_of_frm[idx_1] = idx_2 of each inlier pair, else -1.
    //! bearings_*: 3 doubles per keypoint (frm.bearings_, keyfrm->bearings_).  Returns the reference's count (0: no valid solution).
    unsigned int match_frame_and_keyframe(const std::uint8_t* descs_frm, const double* bearings_frm, const int num_keypts_frm,
                                          const std::uint8_t* descs_keyfrm, const double* bearings_keyfrm, const int num_keypts_keyfrm,
                                          const std::uint8_t* keyfrm_lm_valid, std::vector<int>& matched_keyfrm_idx_of_frm,
                                          const unsigned int max_num_iter = 50, const std::uint64_t seed = 0) const {
        std::vector<std::int32_t> m(static_cast<std::size_t>(std::max(1, num_keypts_frm)), -1);
        int n = 0;
        detail::check(ovs_robust_match_frame_and_keyframe_host(h_, descs_frm, bearings_frm, num_keypts_frm, descs_keyfrm, bearings_keyfrm,
                                                               num_keypts_keyfrm, keyfrm_lm_valid, lowe_ratio_, static_cast<int>(max_num_iter),
                                                               seed, m.data(), &n));
        matched_keyfrm_idx_of_frm.assign(m.begin(), m.begin() + std::max(0, num_keypts_frm));
        return static_cast<unsigned int>(n);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (match/robust.h); bodies in adapters.hpp.  match_frame_and_keyframe reads bearings_ of the frame
    //! and the keyframe: it is a template deduced from the arguments (data::frame / data::keyframe in the reference tree), so its
    //! body is compiled only where it is called, and a data model whose frame does not carry bearings_ can use the other methods.
    unsigned int brute_force_match(data::frame& frm, data::keyframe* keyfrm, std::vector<std::pair<int, int>>& matches) const;
    template <class Frame, class Keyframe>
    unsigned int match_frame_and_keyframe(Frame& frm, Keyframe* keyfrm, std::vector<data::landmark*>& matched_lms_in_frm) const;
#endif
    //! match_for_triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs): the keyframes' BoW feature vectors come in as
    //! per-keypoint node ids; matched pairs = (idx in keyframe 1, idx in keyframe 2)
    struct triangulation_view {
        int num_keypts; const std::uint8_t* descriptors; const double* bearings; const std::int32_t* octave; const float* angle;
        const std::uint8_t* has_landmark; const std::uint8_t* is_stereo; const std::int32_t* bow_node;
    };
    unsigned int match_for_triangulation(const triangulation_view& keyfrm_1, const triangulation_view& keyfrm_2, const double* E_12,
                                         const double* epipole_in_keyfrm_2, const std::vector<float>& scale_factors_1,
                                         std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs) const {
        std::vector<std::int32_t> m(static_cast<std::size_t>(std::max(1, keyfrm_1.num_keypts)), -1);
        int n = 0;
        detail::check(ovs_robust_match_for_triangulation_host(h_, keyfrm_1.num_keypts, keyfrm_1.descriptors, keyfrm_1.bearings, keyfrm_1.octave,
                                                              keyfrm_1.angle, keyfrm_1.has_landmark, keyfrm_1.is_stereo, keyfrm_1.bow_node,
                                                              keyfrm_2.num_keypts, keyfrm_2.descriptors, keyfrm_2.bearings, keyfrm_2.angle,
                                                              keyfrm_2.has_landmark, keyfrm_2.is_stereo, keyfrm_2.bow_node, E_12, epipole_in_keyfrm_2,
                                                              scale_factors_1.data(), static_cast<int>(scale_factors_1.size()), check_orientation_,
                                                              m.data(), &n));
        matched_idx_pairs.clear();
        for (int i = 0; i < keyfrm_1.num_keypts; ++i)
            if (m[i] >= 0) matched_idx_pairs.emplace_back(static_cast<unsigned int>(i), static_cast<unsigned int>(m[i]));
        return static_cast<unsigned int>(n);
    }
};

class projection final : public base {
public:
    explicit projection(const float lowe_ratio = 0.6, const bool check_orientation = true, const int device = 0)
        : base(lowe_ratio, check_orientation, device) {}
    //! match_frame_and_landmarks(frm, local_landmarks, margin)
    unsigned int match_frame_and_landmarks(const frame_index& frm, const std::vector<float>& scale_factors, const int num_landmarks,
                                           const std::uint8_t* lm_usable, const float* reproj_in_tracking, const float* x_right_in_tracking,
                                           const std::int32_t* scale_level_in_tracking, const std::uint8_t* lm_descriptors,
                                           const std::uint8_t* kp_has_observed_lm, std::vector<std::int32_t>& matched_lm_of_kp,
                                           const float margin = 5.0) const {
        matched_lm_of_kp.assign(std::max(1, frm.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_match_frame_and_landmarks_host(frm.handle(), scale_factors.data(), static_cast<int>(scale_factors.size()), num_landmarks, lm_usable, reproj_in_tracking,
                                                                    x_right_in_tracking, scale_level_in_tracking, lm_descriptors, kp_has_observed_lm,
                                                                    margin, lowe_ratio_, matched_lm_of_kp.data(), &n));
        matched_lm_of_kp.resize(frm.num_keypts());
        return static_cast<unsigned int>(n);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signature (match/projection.h); body in adapters.hpp.
    unsigned int match_frame_and_landmarks(data::frame& frm, const std::vector<data::landmark*>& local_landmarks, const float margin = 5.0) const;
#endif
    //! match_current_and_last_frames(curr_frm, last_frm, margin)
    unsigned int match_current_and_last_frames(const frame_index& curr, const std::vector<float>& scale_factors, const int num_last_keypts,
                                               const std::uint8_t* last_usable, const float* reproj, const float* reproj_x_right,
                                               const std::int32_t* last_scale_level, const float* last_angle, const std::uint8_t* lm_descriptors,
                                               const std::uint8_t* kp_has_observed_lm, std::vector<std::int32_t>& matched_last_of_kp,
                                               const float margin, const bool assume_forward, const bool assume_backward) const {
        matched_last_of_kp.assign(std::max(1, curr.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_match_current_and_last_host(curr.handle(), scale_factors.data(), static_cast<int>(scale_factors.size()),
                                                                 num_last_keypts, last_usable, reproj, reproj_x_right, last_scale_level, last_angle,
                                                                 lm_descriptors, kp_has_observed_lm, margin, assume_forward, assume_backward,
                                                                 check_orientation_, matched_last_of_kp.data(), &n));
        matched_last_of_kp.resize(curr.num_keypts());
        return static_cast<unsigned int>(n);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signature (match/projection.h); body in adapters.hpp.  The last frame's landmarks are reprojected on the device.
    //! A template deduced from the arguments (data::frame in the reference tree), compiled only where it is called.
    template <class Frame>
    unsigned int match_current_and_last_frames(Frame& curr_frm, const Frame& last_frm, const float margin) const;
#endif
    //! frame::can_observe(lm, ray_cos_thr, reproj, x_right, pred_scale_level) for num_landmarks landmarks in one launch
    //! (ovs_frame_can_observe_host): usable = the tracker's skip rule (nullptr: all), pos_w / mean_normal 3 doubles per landmark,
    //! the raw min_valid_dist_ / max_valid_dist_; outputs one entry per landmark (reproj: 2 floats).  Returns how many are observable.
    unsigned int can_observe(const ovs_frame_geometry& geometry, const int num_landmarks, const std::uint8_t* usable, const double* pos_w,
                             const double* mean_normal, const float* min_valid_dist, const float* max_valid_dist, const float ray_cos_thr,
                             std::uint8_t* observable, float* reproj, float* x_right, std::int32_t* pred_scale_level) const {
        detail::check(ovs_frame_can_observe_host(h_, &geometry, num_landmarks, usable, pos_w, mean_normal, min_valid_dist, max_valid_dist,
                                                 ray_cos_thr, observable, reproj, x_right, pred_scale_level));
        unsigned int num = 0;
        for (int l = 0; l < num_landmarks; ++l) num += observable[l] ? 1u : 0u;
        return num;
    }
    //! The compute of tracking_module::search_local_landmarks (ovs_projection_search_local_landmarks_host): can_observe on the device,
    //! then match_frame_and_landmarks on its outputs.  The matcher is frm's (built on this or another projection handle).
    unsigned int search_local_landmarks(const frame_index& frm, const ovs_frame_geometry& geometry, const std::vector<float>& scale_factors,
                                        const int num_landmarks, const std::uint8_t* usable, const double* pos_w, const double* mean_normal,
                                        const float* min_valid_dist, const float* max_valid_dist, const std::uint8_t* lm_descriptors,
                                        const std::uint8_t* kp_has_observed_lm, std::uint8_t* observable, float* reproj, float* x_right,
                                        std::int32_t* pred_scale_level, std::vector<std::int32_t>& matched_lm_of_kp, const float margin = 5.0,
                                        const float ray_cos_thr = 0.5) const {
        if (static_cast<int>(scale_factors.size()) != geometry.num_scale_levels)
            throw std::invalid_argument("search_local_landmarks: one scale factor per level of the frame geometry");
        matched_lm_of_kp.assign(std::max(1, frm.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_search_local_landmarks_host(frm.handle(), &geometry, scale_factors.data(), num_landmarks, usable, pos_w,
                                                                 mean_normal, min_valid_dist, max_valid_dist, lm_descriptors, kp_has_observed_lm,
                                                                 ray_cos_thr, margin, lowe_ratio_, observable, reproj, x_right, pred_scale_level,
                                                                 matched_lm_of_kp.data(), &n));
        matched_lm_of_kp.resize(frm.num_keypts());
        return static_cast<unsigned int>(n);
    }
    //! match_current_and_last_frames(curr_frm, last_frm, margin) with the reprojections made on the device
    //! (ovs_projection_match_current_and_last_reproject_host): last_pose_cw = last_frm.cam_pose_cw_ as {R row-major, t}; per last
    //! keypoint: usable (landmark present, not an outlier; nullptr: all), pos_w (3 doubles), octave, angle, descriptor.
    //! in_image / reproj (optional, together): the device's reprojection of each last keypoint's landmark.
    unsigned int match_current_and_last_frames_reproject(const frame_index& curr, const ovs_frame_geometry& geometry, const bool is_monocular,
                                                         const double true_baseline, const double* last_pose_cw,
                                                         const std::vector<float>& scale_factors, const int num_last_keypts,
                                                         const std::uint8_t* last_usable, const double* pos_w, const std::int32_t* last_octave,
                                                         const float* last_angle, const std::uint8_t* lm_descriptors,
                                                         const std::uint8_t* kp_has_observed_lm, std::vector<std::int32_t>& matched_last_of_kp,
                                                         const float margin, std::uint8_t* in_image = nullptr, float* reproj = nullptr) const {
        if (static_cast<int>(scale_factors.size()) != geometry.num_scale_levels)
            throw std::invalid_argument("match_current_and_last_frames_reproject: one scale factor per level of the frame geometry");
        matched_last_of_kp.assign(std::max(1, curr.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_match_current_and_last_reproject_host(curr.handle(), &geometry, is_monocular, true_baseline, last_pose_cw,
                                                                           scale_factors.data(), num_last_keypts, last_usable, pos_w, last_octave,
                                                                           last_angle, lm_descriptors, kp_has_observed_lm, margin, check_orientation_,
                                                                           matched_last_of_kp.data(), &n, in_image, reproj));
        matched_last_of_kp.resize(curr.num_keypts());
        return static_cast<unsigned int>(n);
    }
    //! match_frame_and_keyframe(curr_frm, keyfrm, already_matched_lms, margin, hamm_dist_thr): the keyframe's landmarks
    //! reprojected into curr_frm by the caller (reproj, pred_scale_level, usable); window levels [pred - 1, pred + 1]
    unsigned int match_frame_and_keyframe(const frame_index& curr, const std::vector<float>& scale_factors, const int num_landmarks,
                                          const std::uint8_t* usable, const float* reproj, const std::int32_t* pred_scale_level,
                                          const float* keyfrm_angle, const std::uint8_t* lm_descriptors, const std::uint8_t* kp_has_lm,
                                          std::vector<std::int32_t>& matched_lm_of_kp, const float margin, const unsigned int hamm_dist_thr) const {
        return match_best_(curr, scale_factors, num_landmarks, usable, reproj, pred_scale_level, 1, keyfrm_angle, lm_descriptors, kp_has_lm,
                           matched_lm_of_kp, margin, hamm_dist_thr, check_orientation_);
    }
    //! match_by_Sim3_transform(keyfrm, Sim3_cw, landmarks, matched_lms_in_keyfrm, margin): window levels [pred - 1, pred],
    //! distance <= HAMMING_DIST_THR_LOW, no orientation check
    unsigned int match_by_Sim3_transform(const frame_index& keyfrm, const std::vector<float>& scale_factors, const int num_landmarks,
                                         const std::uint8_t* usable, const float* reproj, const std::int32_t* pred_scale_level,
                                         const std::uint8_t* lm_descriptors, const std::uint8_t* kp_already_matched,
                                         std::vector<std::int32_t>& matched_lm_of_kp, const float margin) const {
        const std::vector<float> zero(static_cast<std::size_t>(std::max(1, num_landmarks)), 0.0f);
        return match_best_(keyfrm, scale_factors, num_landmarks, usable, reproj, pred_scale_level, 0, zero.data(), lm_descriptors, kp_already_matched,
                           matched_lm_of_kp, margin, OVS_HAMMING_DIST_THR_LOW, false);
    }
    //! match_keyframes_mutually(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, Sim3s, margin): landmark arrays indexed by the
    //! keypoint of their keyframe, reprojected into the other keyframe by the caller
    unsigned int match_keyframes_mutually(const frame_index& keyfrm_1, const frame_index& keyfrm_2, const std::vector<float>& scale_factors,
                                          const std::uint8_t* usable_1, const float* reproj_1_in_2, const std::int32_t* pred_level_1_in_2,
                                          const std::uint8_t* lm_descriptors_1, const std::uint8_t* usable_2, const float* reproj_2_in_1,
                                          const std::int32_t* pred_level_2_in_1, const std::uint8_t* lm_descriptors_2,
                                          std::vector<std::int32_t>& matched_idx_2_of_kp_1, const float margin) const {
        matched_idx_2_of_kp_1.assign(std::max(1, keyfrm_1.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_match_keyframes_mutually_host(keyfrm_1.handle(), keyfrm_2.handle(), scale_factors.data(), usable_1, reproj_1_in_2,
                                                                   pred_level_1_in_2, lm_descriptors_1, usable_2, reproj_2_in_1, pred_level_2_in_1,
                                                                   lm_descriptors_2, margin, matched_idx_2_of_kp_1.data(), &n));
        matched_idx_2_of_kp_1.resize(keyfrm_1.num_keypts());
        return static_cast<unsigned int>(n);
    }

private:
    unsigned int match_best_(const frame_index& frm, const std::vector<float>& scale_factors, const int nq, const std::uint8_t* usable,
                             const float* reproj, const std::int32_t* pred_scale_level, const int levels_above, const float* q_angle,
                             const std::uint8_t* q_desc, const std::uint8_t* kp_unavailable, std::vector<std::int32_t>& matched_query_of_kp,
                             const float margin, const unsigned int hamm_dist_thr, const bool check_orientation) const {
        std::vector<float> mg(static_cast<std::size_t>(std::max(1, nq)));
        std::vector<std::int32_t> lo(mg.size()), hi(mg.size());
        for (int q = 0; q < nq; ++q) {
            const int l = pred_scale_level[q];
            mg[q] = margin * scale_factors[static_cast<std::size_t>(l < 0 ? 0 : l)];
            lo[q] = l - 1; hi[q] = l + levels_above;
        }
        matched_query_of_kp.assign(std::max(1, frm.num_keypts()), -1);
        int n = 0;
        detail::check(ovs_projection_match_best_host(frm.handle(), nq, usable, reproj, nullptr, mg.data(), lo.data(), hi.data(), q_angle, q_desc,
                                                     kp_unavailable, hamm_dist_thr, check_orientation, matched_query_of_kp.data(), &n));
        matched_query_of_kp.resize(frm.num_keypts());
        return static_cast<unsigned int>(n);
    }
};

//! match::fuse (match/fuse.h): the compute of replace_duplication for many target keyframes in one call
//! (ovs_fuse_replace_duplication_host).  The data-model updates stay with the caller: adapters.hpp replays them in the reference's
//! order.
class fuse final : public base {
public:
    explicit fuse(const float lowe_ratio = 0.6, const bool check_orientation = true, const int device = 0)
        : base(lowe_ratio, check_orientation, device) {}
    //! The landmark table the queries index: pos_w / mean_normal 3 doubles per landmark, the raw min_valid_dist_ / max_valid_dist_,
    //! the 32-byte descriptors.
    struct landmark_table {
        int num_landmarks = 0;
        const double* pos_w = nullptr; const double* mean_normal = nullptr;
        const float* min_valid_dist = nullptr; const float* max_valid_dist = nullptr;
        const std::uint8_t* descriptors = nullptr;
    };
    //! replace_duplication(keyfrm, landmarks_to_check, margin) without the data-model updates, for targets.size() target keyframes:
    //! the queries of target t are q_lm[q_off[t] .. q_off[t + 1]) (a landmark row, or -1 to skip); best_idx[q] = the keypoint of
    //! its target the landmark would be fused with, or -1.  Optional per-query geometry (nullptr: not wanted; reproj 2 floats).
    //! Returns the number of queries with a best_idx.
    unsigned int replace_duplication(const std::vector<ovs_fuse_target>& targets, const landmark_table& landmarks,
                                     const std::vector<std::int32_t>& q_off, const std::vector<std::int32_t>& q_lm, const float margin,
                                     std::vector<std::int32_t>& best_idx, std::uint8_t* passed = nullptr, float* reproj = nullptr,
                                     float* x_right = nullptr, std::int32_t* pred_level = nullptr) const {
        if (q_off.size() != targets.size() + 1 || q_off.back() != static_cast<std::int32_t>(q_lm.size()))
            throw std::invalid_argument("replace_duplication: q_off needs one entry per target plus one, ending at q_lm.size()");
        best_idx.assign(std::max<std::size_t>(1, q_lm.size()), -1);
        int n = 0;
        detail::check(ovs_fuse_replace_duplication_host(h_, static_cast<int>(targets.size()), targets.data(), landmarks.num_landmarks, landmarks.pos_w,
                                                        landmarks.mean_normal, landmarks.min_valid_dist, landmarks.max_valid_dist,
                                                        landmarks.descriptors, q_off.data(), q_lm.data(), margin, best_idx.data(), &n, passed,
                                                        reproj, x_right, pred_level));
        best_idx.resize(q_lm.size());
        ++num_calls_;
        return static_cast<unsigned int>(n);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signature (match/fuse.h); body in adapters.hpp.  A template deduced from the arguments (data::keyframe and a
    //! container of data::landmark* in the reference tree), compiled only where it is called.
    template <class Keyframe, class T>
    unsigned int replace_duplication(Keyframe* keyfrm, const T& landmarks_to_check, const float margin = 3.0) const;
#endif
    //! library calls made through this object, and the re-queries among them (adapters::fuse_landmark_duplication)
    unsigned int num_device_calls() const { return num_calls_; }
    unsigned int num_requery_calls() const { return num_requery_calls_; }
    void count_requery_call() const { ++num_requery_calls_; }

private:
    mutable unsigned int num_calls_ = 0, num_requery_calls_ = 0;
};

class area final : public base {
public:
    explicit area(const float lowe_ratio = 0.9, const bool check_orientation = true, const int device = 0)
        : base(lowe_ratio, check_orientation, device) {}
    //! match_in_consistent_area(frm_1, frm_2, prev_matched_pts, matched_indices_2_in_frm_1, margin)
    unsigned int match_in_consistent_area(const frame_view& frm_1, const frame_index& frm_2, std::vector<float>& prev_matched_pts_xy,
                                          std::vector<int>& matched_indices_2_in_frm_1, const int margin = 20) const {
        matched_indices_2_in_frm_1.assign(std::max(1, frm_1.num_keypts), -1);
        int n = 0;
        detail::check(ovs_area_match_in_consistent_area_host(frm_2.handle(), frm_1.num_keypts, frm_1.octave, frm_1.angle, frm_1.descriptors,
                                                             prev_matched_pts_xy.data(), matched_indices_2_in_frm_1.data(), margin, lowe_ratio_,
                                                             check_orientation_, &n));
        matched_indices_2_in_frm_1.resize(frm_1.num_keypts);
        return static_cast<unsigned int>(n);
    }
};

class stereo final : public base {
public:
    //! The reference constructor takes the two image pyramids; here they stay on the device inside
    //! the two extractors that produced the keypoints.
    stereo(const feature::orb_extractor& extractor_left, const feature::orb_extractor& extractor_right,
           const float focal_x_baseline, const float true_baseline, const int device = 0)
        : base(0.0f, false, device), left_(extractor_left.handle()), right_(extractor_right.handle()),
          focal_x_baseline_(focal_x_baseline), true_baseline_(true_baseline) {}
    //! compute(stereo_x_right, depths)
    void compute(const frame_view& left, const frame_view& right, std::vector<float>& stereo_x_right, std::vector<float>& depths) const {
        stereo_x_right.assign(std::max(1, left.num_keypts), -1.0f); depths.assign(std::max(1, left.num_keypts), -1.0f);
        detail::check(ovs_stereo_compute_host(h_, left_, right_, left.num_keypts, left.x, left.y, left.octave, left.descriptors, right.num_keypts,
                                              right.x, right.y, right.octave, right.descriptors, focal_x_baseline_, true_baseline_,
                                              stereo_x_right.data(), depths.data(), nullptr));
        stereo_x_right.resize(left.num_keypts); depths.resize(left.num_keypts);
    }
private:
    const ovs_extractor* left_; const ovs_extractor* right_;
    const float focal_x_baseline_, true_baseline_;
};

}  // namespace match

namespace optimize {

class pose_optimizer {
public:
    explicit pose_optimizer(const unsigned int num_trials = 4, const unsigned int num_each_iter = 10, const int device = 0)
        : num_trials_(num_trials), num_each_iter_(num_each_iter) { detail::check(ovs_optimizer_create(device, &h_)); }
    ~pose_optimizer() { ovs_optimizer_destroy(h_); }
    pose_optimizer(const pose_optimizer&) = delete;
    pose_optimizer& operator=(const pose_optimizer&) = delete;
    //! optimize(frm): pose_cw (R row-major, t) is updated in place, outlier_flags filled; returns the inlier count.
    unsigned int optimize(const ovs_camera& camera, const bool setup_is_monocular, const int num_obs, const double* pos_w, const float* undist_xy,
                          const float* stereo_x_right, const float* inv_level_sigma_sq, double* cam_pose_cw, std::vector<std::uint8_t>& outlier_flags) const {
        outlier_flags.assign(std::max(1, num_obs), 0);
        int n = 0;
        detail::check(ovs_pose_optimize_host(h_, &camera, setup_is_monocular, num_obs, pos_w, undist_xy, stereo_x_right, inv_level_sigma_sq, cam_pose_cw,
                                             outlier_flags.data(), static_cast<int>(num_trials_), static_cast<int>(num_each_iter_), &n, nullptr));
        outlier_flags.resize(num_obs);
        return static_cast<unsigned int>(n);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signature (optimize/pose_optimizer.h); body in adapters.hpp.
    unsigned int optimize(data::frame& frm) const;
#endif
private:
    const unsigned int num_trials_, num_each_iter_;
    ovs_optimizer* h_ = nullptr;
};

class local_bundle_adjuster {
public:
    explicit local_bundle_adjuster(const unsigned int num_first_iter = 5, const unsigned int num_second_iter = 10, const int device = 0)
        : num_first_iter_(num_first_iter), num_second_iter_(num_second_iter) { detail::check(ovs_optimizer_create(device, &h_)); }
    ~local_bundle_adjuster() { ovs_optimizer_destroy(h_); }
    local_bundle_adjuster(const local_bundle_adjuster&) = delete;
    local_bundle_adjuster& operator=(const local_bundle_adjuster&) = delete;
    //! optimize(curr_keyfrm, force_stop_flag) on the flattened local graph (see include/ovs_b200.h).
    void optimize(const ovs_camera& camera, const bool setup_is_monocular, const int num_keyfrms, double* cam_poses_cw, const std::uint8_t* is_fixed,
                  const int num_landmarks, double* pos_w, const int num_obs, const std::int32_t* obs_keyfrm, const std::int32_t* obs_landmark,
                  const float* undist_xy, const float* stereo_x_right, const float* inv_level_sigma_sq, bool* const force_stop_flag,
                  std::vector<std::uint8_t>& outlier_observations) const {
        outlier_observations.assign(std::max(1, num_obs), 0);
        static_assert(sizeof(bool) == 1, "the C ABI polls the flag as one byte");
        detail::check(ovs_local_ba_host(h_, &camera, setup_is_monocular, num_keyfrms, cam_poses_cw, is_fixed, num_landmarks, pos_w, num_obs, obs_keyfrm,
                                        obs_landmark, undist_xy, stereo_x_right, inv_level_sigma_sq, static_cast<int>(num_first_iter_),
                                        static_cast<int>(num_second_iter_), reinterpret_cast<const volatile std::uint8_t*>(force_stop_flag), outlier_observations.data(), nullptr));
        outlier_observations.resize(num_obs);
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signature (optimize/local_bundle_adjuster.h); body in adapters.hpp.
    void optimize(data::keyframe* curr_keyfrm, bool* const force_stop_flag) const;
#endif
private:
    const unsigned int num_first_iter_, num_second_iter_;
    ovs_optimizer* h_ = nullptr;
};

class transform_optimizer {
public:
    explicit transform_optimizer(const bool fix_scale, const unsigned int num_iter = 10, const int device = 0)
        : fix_scale_(fix_scale), num_iter_(num_iter) { detail::check(ovs_optimizer_create(device, &h_)); }
    ~transform_optimizer() { ovs_optimizer_destroy(h_); }
    transform_optimizer(const transform_optimizer&) = delete;
    transform_optimizer& operator=(const transform_optimizer&) = delete;
    //! optimize(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, g2o_Sim3_12, chi_sq) on the flattened correspondences (see
    //! include/ovs_b200.h).  sim3_12 = {R row-major (9), t (3), s}, updated only when the return value is non-zero;
    //! is_inlier[i] = 0 where the reference sets matched_lms_in_keyfrm_2 to nullptr.  Returns the inlier count.
    unsigned int optimize(const ovs_camera& camera_1, const ovs_camera& camera_2, const double* cam_pose_1w, const double* cam_pose_2w,
                          const int num_pairs, const double* pos_w_1, const float* undist_xy_1, const float* inv_level_sigma_sq_1,
                          const double* pos_w_2, const float* undist_xy_2, const float* inv_level_sigma_sq_2, double* sim3_12,
                          const float chi_sq, std::vector<std::uint8_t>& is_inlier) const {
        is_inlier.assign(std::max(1, num_pairs), 0);
        int n = 0;
        detail::check(ovs_transform_optimize_host(h_, &camera_1, &camera_2, cam_pose_1w, cam_pose_2w, num_pairs, pos_w_1, undist_xy_1,
                                                  inv_level_sigma_sq_1, pos_w_2, undist_xy_2, inv_level_sigma_sq_2, fix_scale_ ? 1 : 0, chi_sq,
                                                  5, static_cast<int>(num_iter_), sim3_12, is_inlier.data(), &n, nullptr));
        is_inlier.resize(num_pairs);
        return static_cast<unsigned int>(n);
    }
private:
    const bool fix_scale_;
    const unsigned int num_iter_;
    ovs_optimizer* h_ = nullptr;
};

class graph_optimizer {
public:
    explicit graph_optimizer(const bool fix_scale, const unsigned int num_iter = 50, const int device = 0)
        : fix_scale_(fix_scale), num_iter_(num_iter) { detail::check(ovs_optimizer_create(device, &h_)); }
    ~graph_optimizer() { ovs_optimizer_destroy(h_); }
    graph_optimizer(const graph_optimizer&) = delete;
    graph_optimizer& operator=(const graph_optimizer&) = delete;
    //! optimize(loop_keyfrm, curr_keyfrm, non_corrected_Sim3s, pre_corrected_Sim3s, loop_connections) on the flattened pose graph
    //! (see include/ovs_b200.h and INTEGRATION.md): sim3_cw[K*13] = S_iw {R row-major (9), t (3), s}, updated in place;
    //! landmarks pos_w[L*3] corrected through their reference vertex (-1: unchanged); cam_poses_cw[K*12] = {R, t / s} (may be null).
    void optimize(const int num_keyfrms, double* sim3_cw, const std::uint8_t* is_fixed, const int num_edges, const std::int32_t* edge_i,
                  const std::int32_t* edge_j, const double* meas_Sji, const int num_landmarks, double* pos_w, const std::int32_t* ref_vertex,
                  double* cam_poses_cw) const {
        detail::check(ovs_graph_optimize_host(h_, num_keyfrms, sim3_cw, is_fixed, num_edges, edge_i, edge_j, meas_Sji, fix_scale_ ? 1 : 0,
                                              static_cast<int>(num_iter_), num_landmarks, pos_w, ref_vertex, cam_poses_cw, nullptr));
    }
private:
    const bool fix_scale_;
    const unsigned int num_iter_;
    ovs_optimizer* h_ = nullptr;
};

}  // namespace optimize

namespace solve {

//! solve::sim3_solver (loop detection): RANSAC over Horn's closed-form Sim3 on three landmark pairs.  The reference builds one
//! solver per loop candidate; here find_via_ransac(problems, max_num_iter) solves a whole batch of candidates in one call, and
//! the reference's per-candidate constructor / find_via_ransac(max_num_iter) / getters are in adapters.hpp.
class sim3_solver {
public:
    //! One loop candidate on array views (see include/ovs_b200.h, ovs_sim3_solve_ransac_host).
    struct problem_view {
        ovs_camera camera_1{}, camera_2{};
        const double* cam_pose_1w = nullptr; const double* cam_pose_2w = nullptr;   // {R row-major (9), t (3)}
        int num_pairs = 0;
        const double* pos_w_1 = nullptr; const float* level_sigma_sq_1 = nullptr;
        const double* pos_w_2 = nullptr; const float* level_sigma_sq_2 = nullptr;
        std::uint64_t seed = 0;
    };
    struct solution {
        bool valid = false;
        double sim3_12[13] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1};   // {R row-major (9), t (3), s}
        unsigned int num_inliers = 0;
        int best_iter = -1;
        std::vector<std::uint8_t> is_inlier;
    };

    explicit sim3_solver(const bool fix_scale, const unsigned int min_num_inliers = 20, const int device = 0)
        : fix_scale_(fix_scale), min_num_inliers_(min_num_inliers) { detail::check(ovs_optimizer_create(device, &h_)); }
    ~sim3_solver() { ovs_optimizer_destroy(h_); }
    sim3_solver(const sim3_solver&) = delete;
    sim3_solver& operator=(const sim3_solver&) = delete;

    //! find_via_ransac(max_num_iter) for every problem, one GPU call
    std::vector<solution> find_via_ransac(const std::vector<problem_view>& problems, const unsigned int max_num_iter = 200) const {
        const int B = static_cast<int>(problems.size());
        std::vector<std::int32_t> off(static_cast<std::size_t>(B) + 1, 0);
        for (int b = 0; b < B; ++b) off[b + 1] = off[b] + problems[b].num_pairs;
        const std::size_t N = static_cast<std::size_t>(off[B]);
        std::vector<ovs_camera> c1(B), c2(B);
        std::vector<double> p1(12 * static_cast<std::size_t>(B)), p2(12 * static_cast<std::size_t>(B)), w1(3 * N), w2(3 * N);
        std::vector<float> s1(N), s2(N);
        std::vector<std::uint64_t> seeds(B);
        for (int b = 0; b < B; ++b) {
            const problem_view& p = problems[b];
            c1[b] = p.camera_1; c2[b] = p.camera_2; seeds[b] = p.seed;
            std::memcpy(&p1[12 * b], p.cam_pose_1w, 96); std::memcpy(&p2[12 * b], p.cam_pose_2w, 96);
            const std::size_t o = static_cast<std::size_t>(off[b]), n = static_cast<std::size_t>(p.num_pairs);
            if (n == 0) continue;
            std::memcpy(&w1[3 * o], p.pos_w_1, 24 * n); std::memcpy(&w2[3 * o], p.pos_w_2, 24 * n);
            std::memcpy(&s1[o], p.level_sigma_sq_1, 4 * n); std::memcpy(&s2[o], p.level_sigma_sq_2, 4 * n);
        }
        std::vector<double> S(13 * static_cast<std::size_t>(std::max(B, 1)));
        std::vector<std::uint8_t> valid(std::max(B, 1)), flags(std::max<std::size_t>(N, 1));
        std::vector<std::int32_t> num(std::max(B, 1)), best(std::max(B, 1));
        detail::check(ovs_sim3_solve_ransac_host(h_, B, off.data(), c1.data(), p1.data(), c2.data(), p2.data(), w1.data(), s1.data(), w2.data(),
                                                 s2.data(), fix_scale_ ? 1 : 0, static_cast<int>(min_num_inliers_), static_cast<int>(max_num_iter),
                                                 seeds.data(), S.data(), valid.data(), num.data(), best.data(), flags.data()));
        std::vector<solution> out(B);
        for (int b = 0; b < B; ++b) {
            out[b].valid = valid[b] != 0;
            std::memcpy(out[b].sim3_12, &S[13 * static_cast<std::size_t>(b)], 13 * sizeof(double));
            out[b].num_inliers = static_cast<unsigned int>(num[b]);
            out[b].best_iter = best[b];
            out[b].is_inlier.assign(flags.begin() + off[b], flags.begin() + off[b + 1]);
        }
        return out;
    }

#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (solve/sim3_solver.h); bodies in adapters.hpp.  The sampler is seeded with
    //! (keyfrm_1->id_ << 32) | keyfrm_2->id_.
    sim3_solver(data::keyframe* keyfrm_1, data::keyframe* keyfrm_2, const std::vector<data::landmark*>& matched_lms_in_keyfrm_2,
                const bool fix_scale, const unsigned int min_num_inliers = 20);
    void find_via_ransac(const unsigned int max_num_iter);
    bool solution_is_valid() const { return best_.valid; }
    Mat33_t get_best_rotation_12() const;
    Vec3_t get_best_translation_12() const;
    float get_best_scale_12() const { return static_cast<float>(best_.sim3_12[12]); }
#endif
    //! the last find_via_ransac(max_num_iter) of a solver built with the reference's constructor
    const solution& best_solution() const { return best_; }

private:
    const bool fix_scale_;
    const unsigned int min_num_inliers_;
    ovs_optimizer* h_ = nullptr;
    problem_view own_{};                                   // the reference constructor's flattened candidate
    std::vector<double> own_pos_w_1_, own_pos_w_2_, own_poses_;
    std::vector<float> own_sigma_sq_1_, own_sigma_sq_2_;
    solution best_{};
};

//! solve::pnp_solver (relocalisation): RANSAC over EPnP on minimal sets of 6 bearing-landmark correspondences, with an optional
//! EPnP recompute on all inliers.  The reference builds one solver per relocalisation candidate; here
//! find_via_ransac(problems, max_num_iter, recompute) solves a whole batch of candidates in one call, and the reference's
//! per-candidate constructor / find_via_ransac(max_num_iter, recompute) / getters are in adapters.hpp.
class pnp_solver {
public:
    //! One relocalisation candidate on array views (see include/ovs_b200.h, ovs_pnp_solve_ransac_host).
    struct problem_view {
        int num_corrs = 0;
        const double* bearings = nullptr;                  // 3 per correspondence, unit
        const double* pos_w = nullptr;                     // 3 per correspondence
        const float* scale_factor = nullptr;               // scale_factors_[octave] per correspondence
        std::uint64_t seed = 0;
    };
    struct solution {
        bool valid = false;
        double pose_cw[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};   // {R row-major (9), t (3)}
        unsigned int num_inliers = 0;
        int best_iter = -1;
        std::vector<std::uint8_t> is_inlier;
    };

    explicit pnp_solver(const unsigned int min_num_inliers = 10, const int device = 0) : min_num_inliers_(min_num_inliers) {
        detail::check(ovs_optimizer_create(device, &h_));
    }
    ~pnp_solver() { ovs_optimizer_destroy(h_); }
    pnp_solver(const pnp_solver&) = delete;
    pnp_solver& operator=(const pnp_solver&) = delete;

    //! find_via_ransac(max_num_iter, recompute) for every problem, one GPU call
    std::vector<solution> find_via_ransac(const std::vector<problem_view>& problems, const unsigned int max_num_iter = 30,
                                          const bool recompute = true) const {
        const int B = static_cast<int>(problems.size());
        std::vector<std::int32_t> off(static_cast<std::size_t>(B) + 1, 0);
        for (int b = 0; b < B; ++b) off[b + 1] = off[b] + problems[b].num_corrs;
        const std::size_t N = static_cast<std::size_t>(off[B]);
        std::vector<double> bear(3 * N), pw(3 * N);
        std::vector<float> sf(N);
        std::vector<std::uint64_t> seeds(B);
        for (int b = 0; b < B; ++b) {
            const problem_view& p = problems[b];
            seeds[b] = p.seed;
            const std::size_t o = static_cast<std::size_t>(off[b]), n = static_cast<std::size_t>(p.num_corrs);
            if (n == 0) continue;
            std::memcpy(&bear[3 * o], p.bearings, 24 * n); std::memcpy(&pw[3 * o], p.pos_w, 24 * n);
            std::memcpy(&sf[o], p.scale_factor, 4 * n);
        }
        std::vector<double> pose(12 * static_cast<std::size_t>(std::max(B, 1)));
        std::vector<std::uint8_t> valid(std::max(B, 1)), flags(std::max<std::size_t>(N, 1));
        std::vector<std::int32_t> num(std::max(B, 1)), best(std::max(B, 1));
        detail::check(ovs_pnp_solve_ransac_host(h_, B, off.data(), bear.data(), pw.data(), sf.data(), static_cast<int>(min_num_inliers_),
                                                static_cast<int>(max_num_iter), recompute ? 1 : 0, seeds.data(), pose.data(), valid.data(),
                                                num.data(), best.data(), flags.data()));
        std::vector<solution> out(B);
        for (int b = 0; b < B; ++b) {
            out[b].valid = valid[b] != 0;
            std::memcpy(out[b].pose_cw, &pose[12 * static_cast<std::size_t>(b)], 12 * sizeof(double));
            out[b].num_inliers = static_cast<unsigned int>(num[b]);
            out[b].best_iter = best[b];
            out[b].is_inlier.assign(flags.begin() + off[b], flags.begin() + off[b + 1]);
        }
        return out;
    }

#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (solve/pnp_solver.h); bodies in adapters.hpp.  The constructor receives no frame or keyframe
    //! id, so the sampler is seeded with a splitmix64 hash of the input bits (the batched call takes explicit seeds).  The bearing
    //! and point containers are template parameters: the reference passes eigen_alloc_vector<bearing_t> / eigen_alloc_vector<Vec3_t>
    //! (std::vector with Eigen's aligned allocator); any random-access container of 3-vectors indexed as v(k) is accepted.
    template <class BearingVector, class PointVector>
    pnp_solver(const BearingVector& valid_bearings, const std::vector<cv::KeyPoint>& valid_keypts, const PointVector& valid_points,
               const std::vector<float>& scale_factors, const unsigned int min_num_inliers = 10);
    void find_via_ransac(const unsigned int max_num_iter, const bool recompute = true);
    bool solution_is_valid() const { return best_.valid; }
    Mat33_t get_best_rotation() const;
    Vec3_t get_best_translation() const;
    Mat44_t get_best_cam_pose() const;
    std::vector<bool> get_inlier_flags() const { return std::vector<bool>(best_.is_inlier.begin(), best_.is_inlier.end()); }
#endif
    //! the last find_via_ransac(max_num_iter, recompute) of a solver built with the reference's constructor
    const solution& best_solution() const { return best_; }

private:
    const unsigned int min_num_inliers_;
    ovs_optimizer* h_ = nullptr;
    problem_view own_{};                                   // the reference constructor's flattened candidate
    std::vector<double> own_bearings_, own_pos_w_;
    std::vector<float> own_scale_factor_;
    solution best_{};
};

//! solve::essential_solver (the tracker's robust match, equirectangular map initialisation): RANSAC over the eight-point algorithm
//! on bearing matches, with an optional refit on all inliers.  The reference builds one solver per pair of views; here
//! find_via_ransac(problems, max_num_iter, recompute) solves a whole batch in one call, and the reference's constructor /
//! find_via_ransac(max_num_iter, recompute) / getters are in adapters.hpp.
class essential_solver {
public:
    //! One problem on array views (see include/ovs_b200.h, ovs_essential_solve_ransac_host).
    struct problem_view {
        int num_matches = 0;
        const double* bearings_1 = nullptr;               // 3 per match, unit: bearings_1_[matches_12_[i].first]
        const double* bearings_2 = nullptr;               // 3 per match, unit: bearings_2_[matches_12_[i].second]
        std::uint64_t seed = 0;
    };
    struct solution {
        bool valid = false;
        double E_21[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};     // row-major, b2^T E_21 b1 = 0
        unsigned int num_inliers = 0;
        int best_iter = -1;
        double best_score = 0.0;
        std::vector<std::uint8_t> is_inlier;
    };

    explicit essential_solver(const int device = 0) { detail::check(ovs_matcher_create(device, &h_)); }
    ~essential_solver() { ovs_matcher_destroy(h_); }
    essential_solver(const essential_solver&) = delete;
    essential_solver& operator=(const essential_solver&) = delete;

    //! find_via_ransac(max_num_iter, recompute) for every problem, one GPU call
    std::vector<solution> find_via_ransac(const std::vector<problem_view>& problems, const unsigned int max_num_iter,
                                          const bool recompute = true) const {
        const int B = static_cast<int>(problems.size());
        std::vector<std::int32_t> off(static_cast<std::size_t>(B) + 1, 0);
        for (int b = 0; b < B; ++b) off[b + 1] = off[b] + problems[b].num_matches;
        const std::size_t N = static_cast<std::size_t>(off[B]);
        std::vector<double> b1(std::max<std::size_t>(3 * N, 3)), b2(std::max<std::size_t>(3 * N, 3));
        std::vector<std::uint64_t> seeds(std::max(B, 1));
        for (int b = 0; b < B; ++b) {
            const problem_view& p = problems[b];
            seeds[b] = p.seed;
            const std::size_t o = static_cast<std::size_t>(off[b]), n = static_cast<std::size_t>(p.num_matches);
            if (n == 0) continue;
            std::memcpy(&b1[3 * o], p.bearings_1, 24 * n); std::memcpy(&b2[3 * o], p.bearings_2, 24 * n);
        }
        std::vector<double> E(9 * static_cast<std::size_t>(std::max(B, 1))), score(std::max(B, 1));
        std::vector<std::uint8_t> valid(std::max(B, 1)), flags(std::max<std::size_t>(N, 1));
        std::vector<std::int32_t> num(std::max(B, 1)), best(std::max(B, 1));
        detail::check(ovs_essential_solve_ransac_host(h_, B, off.data(), b1.data(), b2.data(), static_cast<int>(max_num_iter), recompute ? 1 : 0,
                                                      seeds.data(), E.data(), valid.data(), num.data(), best.data(), score.data(), flags.data()));
        std::vector<solution> out(B);
        for (int b = 0; b < B; ++b) {
            out[b].valid = valid[b] != 0;
            std::memcpy(out[b].E_21, &E[9 * static_cast<std::size_t>(b)], 9 * sizeof(double));
            out[b].num_inliers = static_cast<unsigned int>(num[b]);
            out[b].best_iter = best[b];
            out[b].best_score = score[b];
            out[b].is_inlier.assign(flags.begin() + off[b], flags.begin() + off[b + 1]);
        }
        return out;
    }

#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (solve/essential_solver.h); bodies in adapters.hpp.  The sampler is seeded with a splitmix64 hash
    //! of the input bits (the batched call takes explicit seeds).  The bearing container is a template parameter: the reference
    //! passes eigen_alloc_vector<bearing_t>; any random-access container of 3-vectors indexed as v(k) is accepted.
    template <class BearingVector>
    essential_solver(const BearingVector& bearings_1, const BearingVector& bearings_2, const std::vector<std::pair<int, int>>& matches_12);
    void find_via_ransac(const unsigned int max_num_iter, const bool recompute = true);
    bool solution_is_valid() const { return best_.valid; }
    Mat33_t get_best_E_21() const;
    std::vector<bool> get_inlier_matches() const { return std::vector<bool>(best_.is_inlier.begin(), best_.is_inlier.end()); }
#endif
    //! the last find_via_ransac(max_num_iter, recompute) of a solver built with the reference's constructor
    const solution& best_solution() const { return best_; }

private:
    ovs_matcher* h_ = nullptr;
    problem_view own_{};                                   // the reference constructor's flattened matches
    std::vector<double> own_bearings_1_, own_bearings_2_;
    solution best_{};
};

//! The batched find_via_ransac shared by homography_solver and fundamental_solver (the same arguments, one entry point each).
class two_view_solver_base {
public:
    //! One problem on array views (see include/ovs_b200.h, ovs_homography_solve_ransac_host).
    struct problem_view {
        int num_keypts_1 = 0, num_keypts_2 = 0;
        const ovs_keypoint* keypts_1 = nullptr;           // all undistorted keypoints of view 1 (only pt is read)
        const ovs_keypoint* keypts_2 = nullptr;           // the same of view 2
        int num_matches = 0;
        const std::int32_t* matches_12 = nullptr;         // 2 per match: idx_1, idx_2
        std::uint64_t seed = 0;
    };
    struct solution {
        bool valid = false;
        double M_21[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};     // row-major H_21 or F_21
        unsigned int num_inliers = 0;
        int best_iter = -1;
        double best_score = 0.0;
        std::vector<std::uint8_t> is_inlier;
    };
    using entry_t = int (*)(ovs_matcher*, int, const std::int32_t*, const ovs_keypoint*, const std::int32_t*, const ovs_keypoint*,
                            const std::int32_t*, const std::int32_t*, float, int, int, const std::uint64_t*, double*, std::uint8_t*,
                            std::int32_t*, std::int32_t*, double*, std::uint8_t*);

    two_view_solver_base(entry_t entry, const float sigma, const int device) : entry_(entry), sigma_(sigma) {
        detail::check(ovs_matcher_create(device, &h_));
    }
    ~two_view_solver_base() { ovs_matcher_destroy(h_); }
    two_view_solver_base(const two_view_solver_base&) = delete;
    two_view_solver_base& operator=(const two_view_solver_base&) = delete;

    //! find_via_ransac(max_num_iter, recompute) for every problem, one GPU call
    std::vector<solution> find_via_ransac(const std::vector<problem_view>& problems, const unsigned int max_num_iter,
                                          const bool recompute = true) const {
        const int B = static_cast<int>(problems.size());
        std::vector<std::int32_t> o1(static_cast<std::size_t>(B) + 1, 0), o2(o1), om(o1);
        for (int b = 0; b < B; ++b) {
            o1[b + 1] = o1[b] + problems[b].num_keypts_1;
            o2[b + 1] = o2[b] + problems[b].num_keypts_2;
            om[b + 1] = om[b] + problems[b].num_matches;
        }
        std::vector<ovs_keypoint> k1(std::max(o1[B], 1)), k2(std::max(o2[B], 1));
        std::vector<std::int32_t> mt(2 * static_cast<std::size_t>(std::max(om[B], 1)));
        std::vector<std::uint64_t> seeds(std::max(B, 1));
        for (int b = 0; b < B; ++b) {
            const problem_view& p = problems[b];
            seeds[b] = p.seed;
            if (p.num_keypts_1) std::memcpy(&k1[o1[b]], p.keypts_1, sizeof(ovs_keypoint) * p.num_keypts_1);
            if (p.num_keypts_2) std::memcpy(&k2[o2[b]], p.keypts_2, sizeof(ovs_keypoint) * p.num_keypts_2);
            if (p.num_matches) std::memcpy(&mt[2 * static_cast<std::size_t>(om[b])], p.matches_12, 8 * static_cast<std::size_t>(p.num_matches));
        }
        std::vector<double> M(9 * static_cast<std::size_t>(std::max(B, 1))), score(std::max(B, 1));
        std::vector<std::uint8_t> valid(std::max(B, 1)), flags(std::max(om[B], 1));
        std::vector<std::int32_t> num(std::max(B, 1)), best(std::max(B, 1));
        detail::check(entry_(h_, B, o1.data(), k1.data(), o2.data(), k2.data(), om.data(), mt.data(), sigma_, static_cast<int>(max_num_iter),
                     recompute ? 1 : 0, seeds.data(), M.data(), valid.data(), num.data(), best.data(), score.data(), flags.data()));
        std::vector<solution> out(B);
        for (int b = 0; b < B; ++b) {
            out[b].valid = valid[b] != 0;
            std::memcpy(out[b].M_21, &M[9 * static_cast<std::size_t>(b)], 9 * sizeof(double));
            out[b].num_inliers = static_cast<unsigned int>(num[b]);
            out[b].best_iter = best[b];
            out[b].best_score = score[b];
            out[b].is_inlier.assign(flags.begin() + om[b], flags.begin() + om[b + 1]);
        }
        return out;
    }

    //! the last find_via_ransac(max_num_iter, recompute) of a solver built with the reference's constructor
    const solution& best_solution() const { return best_; }

protected:
    entry_t entry_;
    float sigma_;
    ovs_matcher* h_ = nullptr;
    problem_view own_{};                                   // the reference constructor's problem
    std::vector<ovs_keypoint> own_keypts_1_, own_keypts_2_;
    std::vector<std::int32_t> own_matches_;
    solution best_{};
};

//! solve::homography_solver (perspective map initialisation): RANSAC over the normalised 8-point DLT on keypoint matches, with an
//! optional refit on all inliers.  The reference builds one solver per pair of views; here find_via_ransac(problems, max_num_iter,
//! recompute) solves a whole batch in one call, and the reference's constructor / find_via_ransac(max_num_iter, recompute) /
//! getters are in adapters.hpp.  H_21 maps view 1 to view 2: p2 ~ H_21 p1.
class homography_solver : public two_view_solver_base {
public:
    explicit homography_solver(const float sigma = 1.0f, const int device = 0)
        : two_view_solver_base(&ovs_homography_solve_ransac_host, sigma, device) {}
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (solve/homography_solver.h); bodies in adapters.hpp.  The sampler is seeded with a splitmix64
    //! hash of the input bits (the batched call takes explicit seeds).
    homography_solver(const std::vector<cv::KeyPoint>& undist_keypts_1, const std::vector<cv::KeyPoint>& undist_keypts_2,
                      const std::vector<std::pair<int, int>>& matches_12, const float sigma);
    void find_via_ransac(const unsigned int max_num_iter, const bool recompute = true);
    bool solution_is_valid() const { return best_.valid; }
    float get_best_score() const { return static_cast<float>(best_.best_score); }
    Mat33_t get_best_H_21() const;
    std::vector<bool> get_inlier_matches() const { return std::vector<bool>(best_.is_inlier.begin(), best_.is_inlier.end()); }
#endif
    using two_view_solver_base::find_via_ransac;
};

//! solve::fundamental_solver (perspective map initialisation): RANSAC over the normalised eight-point algorithm with a rank-2
//! projection; the same interface as homography_solver.  p2^T F_21 p1 = 0.
class fundamental_solver : public two_view_solver_base {
public:
    explicit fundamental_solver(const float sigma = 1.0f, const int device = 0)
        : two_view_solver_base(&ovs_fundamental_solve_ransac_host, sigma, device) {}
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's signatures (solve/fundamental_solver.h); bodies in adapters.hpp.
    fundamental_solver(const std::vector<cv::KeyPoint>& undist_keypts_1, const std::vector<cv::KeyPoint>& undist_keypts_2,
                       const std::vector<std::pair<int, int>>& matches_12, const float sigma);
    void find_via_ransac(const unsigned int max_num_iter, const bool recompute = true);
    bool solution_is_valid() const { return best_.valid; }
    float get_best_score() const { return static_cast<float>(best_.best_score); }
    Mat33_t get_best_F_21() const;
    std::vector<bool> get_inlier_matches() const { return std::vector<bool>(best_.is_inlier.begin(), best_.is_inlier.end()); }
#endif
    using two_view_solver_base::find_via_ransac;
};

}  // namespace solve

namespace module {

//! module::two_view_triangulator (module/two_view_triangulator.h) on array views (ovs_keyframe_view: a keyframe's own vectors),
//! and the compute step of mapping_module::create_new_landmarks.  Owns a matcher handle (its CUDA stream and buffers).
class two_view_triangulator {
public:
    //! One keyframe pair and its pairs (idx_1, idx_2) for the batched triangulate.
    struct problem {
        const ovs_keyframe_view* keyfrm_1;
        const ovs_keyframe_view* keyfrm_2;
        std::vector<std::pair<unsigned int, unsigned int>> pairs;
    };

    explicit two_view_triangulator(const float rays_parallax_deg_thr = 1.0, const int device = 0)
        : rays_parallax_deg_thr_(rays_parallax_deg_thr) {
        detail::check(ovs_matcher_create(device, &h_));
    }
    //! The reference's constructor arguments: keyfrm_1, keyfrm_2 (the views must outlive the object), rays_parallax_deg_thr.
    two_view_triangulator(const ovs_keyframe_view& keyfrm_1, const ovs_keyframe_view& keyfrm_2, const float rays_parallax_deg_thr,
                          const int device = 0)
        : two_view_triangulator(rays_parallax_deg_thr, device) {
        keyfrm_1_ = &keyfrm_1; keyfrm_2_ = &keyfrm_2;
    }
    ~two_view_triangulator() { ovs_matcher_destroy(h_); }
    two_view_triangulator(const two_view_triangulator&) = delete;
    two_view_triangulator& operator=(const two_view_triangulator&) = delete;
    ovs_matcher* handle() const { return h_; }

    //! triangulate(idx_1, idx_2, pos_w) of the constructor's keyframe pair for every pair of the list in one GPU call:
    //! valid[m] = the reference's return value, pos_w[3 m] = the point (zero where invalid).
    void triangulate(const std::vector<std::pair<unsigned int, unsigned int>>& pairs, std::vector<std::uint8_t>& valid,
                     std::vector<double>& pos_w) const {
        if (!keyfrm_1_ || !keyfrm_2_) throw std::runtime_error("ovs_b200: two_view_triangulator built without its keyframes");
        std::vector<std::vector<std::uint8_t>> v;
        std::vector<std::vector<double>> p;
        triangulate(std::vector<problem>{problem{keyfrm_1_, keyfrm_2_, pairs}}, v, p);
        valid = std::move(v.front()); pos_w = std::move(p.front());
    }
    //! The same for B keyframe pairs in one GPU call; valid[b] / pos_w[b] per problem.
    void triangulate(const std::vector<problem>& problems, std::vector<std::vector<std::uint8_t>>& valid,
                     std::vector<std::vector<double>>& pos_w) const {
        const std::size_t B = problems.size();
        std::vector<ovs_keyframe_view> k1(B), k2(B);
        std::vector<std::int32_t> off(B + 1, 0), pairs;
        for (std::size_t b = 0; b < B; ++b) {
            k1[b] = *problems[b].keyfrm_1; k2[b] = *problems[b].keyfrm_2;
            for (const auto& pr : problems[b].pairs) { pairs.push_back(static_cast<std::int32_t>(pr.first)); pairs.push_back(static_cast<std::int32_t>(pr.second)); }
            off[b + 1] = static_cast<std::int32_t>(pairs.size() / 2);
        }
        const std::size_t M = pairs.size() / 2;
        std::vector<std::uint8_t> v(std::max<std::size_t>(M, 1));
        std::vector<double> p(3 * std::max<std::size_t>(M, 1));
        detail::check(ovs_two_view_triangulate_host(h_, static_cast<int>(B), k1.data(), k2.data(), off.data(), pairs.data(),
                                                    rays_parallax_deg_thr_, v.data(), p.data()));
        valid.assign(B, {}); pos_w.assign(B, {});
        for (std::size_t b = 0; b < B; ++b) {
            valid[b].assign(v.begin() + off[b], v.begin() + off[b + 1]);
            pos_w[b].assign(p.begin() + 3 * static_cast<std::size_t>(off[b]), p.begin() + 3 * static_cast<std::size_t>(off[b + 1]));
        }
    }

    //! create_new_landmarks' compute step (ovs_create_new_landmarks_host): for each neighbour in order, match_for_triangulation
    //! with keyframe 1's landmark flags as they stand (E_12[b] row-major, epipole_in_2[b] = keyframe 1's centre as a bearing of
    //! neighbour b), then this triangulator on its pairs.  Returns the records in creation order; creating the landmarks stays with
    //! the caller.  Neighbour b's records depend on neighbours 0 .. b only (the prefix rule of ovs_b200.h).
    std::vector<ovs_new_landmark> create_new_landmarks(const ovs_keyframe_view& keyfrm_1, const std::vector<ovs_keyframe_view>& neighbours,
                                                       const std::vector<std::array<double, 9>>& E_12,
                                                       const std::vector<std::array<double, 3>>& epipole_in_2,
                                                       const bool check_orientation) const {
        const std::size_t B = neighbours.size();
        if (E_12.size() != B || epipole_in_2.size() != B) throw std::runtime_error("ovs_b200: one E_12 and one epipole per neighbour");
        std::vector<double> E(9 * B), ep(3 * B);
        for (std::size_t b = 0; b < B; ++b) {
            std::copy(E_12[b].begin(), E_12[b].end(), E.begin() + 9 * b);
            std::copy(epipole_in_2[b].begin(), epipole_in_2[b].end(), ep.begin() + 3 * b);
        }
        std::vector<ovs_new_landmark> out(static_cast<std::size_t>(std::max(keyfrm_1.num_keypts, 1)));
        int n = 0;
        detail::check(ovs_create_new_landmarks_host(h_, &keyfrm_1, static_cast<int>(B), neighbours.data(), E.data(), ep.data(),
                                                    check_orientation ? 1 : 0, rays_parallax_deg_thr_, out.data(),
                                                    keyfrm_1.num_keypts, &n));
        out.resize(static_cast<std::size_t>(n));
        return out;
    }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The same on the reference's keyframes (data::keyframe in the reference tree; body in adapters.hpp): flattens each keyframe,
    //! forms E_12 and the epipole from the poses as the reference does.  A template deduced from its arguments, so it is compiled
    //! only where it is called.
    template <class Keyframe>
    std::vector<ovs_new_landmark> create_new_landmarks(Keyframe* keyfrm_1, const std::vector<Keyframe*>& neighbours,
                                                       const bool check_orientation) const;
#endif

private:
    const float rays_parallax_deg_thr_;
    const ovs_keyframe_view* keyfrm_1_ = nullptr;
    const ovs_keyframe_view* keyfrm_2_ = nullptr;
    ovs_matcher* h_ = nullptr;
};

}  // namespace module

namespace initialize {

//! What initialize::perspective and initialize::bearing_vector share (initialize/base.h): the constructor's settings, a matcher
//! handle (its CUDA stream and buffers) and the outcome of the last initialize().  On array views (ovs_init_view: a frame's
//! camera, undist_keypts_.data() and its bearings as 3 doubles per keypoint; the views must outlive the call).
class base {
public:
    //! One problem of the batched form: a reference view, a current view, ref_matches_with_cur (one entry per reference keypoint,
    //! -1 = none) and the sampler seed.
    struct problem {
        const ovs_init_view* ref;
        const ovs_init_view* cur;
        std::vector<int> ref_matches_with_cur;
        std::uint64_t seed;
    };
    //! One problem's outcome: the C ABI's record, and per reference keypoint the flag and the point (3 doubles).
    struct result {
        ovs_init_result record;
        std::vector<std::uint8_t> is_triangulated;
        std::vector<double> triangulated_pts;
    };

    base(const base&) = delete;
    base& operator=(const base&) = delete;
    virtual ~base() { ovs_matcher_destroy(h_); }
    ovs_matcher* handle() const { return h_; }

    //! initialize(cur_frm, ref_matches_with_cur) on the constructor's reference view with one sampler seed (used by every solver
    //! of the call).  True when the map can be built from the getters below.
    bool initialize(const ovs_init_view& cur, const std::vector<int>& ref_matches_with_cur, const std::uint64_t seed) {
        if (!ref_) throw std::runtime_error("ovs_b200: initializer built without its reference view");
        std::vector<result> r;
        initialize(std::vector<problem>{problem{ref_, &cur, ref_matches_with_cur, seed}}, r);
        last_ = std::move(r.front());
        return last_.record.status == OVS_INIT_OK;
    }
    //! The same for B problems in one GPU call, with this object's settings; results[b] per problem.
    void initialize(const std::vector<problem>& problems, std::vector<result>& results) const {
        const std::size_t B = problems.size();
        std::vector<ovs_init_view> refs(B), curs(B);
        std::vector<std::int32_t> rm;
        std::vector<std::uint64_t> seeds(B);
        std::vector<std::size_t> off(B + 1, 0);
        for (std::size_t b = 0; b < B; ++b) {
            refs[b] = *problems[b].ref; curs[b] = *problems[b].cur; seeds[b] = problems[b].seed;
            if (problems[b].ref_matches_with_cur.size() != static_cast<std::size_t>(refs[b].num_keypts))
                throw std::runtime_error("ovs_b200: ref_matches_with_cur needs one entry per reference keypoint");
            rm.insert(rm.end(), problems[b].ref_matches_with_cur.begin(), problems[b].ref_matches_with_cur.end());
            off[b + 1] = rm.size();
        }
        const std::size_t K = rm.size();
        std::vector<ovs_init_result> rec(std::max<std::size_t>(B, 1));
        std::vector<std::uint8_t> flags(std::max<std::size_t>(K, 1));
        std::vector<double> pts(3 * std::max<std::size_t>(K, 1));
        detail::check((perspective_ ? ovs_initialize_perspective_host : ovs_initialize_bearing_vector_host)(
            h_, static_cast<int>(B), refs.data(), curs.data(), rm.data(), static_cast<int>(num_ransac_iters_),
            static_cast<int>(min_num_triangulated_), parallax_deg_thr_, reproj_err_thr_sq_, seeds.data(), rec.data(), flags.data(), pts.data()));
        results.assign(B, result{});
        for (std::size_t b = 0; b < B; ++b) {
            results[b].record = rec[b];
            results[b].is_triangulated.assign(flags.begin() + off[b], flags.begin() + off[b + 1]);
            results[b].triangulated_pts.assign(pts.begin() + 3 * off[b], pts.begin() + 3 * off[b + 1]);
        }
    }

    //! The last initialize()'s outcome on arrays: R row-major, t (unit norm), the flags and points per reference keypoint.
    const ovs_init_result& last_result() const { return last_.record; }
    std::array<double, 9> rotation_ref_to_cur() const {
        std::array<double, 9> R;
        std::copy(last_.record.rot_ref_to_cur, last_.record.rot_ref_to_cur + 9, R.begin());
        return R;
    }
    std::array<double, 3> translation_ref_to_cur() const {
        return {last_.record.trans_ref_to_cur[0], last_.record.trans_ref_to_cur[1], last_.record.trans_ref_to_cur[2]};
    }
    const std::vector<double>& triangulated_pts() const { return last_.triangulated_pts; }
    const std::vector<std::uint8_t>& triangulated_flags() const { return last_.is_triangulated; }
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's getters (bodies in adapters.hpp).
    Mat33_t get_rotation_ref_to_cur() const;
    Vec3_t get_translation_ref_to_cur() const;
    std::vector<Vec3_t> get_triangulated_pts() const;
    std::vector<bool> get_triangulated_flags() const;
    //! initialize(cur_frm, ref_matches_with_cur) on the reference's frame (data::frame in the reference tree; body in adapters.hpp):
    //! reads camera_, undist_keypts_ and bearings_; the sampler seed hashes both views and the matches.  A template deduced from its
    //! argument, so it is compiled only where it is called.
    template <class Frame>
    bool initialize(const Frame& cur_frm, const std::vector<int>& ref_matches_with_cur);
#endif

protected:
    //! The reference's constructor arguments (reproj_err_thr is compared with the squared pixel error, as check_pose does).
    base(const bool perspective, const ovs_init_view* ref, const unsigned int num_ransac_iters, const unsigned int min_num_triangulated,
         const float parallax_deg_thr, const float reproj_err_thr, const int device)
        : perspective_(perspective), ref_(ref), num_ransac_iters_(num_ransac_iters), min_num_triangulated_(min_num_triangulated),
          parallax_deg_thr_(parallax_deg_thr), reproj_err_thr_sq_(reproj_err_thr) {
        detail::check(ovs_matcher_create(device, &h_));
    }

    const bool perspective_;
    const ovs_init_view* ref_;
    // the reference view's own arrays when the object was built from a frame (adapters.hpp)
    ovs_init_view own_ref_{};
    std::vector<double> own_ref_bearings_;
    const unsigned int num_ransac_iters_, min_num_triangulated_;
    const float parallax_deg_thr_, reproj_err_thr_sq_;
    ovs_matcher* h_ = nullptr;
    result last_{};
};

//! initialize::perspective (initialize/perspective.h): perspective cameras, and fisheye ones passed as perspective on their
//! undistorted keypoints.  The homography and fundamental-matrix solvers, the model choice, the decomposition and check_pose.
class perspective : public base {
public:
    perspective(const ovs_init_view& ref, const unsigned int num_ransac_iters = 100, const unsigned int min_num_triangulated = 50,
                const float parallax_deg_thr = 1.0f, const float reproj_err_thr = 4.0f, const int device = 0)
        : base(true, &ref, num_ransac_iters, min_num_triangulated, parallax_deg_thr, reproj_err_thr, device) {}
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    //! The reference's constructor on its frame (body in adapters.hpp).
    template <class Frame>
    perspective(const Frame& ref_frm, const unsigned int num_ransac_iters, const unsigned int min_num_triangulated,
                const float parallax_deg_thr, const float reproj_err_thr, const int device = 0);
#endif
};

//! initialize::bearing_vector (initialize/bearing_vector.h): equirectangular cameras; the essential solver, 4 hypotheses, no depth
//! test.
class bearing_vector : public base {
public:
    bearing_vector(const ovs_init_view& ref, const unsigned int num_ransac_iters = 100, const unsigned int min_num_triangulated = 50,
                   const float parallax_deg_thr = 1.0f, const float reproj_err_thr = 4.0f, const int device = 0)
        : base(false, &ref, num_ransac_iters, min_num_triangulated, parallax_deg_thr, reproj_err_thr, device) {}
#ifdef OVS_B200_WITH_REFERENCE_TYPES
    template <class Frame>
    bearing_vector(const Frame& ref_frm, const unsigned int num_ransac_iters, const unsigned int min_num_triangulated,
                   const float parallax_deg_thr, const float reproj_err_thr, const int device = 0);
#endif
};

}  // namespace initialize
}  // namespace openvslam
