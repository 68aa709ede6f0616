// adapters.hpp -- the reference's own method signatures on the reference's own data model, implemented over the class layer
// of openvslam_b200.hpp (which works on array views).  This is the binding a maintainer adds to the reference tree:
//
//   feature::orb_extractor::extract(const cv::_InputArray&, const cv::_InputArray&, std::vector<cv::KeyPoint>&, const cv::_OutputArray&)
//   util::stereo_rectifier(camera, StereoRectifier block) and rectify(const cv::Mat&, const cv::Mat&, cv::Mat&, cv::Mat&) const
//     (util/stereo_rectifier.h; the config / YAML parsing stays with the caller, which passes stereo_rectifier::params)
//   match::robust::brute_force_match(data::frame&, data::keyframe*, std::vector<std::pair<int, int>>&)           (match/robust.h)
//   match::projection::match_frame_and_landmarks(data::frame&, const std::vector<data::landmark*>&, float)      (match/projection.h)
//   optimize::pose_optimizer::optimize(data::frame&)                                                             (optimize/pose_optimizer.h)
//   optimize::local_bundle_adjuster::optimize(data::keyframe*, bool* const)                                      (optimize/local_bundle_adjuster.h)
//   solve::sim3_solver(data::keyframe*, data::keyframe*, const std::vector<data::landmark*>&, bool, unsigned),
//     find_via_ransac(unsigned), solution_is_valid(), get_best_{rotation,translation,scale}_12()                 (solve/sim3_solver.h)
//   solve::pnp_solver(const eigen_alloc_vector<bearing_t>&, const std::vector<cv::KeyPoint>&, const eigen_alloc_vector<Vec3_t>&,
//     const std::vector<float>&, unsigned), find_via_ransac(unsigned, bool), solution_is_valid(), get_best_{rotation,translation,
//     cam_pose}(), get_inlier_flags()                                                                            (solve/pnp_solver.h)
//   solve::essential_solver(const eigen_alloc_vector<bearing_t>&, const eigen_alloc_vector<bearing_t>&,
//     const std::vector<std::pair<int, int>>&), find_via_ransac(unsigned, bool), solution_is_valid(), get_best_E_21(),
//     get_inlier_matches()                                                                                       (solve/essential_solver.h)
//   match::robust::match_frame_and_keyframe(data::frame&, data::keyframe*, std::vector<data::landmark*>&)       (match/robust.h)
//   solve::homography_solver / solve::fundamental_solver(const std::vector<cv::KeyPoint>&, const std::vector<cv::KeyPoint>&,
//     const std::vector<std::pair<int, int>>&, float), find_via_ransac(unsigned, bool), solution_is_valid(), get_best_score(),
//     get_best_H_21() / get_best_F_21(), get_inlier_matches()                    (solve/{homography,fundamental}_solver.h)
//   the compute step of mapping_module::create_new_landmarks over data::keyframe (module/mapping_module.cc): match_for_triangulation
//     and two_view_triangulator::triangulate for every neighbour, as module::two_view_triangulator::create_new_landmarks
//   initialize::perspective / initialize::bearing_vector(const data::frame&, unsigned, unsigned, float, float),
//     initialize(const data::frame&, const std::vector<int>&), get_{rotation,translation}_ref_to_cur(),
//     get_triangulated_{pts,flags}()                                                           (initialize/{perspective,bearing_vector}.h)
//   match::projection::match_current_and_last_frames(data::frame&, const data::frame&, float)                   (match/projection.h)
//   the body of tracking_module::search_local_landmarks over data::frame and data::landmark, as adapters::search_local_landmarks
//     (both templates deduced from their arguments; tests/cpp/test_tracking_search.cpp runs them on the GPU)
//   match::fuse::replace_duplication(data::keyframe*, const T&, float)                                          (match/fuse.h)
//   the body of mapping_module::fuse_landmark_duplication (module/mapping_module.cc), as adapters::fuse_landmark_duplication
//     (both templates deduced from their arguments; tests/cpp/test_fuse.cpp runs them on the GPU)
//
// Include it INSTEAD of openvslam_b200.hpp in a translation unit that can see the reference's headers (here: the stand-ins
// under tests/cpp/standin, which declare the members used below with the names recalled in SURVEY.md section 2 / 8b;
// /root/reference holds no source, so no file:line can be cited).  tests/test_class_layer.py compiles this file with g++ and
// runs one call of each method on the GPU (tests/cpp/test_adapters.cpp).
#pragma once

#ifndef OVS_B200_WITH_REFERENCE_TYPES
#define OVS_B200_WITH_REFERENCE_TYPES
#endif
#ifndef OVS_B200_WITH_OPENCV
#define OVS_B200_WITH_OPENCV
#endif

#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <type_traits>
#include <unordered_set>
#include <utility>
#include <vector>

#include <opencv2/core.hpp>
#include "openvslam/camera/base.h"
#include "openvslam/data/frame.h"
#include "openvslam/data/keyframe.h"
#include "openvslam/data/landmark.h"
#include "openvslam/type.h"

#include "openvslam_b200.hpp"

namespace openvslam {
namespace adapters {

//! camera::base -> the parameters the reprojection edges read.  Fisheye / radial-division cameras optimise on undistorted
//! keypoints with the perspective edges, as in the reference.
inline ovs_camera to_camera(const camera::base* cam) {
    ovs_camera c{};
    c.focal_x_baseline = cam->focal_x_baseline_; c.cols = cam->cols_; c.rows = cam->rows_;
    switch (cam->model_type_) {
        case camera::model_type_t::Perspective: {
            auto p = static_cast<const camera::perspective*>(cam);
            c.model = OVS_CAMERA_PERSPECTIVE; c.fx = p->fx_; c.fy = p->fy_; c.cx = p->cx_; c.cy = p->cy_; break;
        }
        case camera::model_type_t::Fisheye: {
            auto p = static_cast<const camera::fisheye*>(cam);
            c.model = OVS_CAMERA_PERSPECTIVE; c.fx = p->fx_; c.fy = p->fy_; c.cx = p->cx_; c.cy = p->cy_; break;
        }
        case camera::model_type_t::RadialDivision: {
            auto p = static_cast<const camera::radial_division*>(cam);
            c.model = OVS_CAMERA_PERSPECTIVE; c.fx = p->fx_; c.fy = p->fy_; c.cx = p->cx_; c.cy = p->cy_; break;
        }
        case camera::model_type_t::Equirectangular: c.model = OVS_CAMERA_EQUIRECTANGULAR; break;
    }
    return c;
}

inline void to_Rt(const Mat44_t& T, double* pose12) {
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) pose12[3 * r + c] = T(r, c); pose12[9 + r] = T(r, 3); }
}
inline Mat44_t from_Rt(const double* pose12) {
    Mat44_t T = Mat44_t::Identity();
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) T(r, c) = pose12[3 * r + c]; T(r, 3) = pose12[9 + r]; }
    return T;
}

//! undist_keypts_ / stereo_x_right_ / descriptors_ + the camera's grid constants as a match::frame_view (owns the SoA copies)
struct frame_arrays {
    std::vector<float> x, y, angle, x_right;
    std::vector<std::int32_t> octave;
    std::vector<std::uint8_t> desc;
    match::frame_view view;
    template <class FrameLike>
    explicit frame_arrays(const FrameLike& f) {
        const std::size_t n = f.undist_keypts_.size();
        x.resize(n); y.resize(n); angle.resize(n); octave.resize(n);
        for (std::size_t i = 0; i < n; ++i) {
            const cv::KeyPoint& k = f.undist_keypts_[i];
            x[i] = k.pt.x; y[i] = k.pt.y; angle[i] = k.angle; octave[i] = k.octave;
        }
        x_right.assign(f.stereo_x_right_.begin(), f.stereo_x_right_.end());
        desc.resize(n * 32);
        for (std::size_t i = 0; i < n; ++i) std::memcpy(&desc[32 * i], f.descriptors_.ptr(static_cast<int>(i)), 32);   // rows may be strided
        view.num_keypts = static_cast<int>(n);
        view.x = x.data(); view.y = y.data(); view.octave = octave.data(); view.angle = angle.data();
        view.stereo_x_right = (x_right.size() == n && n > 0) ? x_right.data() : nullptr;
        view.descriptors = desc.data();
        const camera::base* cam = f.camera_;
        view.grid.min_x = cam->img_bounds_.min_x_; view.grid.min_y = cam->img_bounds_.min_y_;
        view.grid.inv_cell_width = cam->inv_cell_width_; view.grid.inv_cell_height = cam->inv_cell_height_;
        view.grid.num_grid_cols = static_cast<std::int32_t>(cam->num_grid_cols_); view.grid.num_grid_rows = static_cast<std::int32_t>(cam->num_grid_rows_);
    }
};

//! The sampler seed of a solver built with the reference's constructor: a splitmix64 hash of the input bits (8-byte words, the
//! last one zero-padded), so the same input always gives the same solution.
struct input_hash {
    std::uint64_t seed;
    explicit input_hash(const std::size_t n) : seed(0x9E3779B97F4A7C15ull ^ static_cast<std::uint64_t>(n)) {}
    void add(const void* p, const std::size_t bytes) {
        const unsigned char* c = static_cast<const unsigned char*>(p);
        for (std::size_t k = 0; k < bytes; k += 8) {
            std::uint64_t w = 0;
            std::memcpy(&w, c + k, std::min<std::size_t>(8, bytes - k));
            std::uint64_t z = seed + w + 0x9E3779B97F4A7C15ull;   // splitmix64's output function over the running state
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
            z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
            seed = z ^ (z >> 31);
        }
    }
};

//! bearings_ of a frame or keyframe as 3 doubles per keypoint
template <class BearingVector>
std::vector<double> flat_bearings(const BearingVector& bearings) {
    std::vector<double> out(3 * bearings.size());
    for (std::size_t i = 0; i < bearings.size(); ++i)
        for (int k = 0; k < 3; ++k) out[3 * i + k] = bearings[i](k);
    return out;
}

}  // namespace adapters

// ---------------------------------------------------------------------------------------------------- match::robust
inline unsigned int match::robust::brute_force_match(data::frame& frm, data::keyframe* keyfrm, std::vector<std::pair<int, int>>& matches) const {
    const auto lms_2 = keyfrm->get_landmarks();
    const int n1 = static_cast<int>(frm.num_keypts_), n2 = static_cast<int>(keyfrm->num_keypts_);
    std::vector<std::uint8_t> valid(static_cast<std::size_t>(std::max(n2, 1)), 0);
    for (int i = 0; i < n2 && i < static_cast<int>(lms_2.size()); ++i) valid[i] = lms_2[i] && !lms_2[i]->will_be_erased();
    std::vector<std::uint8_t> d1(static_cast<std::size_t>(n1) * 32), d2(static_cast<std::size_t>(n2) * 32);
    for (int i = 0; i < n1; ++i) std::memcpy(&d1[32 * static_cast<std::size_t>(i)], frm.descriptors_.ptr(i), 32);
    for (int i = 0; i < n2; ++i) std::memcpy(&d2[32 * static_cast<std::size_t>(i)], keyfrm->descriptors_.ptr(i), 32);
    return brute_force_match(d1.data(), n1, d2.data(), n2, valid.data(), matches);
}

// match_frame_and_keyframe: the brute force over the same arrays as brute_force_match, the essential-matrix RANSAC on the pairs
// (find_via_ransac(50, false)), and matched_lms_in_frm[idx_1] = keyfrm->get_landmarks()[idx_2] for each inlier pair of a valid
// solution.  The sampler seed hashes both bearing sets.  Frame / Keyframe are data::frame / data::keyframe in the reference tree.
template <class Frame, class Keyframe>
inline unsigned int match::robust::match_frame_and_keyframe(Frame& frm, Keyframe* keyfrm,
                                                            std::vector<data::landmark*>& matched_lms_in_frm) const {
    const auto lms_2 = keyfrm->get_landmarks();
    const int n1 = static_cast<int>(frm.num_keypts_), n2 = static_cast<int>(keyfrm->num_keypts_);
    std::vector<std::uint8_t> valid(static_cast<std::size_t>(std::max(n2, 1)), 0);
    for (int i = 0; i < n2 && i < static_cast<int>(lms_2.size()); ++i) valid[i] = lms_2[i] && !lms_2[i]->will_be_erased();
    std::vector<std::uint8_t> d1(static_cast<std::size_t>(n1) * 32), d2(static_cast<std::size_t>(n2) * 32);
    for (int i = 0; i < n1; ++i) std::memcpy(&d1[32 * static_cast<std::size_t>(i)], frm.descriptors_.ptr(i), 32);
    for (int i = 0; i < n2; ++i) std::memcpy(&d2[32 * static_cast<std::size_t>(i)], keyfrm->descriptors_.ptr(i), 32);
    const std::vector<double> b1 = adapters::flat_bearings(frm.bearings_), b2 = adapters::flat_bearings(keyfrm->bearings_);
    adapters::input_hash hash(b1.size() + b2.size());
    hash.add(b1.data(), 8 * b1.size());
    hash.add(b2.data(), 8 * b2.size());
    std::vector<int> idx_2;
    const unsigned int num = match_frame_and_keyframe(d1.data(), b1.data(), n1, d2.data(), b2.data(), n2, valid.data(), idx_2, 50, hash.seed);
    matched_lms_in_frm.assign(static_cast<std::size_t>(n1), nullptr);
    for (int i = 0; i < n1; ++i)
        if (idx_2[i] >= 0) matched_lms_in_frm[i] = lms_2.at(static_cast<std::size_t>(idx_2[i]));
    return num;
}

// ------------------------------------------------------------------------------------------------ match::projection
inline unsigned int match::projection::match_frame_and_landmarks(data::frame& frm, const std::vector<data::landmark*>& local_landmarks,
                                                                 const float margin) const {
    const adapters::frame_arrays arrays(frm);
    const frame_index idx(*this, arrays.view);               // upload + cell index (reusable by every matcher call on this frame)
    const std::size_t L = local_landmarks.size();
    const unsigned int n = frm.num_keypts_;
    std::vector<std::uint8_t> usable(std::max<std::size_t>(L, 1), 0), has(std::max<unsigned int>(n, 1), 0), desc(32 * std::max<std::size_t>(L, 1));
    std::vector<float> reproj(2 * std::max<std::size_t>(L, 1)), xr(std::max<std::size_t>(L, 1));
    std::vector<std::int32_t> lvl(std::max<std::size_t>(L, 1), 0);
    for (std::size_t l = 0; l < L; ++l) {
        const data::landmark* lm = local_landmarks[l];
        usable[l] = lm && lm->is_observable_in_tracking_ && !lm->will_be_erased();
        if (!usable[l]) continue;
        reproj[2 * l] = static_cast<float>(lm->reproj_in_tracking_(0)); reproj[2 * l + 1] = static_cast<float>(lm->reproj_in_tracking_(1));
        xr[l] = lm->x_right_in_tracking_; lvl[l] = lm->scale_level_in_tracking_;
        const cv::Mat d = lm->get_descriptor();
        std::memcpy(&desc[32 * l], d.data, 32);
    }
    for (unsigned int i = 0; i < n; ++i) has[i] = frm.landmarks_.at(i) && frm.landmarks_.at(i)->has_observation();
    std::vector<std::int32_t> matched;
    const unsigned int num = match_frame_and_landmarks(idx, frm.scale_factors_, static_cast<int>(L), usable.data(), reproj.data(), xr.data(), lvl.data(),
                                                       desc.data(), has.data(), matched, margin);
    for (unsigned int i = 0; i < n; ++i) if (matched[i] >= 0) frm.landmarks_.at(i) = local_landmarks[static_cast<std::size_t>(matched[i])];
    return num;
}

namespace adapters {

// The tracking adapters below are templates deduced from their arguments (data::frame / data::landmark in the reference tree), as
// match::robust::match_frame_and_keyframe is: their bodies are compiled only where they are called, so a data model without the
// members they read (here: the landmark's unscaled valid distances, INTEGRATION.md) can use the other adapters.

//! What frame::can_observe and the motion model read of a frame: camera_ (fisheye and radial division reproject with the pinhole
//! formula on undistorted keypoints), camera_->img_bounds_, cam_pose_cw_, get_cam_center(), num_scale_levels_, log_scale_factor_.
template <class Frame>
ovs_frame_geometry frame_geometry(const Frame& frm) {
    ovs_frame_geometry g{};
    g.camera = to_camera(frm.camera_);
    const camera::image_bounds& b = frm.camera_->img_bounds_;
    g.min_x = b.min_x_; g.max_x = b.max_x_; g.min_y = b.min_y_; g.max_y = b.max_y_;
    double pose12[12];
    to_Rt(frm.cam_pose_cw_, pose12);
    for (int k = 0; k < 9; ++k) g.rot_cw[k] = pose12[k];
    for (int k = 0; k < 3; ++k) g.trans_cw[k] = pose12[9 + k];
    const Vec3_t c = frm.get_cam_center();
    for (int k = 0; k < 3; ++k) g.cam_center[k] = c(k);
    g.num_scale_levels = static_cast<std::int32_t>(frm.num_scale_levels_);
    g.log_scale_factor = frm.log_scale_factor_;
    return g;
}

//! kp_has_observed_lm of a frame: frm.landmarks_[i] present and has_observation()
template <class Frame>
std::vector<std::uint8_t> keypoints_with_observed_landmarks(const Frame& frm) {
    const unsigned int n = frm.num_keypts_;
    std::vector<std::uint8_t> has(std::max<unsigned int>(n, 1), 0);
    for (unsigned int i = 0; i < n; ++i) has[i] = frm.landmarks_.at(i) && frm.landmarks_.at(i)->has_observation();
    return has;
}

//! The body of tracking_module::search_local_landmarks (module/tracking_module.cc) with frame::can_observe on the device: the
//! frame's own landmarks are marked (is_observable_in_tracking_ = false, identifier_in_local_lm_search_ = curr_frm.id_,
//! increase_num_observable()); every other local landmark that is not will_be_erased() goes through can_observe(lm, 0.5) and,
//! when observable, gets reproj_in_tracking_, x_right_in_tracking_, scale_level_in_tracking_, is_observable_in_tracking_ = true and
//! increase_num_observable(), else is_observable_in_tracking_ = false; the observable ones are matched into curr_frm.landmarks_
//! by the matcher's match_frame_and_landmarks(curr_frm, local_landmarks, margin).  Returns found_proj_candidate.  The caller picks
//! the margin as the reference does (20 right after a relocalisation, 10 RGBD, 5 otherwise).
template <class Frame, class Landmark>
bool search_local_landmarks(const match::projection& matcher, Frame& curr_frm, const std::vector<Landmark*>& local_landmarks, const float margin) {
    for (Landmark* lm : curr_frm.landmarks_) {
        if (!lm || lm->will_be_erased()) continue;
        lm->is_observable_in_tracking_ = false;
        lm->identifier_in_local_lm_search_ = curr_frm.id_;
        lm->increase_num_observable();
    }
    const std::size_t L = local_landmarks.size(), L1 = std::max<std::size_t>(L, 1);
    std::vector<std::uint8_t> usable(L1, 0), desc(32 * L1), observable(L1, 0);
    std::vector<double> pos(3 * L1, 0.0), nrm(3 * L1, 0.0);
    std::vector<float> lo(L1, 0.0f), hi(L1, 0.0f), reproj(2 * L1), xr(L1);
    std::vector<std::int32_t> lvl(L1);
    for (std::size_t l = 0; l < L; ++l) {
        const Landmark* lm = local_landmarks[l];
        usable[l] = lm && lm->identifier_in_local_lm_search_ != curr_frm.id_ && !lm->will_be_erased();
        if (!usable[l]) continue;
        const Vec3_t p = lm->get_pos_in_world(), n = lm->get_obs_mean_normal();
        for (int k = 0; k < 3; ++k) { pos[3 * l + k] = p(k); nrm[3 * l + k] = n(k); }
        const std::pair<float, float> d = lm->get_unscaled_valid_distances();
        lo[l] = d.first; hi[l] = d.second;
        const cv::Mat dsc = lm->get_descriptor();
        std::memcpy(&desc[32 * l], dsc.data, 32);
    }
    const frame_arrays arrays(curr_frm);
    const match::frame_index idx(matcher, arrays.view);
    const std::vector<std::uint8_t> has = keypoints_with_observed_landmarks(curr_frm);
    std::vector<std::int32_t> matched;
    matcher.search_local_landmarks(idx, frame_geometry(curr_frm), curr_frm.scale_factors_, static_cast<int>(L), usable.data(), pos.data(), nrm.data(),
                                   lo.data(), hi.data(), desc.data(), has.data(), observable.data(), reproj.data(), xr.data(), lvl.data(), matched,
                                   margin, 0.5f);
    bool found_proj_candidate = false;
    for (std::size_t l = 0; l < L; ++l) {
        if (!usable[l]) continue;
        Landmark* lm = local_landmarks[l];
        lm->is_observable_in_tracking_ = observable[l] != 0;
        if (!observable[l]) continue;
        lm->reproj_in_tracking_(0) = reproj[2 * l]; lm->reproj_in_tracking_(1) = reproj[2 * l + 1];
        lm->x_right_in_tracking_ = xr[l];
        lm->scale_level_in_tracking_ = lvl[l];
        lm->increase_num_observable();
        found_proj_candidate = true;
    }
    for (unsigned int i = 0; i < curr_frm.num_keypts_; ++i)
        if (matched[i] >= 0) curr_frm.landmarks_.at(i) = local_landmarks[static_cast<std::size_t>(matched[i])];
    return found_proj_candidate;
}

//! The same with the reference's own matcher, match::projection projection_matcher(0.8), made for the call.
template <class Frame, class Landmark>
bool search_local_landmarks(Frame& curr_frm, const std::vector<Landmark*>& local_landmarks, const float margin) {
    const match::projection projection_matcher(0.8);
    return search_local_landmarks(projection_matcher, curr_frm, local_landmarks, margin);
}

}  // namespace adapters

// match_current_and_last_frames: every keypoint of last_frm with a landmark that is not an outlier is reprojected into curr_frm with
// its pose on the device; the direction comes from the two poses and curr_frm.camera_: setup_type_, and true_baseline =
// focal_x_baseline_ / fx_, the value the reference's perspective-family camera constructors store (as create_new_landmarks reads it).
template <class Frame>
inline unsigned int match::projection::match_current_and_last_frames(Frame& curr_frm, const Frame& last_frm, const float margin) const {
    const unsigned int n_last = last_frm.num_keypts_, N1 = std::max<unsigned int>(n_last, 1);
    std::vector<std::uint8_t> usable(N1, 0), desc(32 * static_cast<std::size_t>(N1));
    std::vector<double> pos(3 * static_cast<std::size_t>(N1), 0.0);
    std::vector<std::int32_t> octave(N1, 0);
    std::vector<float> angle(N1, 0.0f);
    for (unsigned int i = 0; i < n_last; ++i) {
        const auto* lm = last_frm.landmarks_.at(i);
        usable[i] = lm && !last_frm.outlier_flags_.at(i);
        octave[i] = last_frm.undist_keypts_.at(i).octave;
        angle[i] = last_frm.undist_keypts_.at(i).angle;
        if (!usable[i]) continue;
        const Vec3_t p = lm->get_pos_in_world();
        for (int k = 0; k < 3; ++k) pos[3 * i + k] = p(k);
        const cv::Mat d = lm->get_descriptor();
        std::memcpy(&desc[32 * static_cast<std::size_t>(i)], d.data, 32);
    }
    const adapters::frame_arrays arrays(curr_frm);
    const frame_index idx(*this, arrays.view);
    const std::vector<std::uint8_t> has = adapters::keypoints_with_observed_landmarks(curr_frm);
    double last_pose[12];
    adapters::to_Rt(last_frm.cam_pose_cw_, last_pose);
    const ovs_frame_geometry geometry = adapters::frame_geometry(curr_frm);
    const double true_baseline = geometry.camera.fx != 0.0 ? geometry.camera.focal_x_baseline / geometry.camera.fx : 0.0;
    std::vector<std::int32_t> matched;
    const unsigned int num = match_current_and_last_frames_reproject(
        idx, geometry, curr_frm.camera_->setup_type_ == camera::setup_type_t::Monocular, true_baseline, last_pose, curr_frm.scale_factors_,
        static_cast<int>(n_last), usable.data(), pos.data(), octave.data(), angle.data(), desc.data(), has.data(), matched, margin);
    for (unsigned int i = 0; i < curr_frm.num_keypts_; ++i)
        if (matched[i] >= 0) curr_frm.landmarks_.at(i) = last_frm.landmarks_.at(static_cast<std::size_t>(matched[i]));
    return num;
}

// ------------------------------------------------------------------------------------------------------- match::fuse
namespace adapters {

// The fuse adapters are templates deduced from their arguments (data::keyframe / data::landmark in the reference tree), like the
// tracking adapters above.
//
// replace_duplication(keyfrm, landmarks_to_check, margin) runs its geometry and search on the device and replays its data-model
// updates on the host, in the container's order, with the reference's live skips (no landmark, will_be_erased(),
// is_observed_in_keyframe(keyfrm)).  That replay is exact with one device call per target because a query's answer depends only on
// the landmark's position, mean normal, valid distances and descriptor and on the target's own arrays, and the only update that
// changes any of these is landmark::replace, through other->compute_descriptor() on the survivor.  Within one target the survivor
// of a replace is either the query's own landmark, which the container does not hold twice, or the landmark already in the
// target's keypoint, which is observed in the target and so skipped by every later query of it.  So no descriptor changes under a
// later query of the same target.  Across targets it can: fuse_landmark_duplication keeps the set of landmarks that survived a
// replace since its snapshot and, before replaying each target, re-queries that target's queries on such landmarks, in one call,
// with their current descriptors.

//! What replace_duplication reads of a keyframe, as an ovs_fuse_target over copies owned here: camera_, img_bounds_,
//! get_cam_pose(), get_cam_center(), num_scale_levels_, log_scale_factor_, scale_factors_, inv_level_sigma_sq_, undist_keypts_,
//! stereo_x_right_, descriptors_ and the camera's grid.
struct fuse_target_arrays {
    frame_arrays arrays;
    ovs_fuse_target target{};
    template <class Keyframe>
    explicit fuse_target_arrays(const Keyframe& keyfrm) : arrays(keyfrm) {
        ovs_frame_geometry& g = target.geometry;
        g.camera = to_camera(keyfrm.camera_);
        const camera::image_bounds& b = keyfrm.camera_->img_bounds_;
        g.min_x = b.min_x_; g.max_x = b.max_x_; g.min_y = b.min_y_; g.max_y = b.max_y_;
        double pose12[12];
        to_Rt(keyfrm.get_cam_pose(), pose12);
        for (int k = 0; k < 9; ++k) g.rot_cw[k] = pose12[k];
        for (int k = 0; k < 3; ++k) g.trans_cw[k] = pose12[9 + k];
        const Vec3_t c = keyfrm.get_cam_center();
        for (int k = 0; k < 3; ++k) g.cam_center[k] = c(k);
        g.num_scale_levels = static_cast<std::int32_t>(keyfrm.num_scale_levels_);
        g.log_scale_factor = keyfrm.log_scale_factor_;
        target.scale_factors = keyfrm.scale_factors_.data();
        target.inv_level_sigma_sq = keyfrm.inv_level_sigma_sq_.data();
        const match::frame_view& v = arrays.view;
        target.num_keypts = v.num_keypts; target.x = v.x; target.y = v.y; target.octave = v.octave; target.x_right = v.stereo_x_right;
        target.descriptors = v.descriptors; target.grid = v.grid;
    }
};

//! The landmark table of a fuse call: one row per landmark added, read through get_pos_in_world(), get_obs_mean_normal(),
//! get_unscaled_valid_distances() and get_descriptor().
template <class Landmark>
struct fuse_landmark_rows {
    std::vector<Landmark*> lms;
    std::vector<double> pos, nrm;
    std::vector<float> lo, hi;
    std::vector<std::uint8_t> desc;
    int add(Landmark* lm) {
        const Vec3_t p = lm->get_pos_in_world(), n = lm->get_obs_mean_normal();
        for (int k = 0; k < 3; ++k) { pos.push_back(p(k)); nrm.push_back(n(k)); }
        const std::pair<float, float> d = lm->get_unscaled_valid_distances();
        lo.push_back(d.first); hi.push_back(d.second);
        desc.resize(desc.size() + 32);
        lms.push_back(lm);
        refresh_descriptor(static_cast<int>(lms.size()) - 1);
        return static_cast<int>(lms.size()) - 1;
    }
    void refresh_descriptor(const int row) {
        const cv::Mat d = lms[static_cast<std::size_t>(row)]->get_descriptor();
        std::memcpy(&desc[32 * static_cast<std::size_t>(row)], d.data, 32);
    }
    match::fuse::landmark_table table() const {
        match::fuse::landmark_table t;
        t.num_landmarks = static_cast<int>(lms.size());
        t.pos_w = pos.data(); t.mean_normal = nrm.data(); t.min_valid_dist = lo.data(); t.max_valid_dist = hi.data(); t.descriptors = desc.data();
        return t;
    }
};

//! The reference's update for one query of replace_duplication that found best_idx in keyfrm; a replace's survivor goes into
//! `changed` (its descriptor was recomputed).
template <class Keyframe, class Landmark>
void fuse_into_keyframe(Keyframe* keyfrm, Landmark* lm, const int best_idx, std::unordered_set<Landmark*>& changed) {
    auto* lm_in_keyfrm = keyfrm->get_landmark(static_cast<unsigned int>(best_idx));
    if (lm_in_keyfrm) {
        if (!lm_in_keyfrm->will_be_erased()) {
            if (lm->num_observations() < lm_in_keyfrm->num_observations()) {
                lm->replace(lm_in_keyfrm);
                changed.insert(lm_in_keyfrm);
            } else {
                lm_in_keyfrm->replace(lm);
                changed.insert(lm);
            }
        }
    } else {
        lm->add_observation(keyfrm, static_cast<unsigned int>(best_idx));
        keyfrm->add_landmark(lm, static_cast<unsigned int>(best_idx));
    }
}

template <class Keyframe, class Landmark>
bool fuse_skips(Keyframe* keyfrm, const Landmark* lm) {
    return !lm || lm->will_be_erased() || lm->is_observed_in_keyframe(keyfrm);
}

}  // namespace adapters

// replace_duplication: one device call over the landmarks that are usable now, then the reference's loop over the container.
template <class Keyframe, class T>
inline unsigned int match::fuse::replace_duplication(Keyframe* keyfrm, const T& landmarks_to_check, const float margin) const {
    using Landmark = std::remove_pointer_t<typename T::value_type>;
    adapters::fuse_landmark_rows<Landmark> rows;
    std::vector<std::int32_t> q_lm;
    for (Landmark* lm : landmarks_to_check) q_lm.push_back(adapters::fuse_skips(keyfrm, lm) ? -1 : rows.add(lm));
    const adapters::fuse_target_arrays tgt(*keyfrm);   // owns the arrays tgt.target points at
    const std::vector<ovs_fuse_target> targets(1, tgt.target);
    std::vector<std::int32_t> best;
    replace_duplication(targets, rows.table(), {0, static_cast<std::int32_t>(q_lm.size())}, q_lm, margin, best);
    unsigned int num_fused = 0;
    std::unordered_set<Landmark*> changed;
    std::size_t q = 0;
    for (Landmark* lm : landmarks_to_check) {
        const int best_idx = best[q++];
        if (adapters::fuse_skips(keyfrm, lm) || best_idx < 0) continue;
        adapters::fuse_into_keyframe(keyfrm, lm, best_idx, changed);
        ++num_fused;
    }
    return num_fused;
}

namespace adapters {

//! The body of mapping_module::fuse_landmark_duplication(fuse_tgt_keyfrms) (module/mapping_module.cc) with the reference's
//! replace_duplication(keyfrm, landmarks, margin):
//!   - forward: cur_keyfrm->get_landmarks() into every target, in the container's order: one device call for all targets, then
//!     the replay target by target, each preceded by one re-query call if some of its queries are on landmarks that survived a
//!     replace since the call (their descriptors changed);
//!   - backward: every non-null, non-erased landmark of every target, gathered target by target into a
//!     std::unordered_set<Landmark*> as the reference does, into cur_keyfrm: replace_duplication above.
//! Host waits: 2 + the number of targets with re-queries (fuse.num_requery_calls()).
template <class Keyframe, class Targets>
void fuse_landmark_duplication(const match::fuse& fuse, Keyframe* cur_keyfrm, const Targets& fuse_tgt_keyfrms, const float margin = 3.0) {
    using Landmark = std::remove_pointer_t<typename decltype(cur_keyfrm->get_landmarks())::value_type>;
    const auto cur_landmarks = cur_keyfrm->get_landmarks();
    {
        std::vector<Keyframe*> tgts;
        std::vector<fuse_target_arrays> arrays;
        for (Keyframe* t : fuse_tgt_keyfrms) tgts.push_back(t);
        arrays.reserve(tgts.size());   // no reallocation: targets[] points into these
        std::vector<ovs_fuse_target> targets;
        for (Keyframe* t : tgts) { arrays.emplace_back(*t); targets.push_back(arrays.back().target); }
        const std::size_t J = cur_landmarks.size();
        fuse_landmark_rows<Landmark> rows;
        std::vector<std::int32_t> row_of(J, -1);
        for (std::size_t j = 0; j < J; ++j)
            if (cur_landmarks[j] && !cur_landmarks[j]->will_be_erased()) row_of[j] = rows.add(cur_landmarks[j]);
        std::vector<std::int32_t> q_off(1, 0), q_lm;
        for (Keyframe* t : tgts) {
            for (std::size_t j = 0; j < J; ++j) q_lm.push_back(row_of[j] >= 0 && !cur_landmarks[j]->is_observed_in_keyframe(t) ? row_of[j] : -1);
            q_off.push_back(static_cast<std::int32_t>(q_lm.size()));
        }
        std::vector<std::int32_t> best;
        fuse.replace_duplication(targets, rows.table(), q_off, q_lm, margin, best);
        std::unordered_set<Landmark*> changed;
        for (std::size_t t = 0; t < tgts.size(); ++t) {
            Keyframe* tgt = tgts[t];
            const std::size_t q0 = static_cast<std::size_t>(q_off[t]);
            // the queries of this target on landmarks whose descriptor changed since the call, again with the current descriptors
            std::vector<std::int32_t> rq_lm;
            std::vector<std::size_t> rq;
            for (std::size_t j = 0; j < J; ++j) {
                Landmark* lm = cur_landmarks[j];
                if (q_lm[q0 + j] < 0 || !changed.count(lm) || fuse_skips(tgt, lm)) continue;
                rows.refresh_descriptor(row_of[j]);
                rq_lm.push_back(row_of[j]); rq.push_back(q0 + j);
            }
            if (!rq.empty()) {
                std::vector<std::int32_t> rbest;
                fuse.count_requery_call();
                fuse.replace_duplication(std::vector<ovs_fuse_target>(1, targets[t]), rows.table(), {0, static_cast<std::int32_t>(rq_lm.size())}, rq_lm,
                                         margin, rbest);
                for (std::size_t k = 0; k < rq.size(); ++k) best[rq[k]] = rbest[k];
            }
            for (std::size_t j = 0; j < J; ++j) {
                Landmark* lm = cur_landmarks[j];
                const int best_idx = best[q0 + j];
                if (q_lm[q0 + j] < 0 || fuse_skips(tgt, lm) || best_idx < 0) continue;
                fuse_into_keyframe(tgt, lm, best_idx, changed);
            }
        }
    }
    std::unordered_set<Landmark*> candidates_to_fuse;
    for (Keyframe* t : fuse_tgt_keyfrms)
        for (Landmark* lm : t->get_landmarks()) {
            if (!lm || lm->will_be_erased()) continue;
            candidates_to_fuse.insert(lm);
        }
    fuse.replace_duplication(cur_keyfrm, candidates_to_fuse, margin);
}

//! The same with a matcher made for the call, as the reference's match::fuse fuse(0.6).
template <class Keyframe, class Targets>
void fuse_landmark_duplication(Keyframe* cur_keyfrm, const Targets& fuse_tgt_keyfrms, const float margin = 3.0) {
    const match::fuse fuse(0.6);
    fuse_landmark_duplication(fuse, cur_keyfrm, fuse_tgt_keyfrms, margin);
}

}  // namespace adapters

// --------------------------------------------------------------------------------------------- optimize::pose_optimizer
inline unsigned int optimize::pose_optimizer::optimize(data::frame& frm) const {
    // one edge per keypoint with a valid landmark (the reference's loop over frm.landmarks_)
    std::vector<unsigned int> idxs;
    std::vector<double> pos_w; std::vector<float> xy, x_right, inv_sigma_sq;
    const unsigned int num_keypts = frm.num_keypts_;
    for (unsigned int idx = 0; idx < num_keypts; ++idx) {
        data::landmark* lm = frm.landmarks_.at(idx);
        if (!lm) continue;
        if (lm->will_be_erased()) continue;
        frm.outlier_flags_.at(idx) = false;
        const cv::KeyPoint& undist_keypt = frm.undist_keypts_.at(idx);
        const Vec3_t p = lm->get_pos_in_world();
        idxs.push_back(idx);
        pos_w.push_back(p(0)); pos_w.push_back(p(1)); pos_w.push_back(p(2));
        xy.push_back(undist_keypt.pt.x); xy.push_back(undist_keypt.pt.y);
        x_right.push_back(idx < frm.stereo_x_right_.size() ? frm.stereo_x_right_.at(idx) : -1.0f);
        inv_sigma_sq.push_back(frm.inv_level_sigma_sq_.at(static_cast<std::size_t>(undist_keypt.octave)));
    }
    const int num_init_obs = static_cast<int>(idxs.size());
    if (num_init_obs < 5) return 0;
    double pose[12];
    adapters::to_Rt(frm.cam_pose_cw_, pose);
    const ovs_camera cam = adapters::to_camera(frm.camera_);
    std::vector<std::uint8_t> outlier;
    const unsigned int num_inliers = optimize(cam, frm.camera_->setup_type_ == camera::setup_type_t::Monocular, num_init_obs, pos_w.data(), xy.data(),
                                              x_right.data(), inv_sigma_sq.data(), pose, outlier);
    for (int k = 0; k < num_init_obs; ++k) frm.outlier_flags_.at(idxs[static_cast<std::size_t>(k)]) = outlier[static_cast<std::size_t>(k)] != 0;
    frm.set_cam_pose(adapters::from_Rt(pose));
    return num_inliers;
}

// ------------------------------------------------------------------------------------- optimize::local_bundle_adjuster
inline void optimize::local_bundle_adjuster::optimize(data::keyframe* curr_keyfrm, bool* const force_stop_flag) const {
    // 1. local keyframes (the current one and its covisibilities), local landmarks (seen by them), fixed keyframes (other observers
    //    of the local landmarks).  The reference collects them in unordered_maps keyed by id; ordered maps here, so that vertex and
    //    edge order -- and with it the rounding of the sums -- is reproducible.
    std::map<unsigned int, data::keyframe*> local_keyfrms, fixed_keyfrms;
    std::map<unsigned int, data::landmark*> local_lms;
    local_keyfrms[curr_keyfrm->id_] = curr_keyfrm;
    for (data::keyframe* k : curr_keyfrm->graph_node_->get_covisibilities()) {
        if (!k || k->will_be_erased()) continue;
        local_keyfrms[k->id_] = k;
    }
    for (const auto& id_kf : local_keyfrms)
        for (data::landmark* lm : id_kf.second->get_landmarks()) {
            if (!lm || lm->will_be_erased()) continue;
            local_lms[lm->id_] = lm;
        }
    for (const auto& id_lm : local_lms)
        for (const auto& obs : id_lm.second->get_observations()) {
            data::keyframe* k = obs.first;
            if (!k || k->will_be_erased()) continue;
            if (local_keyfrms.count(k->id_)) continue;
            fixed_keyfrms[k->id_] = k;
        }
    if (local_lms.empty()) return;
    // 2. the graph as arrays: keyframe vertices (local ones free, keyframe id 0 and the fixed ones fixed), landmark vertices,
    //    one edge per observation, landmark by landmark
    std::vector<data::keyframe*> kfs; std::map<data::keyframe*, int> kf_index;
    std::vector<std::uint8_t> is_fixed;
    for (const auto& id_kf : local_keyfrms) { kf_index[id_kf.second] = static_cast<int>(kfs.size()); kfs.push_back(id_kf.second); is_fixed.push_back(id_kf.first == 0); }
    for (const auto& id_kf : fixed_keyfrms) { kf_index[id_kf.second] = static_cast<int>(kfs.size()); kfs.push_back(id_kf.second); is_fixed.push_back(1); }
    const int K = static_cast<int>(kfs.size());
    std::vector<double> poses(static_cast<std::size_t>(K) * 12);
    for (int k = 0; k < K; ++k) adapters::to_Rt(kfs[static_cast<std::size_t>(k)]->get_cam_pose(), &poses[static_cast<std::size_t>(k) * 12]);
    std::vector<data::landmark*> lms;
    std::vector<double> points;
    std::vector<std::int32_t> obs_kf, obs_lm; std::vector<float> obs_xy, obs_xr, obs_w;
    std::vector<std::pair<data::keyframe*, data::landmark*>> obs_pairs;
    for (const auto& id_lm : local_lms) {
        data::landmark* lm = id_lm.second;
        const int l = static_cast<int>(lms.size());
        bool any = false;
        // observers in keyframe-id order (std::map<keyframe*, unsigned> iterates by address in the reference)
        std::map<unsigned int, std::pair<data::keyframe*, unsigned int>> by_id;
        for (const auto& obs : lm->get_observations()) if (obs.first && !obs.first->will_be_erased() && kf_index.count(obs.first)) by_id[obs.first->id_] = {obs.first, obs.second};
        for (const auto& e : by_id) {
            data::keyframe* k = e.second.first; const unsigned int idx = e.second.second;
            const cv::KeyPoint& undist_keypt = k->undist_keypts_.at(idx);
            obs_kf.push_back(kf_index[k]); obs_lm.push_back(l);
            obs_xy.push_back(undist_keypt.pt.x); obs_xy.push_back(undist_keypt.pt.y);
            obs_xr.push_back(idx < k->stereo_x_right_.size() ? k->stereo_x_right_.at(idx) : -1.0f);
            obs_w.push_back(k->inv_level_sigma_sq_.at(static_cast<std::size_t>(undist_keypt.octave)));
            obs_pairs.emplace_back(k, lm);
            any = true;
        }
        if (!any) continue;
        lms.push_back(lm);
        const Vec3_t p = lm->get_pos_in_world();
        points.push_back(p(0)); points.push_back(p(1)); points.push_back(p(2));
    }
    const int L = static_cast<int>(lms.size()), M = static_cast<int>(obs_kf.size());
    if (L == 0 || M == 0) return;
    // 3.-7. the two Levenberg rounds with the outlier cut in between (replaces the g2o call)
    const ovs_camera cam = adapters::to_camera(curr_keyfrm->camera_);
    std::vector<std::uint8_t> outlier;
    optimize(cam, curr_keyfrm->camera_->setup_type_ == camera::setup_type_t::Monocular, K, poses.data(), is_fixed.data(), L, points.data(), M,
             obs_kf.data(), obs_lm.data(), obs_xy.data(), obs_xr.data(), obs_w.data(), force_stop_flag, outlier);
    // 8. under the map lock: erase the outlier observations, write the estimates back
    {
        std::lock_guard<std::mutex> lock(data::map_database::mtx_database_);
        for (int i = 0; i < M; ++i) {
            if (!outlier[static_cast<std::size_t>(i)]) continue;
            data::keyframe* k = obs_pairs[static_cast<std::size_t>(i)].first; data::landmark* lm = obs_pairs[static_cast<std::size_t>(i)].second;
            k->erase_landmark(lm);
            lm->erase_observation(k);
        }
        for (int k = 0; k < K; ++k)
            if (!is_fixed[static_cast<std::size_t>(k)] && local_keyfrms.count(kfs[static_cast<std::size_t>(k)]->id_))
                kfs[static_cast<std::size_t>(k)]->set_cam_pose(adapters::from_Rt(&poses[static_cast<std::size_t>(k) * 12]));
        for (int l = 0; l < L; ++l) {
            Vec3_t p; p(0) = points[3 * static_cast<std::size_t>(l)]; p(1) = points[3 * static_cast<std::size_t>(l) + 1]; p(2) = points[3 * static_cast<std::size_t>(l) + 2];
            lms[static_cast<std::size_t>(l)]->set_pos_in_world(p);
            lms[static_cast<std::size_t>(l)]->update_normal_and_depth();
        }
    }
}

// ------------------------------------------------------------------------------------------------ solve::sim3_solver
// The reference's constructor keeps, in keyframe 1's keypoint order, the pairs whose two landmarks exist and are not to be erased
// and whose lm_2 is observed in keyframe 2; each side contributes its landmark's world position and level_sigma_sq_ at the octave
// of its keypoint.  The sampler seed is (keyfrm_1->id_ << 32) | keyfrm_2->id_, so a candidate always gives the same solution.
namespace adapters {
//! level_sigma_sq_[octave] of a keyframe, formed as orb_params::calc_level_sigma_sq defines it: the float square of the level's
//! scale factor (the same bits; ovs_extractor_scale_factors computes it the same way).  Only scale_factors_ is read, so the
//! adapter needs no member beyond those the other adapters use.
inline float level_sigma_sq(const data::keyframe* keyfrm, const int octave) {
    const float s = keyfrm->scale_factors_.at(static_cast<std::size_t>(octave));
    return s * s;
}
}  // namespace adapters

inline solve::sim3_solver::sim3_solver(data::keyframe* keyfrm_1, data::keyframe* keyfrm_2, const std::vector<data::landmark*>& matched_lms_in_keyfrm_2,
                                       const bool fix_scale, const unsigned int min_num_inliers)
    : sim3_solver(fix_scale, min_num_inliers) {
    const auto keyfrm_1_lms = keyfrm_1->get_landmarks();
    for (std::size_t idx1 = 0; idx1 < keyfrm_1_lms.size() && idx1 < matched_lms_in_keyfrm_2.size(); ++idx1) {
        data::landmark* lm_1 = keyfrm_1_lms[idx1];
        data::landmark* lm_2 = matched_lms_in_keyfrm_2[idx1];
        if (!lm_1 || !lm_2) continue;
        if (lm_1->will_be_erased() || lm_2->will_be_erased()) continue;
        const int idx2 = lm_2->get_index_in_keyframe(keyfrm_2);
        if (idx2 < 0) continue;
        const Vec3_t p1 = lm_1->get_pos_in_world(), p2 = lm_2->get_pos_in_world();
        for (int k = 0; k < 3; ++k) { own_pos_w_1_.push_back(p1(k)); own_pos_w_2_.push_back(p2(k)); }
        own_sigma_sq_1_.push_back(adapters::level_sigma_sq(keyfrm_1, keyfrm_1->undist_keypts_.at(idx1).octave));
        own_sigma_sq_2_.push_back(adapters::level_sigma_sq(keyfrm_2, keyfrm_2->undist_keypts_.at(static_cast<std::size_t>(idx2)).octave));
    }
    own_poses_.resize(24);
    adapters::to_Rt(keyfrm_1->get_cam_pose(), own_poses_.data());
    adapters::to_Rt(keyfrm_2->get_cam_pose(), own_poses_.data() + 12);
    own_.camera_1 = adapters::to_camera(keyfrm_1->camera_);
    own_.camera_2 = adapters::to_camera(keyfrm_2->camera_);
    own_.cam_pose_1w = own_poses_.data(); own_.cam_pose_2w = own_poses_.data() + 12;
    own_.num_pairs = static_cast<int>(own_sigma_sq_1_.size());
    own_.pos_w_1 = own_pos_w_1_.data(); own_.level_sigma_sq_1 = own_sigma_sq_1_.data();
    own_.pos_w_2 = own_pos_w_2_.data(); own_.level_sigma_sq_2 = own_sigma_sq_2_.data();
    own_.seed = (static_cast<std::uint64_t>(keyfrm_1->id_) << 32) | static_cast<std::uint64_t>(keyfrm_2->id_);
}

inline void solve::sim3_solver::find_via_ransac(const unsigned int max_num_iter) {
    best_ = find_via_ransac(std::vector<problem_view>{own_}, max_num_iter).front();
}

inline Mat33_t solve::sim3_solver::get_best_rotation_12() const {
    Mat33_t R;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R(r, c) = best_.sim3_12[3 * r + c];
    return R;
}

inline Vec3_t solve::sim3_solver::get_best_translation_12() const {
    Vec3_t t;
    for (int k = 0; k < 3; ++k) t(k) = best_.sim3_12[9 + k];
    return t;
}

// ------------------------------------------------------------------------------------------------ solve::pnp_solver
// The reference's constructor takes, per correspondence, the frame keypoint's bearing, the keypoint (for its octave) and the
// landmark's world position; max_cos_error is formed on the device from scale_factors[octave].  The sampler seed is a splitmix64
// hash of the input bits, so the same input always gives the same solution.
template <class BearingVector, class PointVector>
inline solve::pnp_solver::pnp_solver(const BearingVector& valid_bearings, const std::vector<cv::KeyPoint>& valid_keypts,
                                     const PointVector& valid_points, const std::vector<float>& scale_factors,
                                     const unsigned int min_num_inliers)
    : pnp_solver(min_num_inliers) {
    const std::size_t n = valid_bearings.size();
    adapters::input_hash hash(n);
    for (std::size_t i = 0; i < n; ++i) {
        const auto& b = valid_bearings[i];
        const auto& p = valid_points.at(i);
        for (int k = 0; k < 3; ++k) { own_bearings_.push_back(b(k)); own_pos_w_.push_back(p(k)); }
        own_scale_factor_.push_back(scale_factors.at(static_cast<std::size_t>(valid_keypts.at(i).octave)));
    }
    hash.add(own_bearings_.data(), 8 * own_bearings_.size());
    hash.add(own_pos_w_.data(), 8 * own_pos_w_.size());
    hash.add(own_scale_factor_.data(), 4 * own_scale_factor_.size());
    own_.num_corrs = static_cast<int>(n);
    own_.bearings = own_bearings_.data(); own_.pos_w = own_pos_w_.data(); own_.scale_factor = own_scale_factor_.data();
    own_.seed = hash.seed;
}

inline void solve::pnp_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute) {
    best_ = find_via_ransac(std::vector<problem_view>{own_}, max_num_iter, recompute).front();
}

inline Mat33_t solve::pnp_solver::get_best_rotation() const {
    Mat33_t R;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R(r, c) = best_.pose_cw[3 * r + c];
    return R;
}

inline Vec3_t solve::pnp_solver::get_best_translation() const {
    Vec3_t t;
    for (int k = 0; k < 3; ++k) t(k) = best_.pose_cw[9 + k];
    return t;
}

inline Mat44_t solve::pnp_solver::get_best_cam_pose() const { return adapters::from_Rt(best_.pose_cw); }

// ------------------------------------------------------------------------------------------- solve::essential_solver
// The reference's constructor takes both views' bearings and the matches (idx_1, idx_2); the bearings are gathered per match here.
// The sampler seed is a splitmix64 hash of the gathered bearings (the PnP adapter's rule).
template <class BearingVector>
inline solve::essential_solver::essential_solver(const BearingVector& bearings_1, const BearingVector& bearings_2,
                                                 const std::vector<std::pair<int, int>>& matches_12)
    : essential_solver() {
    const std::size_t n = matches_12.size();
    for (const auto& m : matches_12) {
        const auto& b1 = bearings_1.at(static_cast<std::size_t>(m.first));
        const auto& b2 = bearings_2.at(static_cast<std::size_t>(m.second));
        for (int k = 0; k < 3; ++k) { own_bearings_1_.push_back(b1(k)); own_bearings_2_.push_back(b2(k)); }
    }
    adapters::input_hash hash(n);
    hash.add(own_bearings_1_.data(), 8 * own_bearings_1_.size());
    hash.add(own_bearings_2_.data(), 8 * own_bearings_2_.size());
    own_.num_matches = static_cast<int>(n);
    own_.bearings_1 = own_bearings_1_.data(); own_.bearings_2 = own_bearings_2_.data();
    own_.seed = hash.seed;
}

inline void solve::essential_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute) {
    best_ = find_via_ransac(std::vector<problem_view>{own_}, max_num_iter, recompute).front();
}

inline Mat33_t solve::essential_solver::get_best_E_21() const {
    Mat33_t E;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) E(r, c) = best_.E_21[3 * r + c];
    return E;
}

// ------------------------------------------------------------------ solve::homography_solver / solve::fundamental_solver
namespace adapters {
//! The reference constructors' problem: all keypoints of both views (cv::KeyPoint is layout-compatible with ovs_keypoint) and the
//! matches.  The sampler seed is a splitmix64 hash of the keypoint coordinates and the matches (the PnP adapter's rule).
inline void two_view_problem(const std::vector<cv::KeyPoint>& k1, const std::vector<cv::KeyPoint>& k2,
                             const std::vector<std::pair<int, int>>& matches_12, std::vector<ovs_keypoint>& own_1,
                             std::vector<ovs_keypoint>& own_2, std::vector<std::int32_t>& own_m,
                             solve::two_view_solver_base::problem_view& view) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(ovs_keypoint), "cv::KeyPoint layout changed");
    own_1.resize(k1.size()); own_2.resize(k2.size());
    if (!k1.empty()) std::memcpy(own_1.data(), k1.data(), sizeof(ovs_keypoint) * k1.size());
    if (!k2.empty()) std::memcpy(own_2.data(), k2.data(), sizeof(ovs_keypoint) * k2.size());
    own_m.clear();
    for (const auto& m : matches_12) { own_m.push_back(m.first); own_m.push_back(m.second); }
    input_hash hash(k1.size() + k2.size() + matches_12.size());
    for (const auto& k : own_1) { hash.add(&k.x, 4); hash.add(&k.y, 4); }
    for (const auto& k : own_2) { hash.add(&k.x, 4); hash.add(&k.y, 4); }
    hash.add(own_m.data(), 4 * own_m.size());
    view.num_keypts_1 = static_cast<int>(own_1.size()); view.keypts_1 = own_1.data();
    view.num_keypts_2 = static_cast<int>(own_2.size()); view.keypts_2 = own_2.data();
    view.num_matches = static_cast<int>(matches_12.size()); view.matches_12 = own_m.data();
    view.seed = hash.seed;
}
inline Mat33_t to_mat33(const double* M) {
    Mat33_t out;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) out(r, c) = M[3 * r + c];
    return out;
}
}  // namespace adapters

inline solve::homography_solver::homography_solver(const std::vector<cv::KeyPoint>& undist_keypts_1,
                                                   const std::vector<cv::KeyPoint>& undist_keypts_2,
                                                   const std::vector<std::pair<int, int>>& matches_12, const float sigma)
    : homography_solver(sigma) {
    adapters::two_view_problem(undist_keypts_1, undist_keypts_2, matches_12, own_keypts_1_, own_keypts_2_, own_matches_, own_);
}

inline void solve::homography_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute) {
    best_ = two_view_solver_base::find_via_ransac(std::vector<problem_view>{own_}, max_num_iter, recompute).front();
}

inline Mat33_t solve::homography_solver::get_best_H_21() const { return adapters::to_mat33(best_.M_21); }

inline solve::fundamental_solver::fundamental_solver(const std::vector<cv::KeyPoint>& undist_keypts_1,
                                                     const std::vector<cv::KeyPoint>& undist_keypts_2,
                                                     const std::vector<std::pair<int, int>>& matches_12, const float sigma)
    : fundamental_solver(sigma) {
    adapters::two_view_problem(undist_keypts_1, undist_keypts_2, matches_12, own_keypts_1_, own_keypts_2_, own_matches_, own_);
}

inline void solve::fundamental_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute) {
    best_ = two_view_solver_base::find_via_ransac(std::vector<problem_view>{own_}, max_num_iter, recompute).front();
}

inline Mat33_t solve::fundamental_solver::get_best_F_21() const { return adapters::to_mat33(best_.M_21); }

// ------------------------------------------------------------------ module::two_view_triangulator / create_new_landmarks
namespace adapters {
//! A keyframe's own vectors as an ovs_keyframe_view (owns the flattened copies): undist_keypts_ (cv::KeyPoint is layout-compatible
//! with ovs_keypoint), bearings_, stereo_x_right_ / depths_ (left out when the keyframe has no stereo keypoint), descriptors_, the
//! landmark flags (get_landmarks()[i] != nullptr), bow_feat_vec_ inverted into node ids, the scale tables, the pose and the camera.
//! true_baseline is focal_x_baseline_ / fx_, the value the reference's perspective-family camera constructors store.
struct keyframe_arrays {
    std::vector<ovs_keypoint> keypts;
    std::vector<double> bearings;
    std::vector<float> x_right, depths;
    std::vector<std::uint8_t> desc, has_landmark;
    std::vector<std::int32_t> bow_node;
    ovs_keyframe_view view{};
    template <class Keyframe>
    explicit keyframe_arrays(Keyframe* k) {
        static_assert(sizeof(cv::KeyPoint) == sizeof(ovs_keypoint), "cv::KeyPoint layout changed");
        const std::size_t n = k->undist_keypts_.size();
        keypts.resize(n);
        if (n) std::memcpy(keypts.data(), k->undist_keypts_.data(), sizeof(ovs_keypoint) * n);
        bearings = flat_bearings(k->bearings_);
        const bool stereo = k->stereo_x_right_.size() == n && k->depths_.size() == n &&
                            std::any_of(k->stereo_x_right_.begin(), k->stereo_x_right_.end(), [](float x) { return 0.0f <= x; });
        if (stereo) { x_right.assign(k->stereo_x_right_.begin(), k->stereo_x_right_.end()); depths.assign(k->depths_.begin(), k->depths_.end()); }
        desc.resize(32 * n);
        for (std::size_t i = 0; i < n; ++i) std::memcpy(&desc[32 * i], k->descriptors_.ptr(static_cast<int>(i)), 32);   // rows may be strided
        const auto lms = k->get_landmarks();
        has_landmark.assign(n, 0);
        for (std::size_t i = 0; i < n && i < lms.size(); ++i) has_landmark[i] = lms[i] != nullptr;
        bow_node.assign(n, -1);
        for (const auto& node : k->bow_feat_vec_)
            for (const auto idx : node.second)
                if (static_cast<std::size_t>(idx) < n) bow_node[idx] = static_cast<std::int32_t>(node.first);
        to_Rt(k->get_cam_pose(), view.pose_cw);
        view.camera = to_camera(k->camera_);
        view.true_baseline = view.camera.fx != 0.0 ? view.camera.focal_x_baseline / view.camera.fx : 0.0;
        view.scale_factor = k->scale_factor_;
        view.num_scale_levels = static_cast<std::int32_t>(k->scale_factors_.size());
        view.scale_factors = k->scale_factors_.data(); view.level_sigma_sq = k->level_sigma_sq_.data();
        view.num_keypts = static_cast<std::int32_t>(n);
        view.undist_keypts = keypts.data(); view.bearings = bearings.data();
        view.stereo_x_right = stereo ? x_right.data() : nullptr; view.depths = stereo ? depths.data() : nullptr;
        view.descriptors = desc.data(); view.has_landmark = has_landmark.data(); view.bow_node = bow_node.data();
    }
};

//! E_12 = [t_12]x R_12 with R_12 = R_1w R_2w^T, t_12 = t_1w - R_12 t_2w (the reference's essential_solver::create_E_21 with the two
//! keyframes swapped), and the epipole: keyframe 1's centre c_1 = -R_1w^T t_1w as a unit bearing of keyframe 2, R_2w c_1 + t_2w.
inline void e12_and_epipole(const double* P1, const double* P2, std::array<double, 9>& E, std::array<double, 3>& epipole) {
    double R12[9], t12[3], c1[3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R12[3 * r + c] = P1[3 * r] * P2[3 * c] + P1[3 * r + 1] * P2[3 * c + 1] + P1[3 * r + 2] * P2[3 * c + 2];
    for (int r = 0; r < 3; ++r) t12[r] = P1[9 + r] - (R12[3 * r] * P2[9] + R12[3 * r + 1] * P2[10] + R12[3 * r + 2] * P2[11]);
    const double tx[9] = {0, -t12[2], t12[1], t12[2], 0, -t12[0], -t12[1], t12[0], 0};
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) E[3 * r + c] = tx[3 * r] * R12[c] + tx[3 * r + 1] * R12[3 + c] + tx[3 * r + 2] * R12[6 + c];
    for (int r = 0; r < 3; ++r) c1[r] = -(P1[r] * P1[9] + P1[3 + r] * P1[10] + P1[6 + r] * P1[11]);
    double e[3];
    for (int r = 0; r < 3; ++r) e[r] = P2[3 * r] * c1[0] + P2[3 * r + 1] * c1[1] + P2[3 * r + 2] * c1[2] + P2[9 + r];
    const double nrm = std::sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    for (int r = 0; r < 3; ++r) epipole[r] = e[r] / nrm;
}
}  // namespace adapters

// create_new_landmarks on data::keyframe: the neighbours are the ones that passed the caller's baseline / depth gates, in the
// reference's order.  Records (neighbour, idx_1, idx_2, pos_w) in creation order; making the landmarks stays with the caller.
template <class Keyframe>
inline std::vector<ovs_new_landmark> module::two_view_triangulator::create_new_landmarks(Keyframe* keyfrm_1,
                                                                                         const std::vector<Keyframe*>& neighbours,
                                                                                         const bool check_orientation) const {
    const adapters::keyframe_arrays k1(keyfrm_1);
    std::vector<adapters::keyframe_arrays> own;
    own.reserve(neighbours.size());
    std::vector<ovs_keyframe_view> views;
    std::vector<std::array<double, 9>> E(neighbours.size());
    std::vector<std::array<double, 3>> ep(neighbours.size());
    for (std::size_t b = 0; b < neighbours.size(); ++b) {
        own.emplace_back(neighbours[b]);
        views.push_back(own.back().view);
        adapters::e12_and_epipole(k1.view.pose_cw, own.back().view.pose_cw, E[b], ep[b]);
    }
    return create_new_landmarks(k1.view, views, E, ep, check_orientation);
}

// ------------------------------------------------------------------------------------------- initialize::perspective / bearing_vector
namespace adapters {

//! camera_, undist_keypts_ (cv::KeyPoint is ovs_keypoint's layout) and bearings_ of a frame as an ovs_init_view; the bearings are
//! copied into `bearings` (3 doubles per keypoint), which must outlive the view.
template <class Frame>
ovs_init_view init_view(const Frame& frm, std::vector<double>& bearings) {
    bearings = flat_bearings(frm.bearings_);
    ovs_init_view v{};
    v.camera = to_camera(frm.camera_);
    v.num_keypts = static_cast<std::int32_t>(frm.undist_keypts_.size());
    v.undist_keypts = reinterpret_cast<const ovs_keypoint*>(frm.undist_keypts_.data());
    v.bearings = bearings.data();
    return v;
}

//! The sampler seed of an initialize() on the reference's frames: the hash of both views' keypoints and bearings and the matches.
inline std::uint64_t init_seed(const ovs_init_view& ref, const ovs_init_view& cur, const std::vector<int>& ref_matches_with_cur) {
    input_hash hash(static_cast<std::size_t>(ref.num_keypts) + static_cast<std::size_t>(cur.num_keypts));
    for (const ovs_init_view* v : {&ref, &cur}) {
        for (int i = 0; i < v->num_keypts; ++i) hash.add(&v->undist_keypts[i].x, 8);
        hash.add(v->bearings, 24 * static_cast<std::size_t>(v->num_keypts));
    }
    hash.add(ref_matches_with_cur.data(), sizeof(int) * ref_matches_with_cur.size());
    return hash.seed;
}

}  // namespace adapters

template <class Frame>
inline initialize::perspective::perspective(const Frame& ref_frm, const unsigned int num_ransac_iters, const unsigned int min_num_triangulated,
                                            const float parallax_deg_thr, const float reproj_err_thr, const int device)
    : base(true, nullptr, num_ransac_iters, min_num_triangulated, parallax_deg_thr, reproj_err_thr, device) {
    own_ref_ = adapters::init_view(ref_frm, own_ref_bearings_);
    ref_ = &own_ref_;
}

template <class Frame>
inline initialize::bearing_vector::bearing_vector(const Frame& ref_frm, const unsigned int num_ransac_iters,
                                                  const unsigned int min_num_triangulated, const float parallax_deg_thr,
                                                  const float reproj_err_thr, const int device)
    : base(false, nullptr, num_ransac_iters, min_num_triangulated, parallax_deg_thr, reproj_err_thr, device) {
    own_ref_ = adapters::init_view(ref_frm, own_ref_bearings_);
    ref_ = &own_ref_;
}

template <class Frame>
inline bool initialize::base::initialize(const Frame& cur_frm, const std::vector<int>& ref_matches_with_cur) {
    std::vector<double> bearings;
    const ovs_init_view cur = adapters::init_view(cur_frm, bearings);
    return initialize(cur, ref_matches_with_cur, adapters::init_seed(*ref_, cur, ref_matches_with_cur));
}

inline Mat33_t initialize::base::get_rotation_ref_to_cur() const {
    Mat33_t R;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R(r, c) = last_.record.rot_ref_to_cur[3 * r + c];
    return R;
}

inline Vec3_t initialize::base::get_translation_ref_to_cur() const {
    Vec3_t t;
    for (int r = 0; r < 3; ++r) t(r) = last_.record.trans_ref_to_cur[r];
    return t;
}

inline std::vector<Vec3_t> initialize::base::get_triangulated_pts() const {
    std::vector<Vec3_t> out(last_.is_triangulated.size());
    for (std::size_t i = 0; i < out.size(); ++i)
        for (int r = 0; r < 3; ++r) out[i](r) = last_.triangulated_pts[3 * i + r];
    return out;
}

inline std::vector<bool> initialize::base::get_triangulated_flags() const {
    return std::vector<bool>(last_.is_triangulated.begin(), last_.is_triangulated.end());
}

template <class Camera>
inline util::stereo_rectifier::stereo_rectifier(const Camera* camera, const params& p, const int device)
    : stereo_rectifier(static_cast<int>(camera->cols_), static_cast<int>(camera->rows_),
                       std::array<double, 9>{camera->fx_, 0.0, camera->cx_, 0.0, camera->fy_, camera->cy_, 0.0, 0.0, 1.0}, p, device) {}

namespace adapters {
// cv::Mat::channels(); a matrix type without it (the single-channel stand-in the tests compile against) has one channel
template <class Mat>
inline auto mat_channels(const Mat& m, int) -> decltype(m.channels()) { return m.channels(); }
template <class Mat>
inline int mat_channels(const Mat&, long) { return 1; }
}  // namespace adapters

inline void util::stereo_rectifier::rectify(const cv::Mat& in_img_l, const cv::Mat& in_img_r, cv::Mat& out_img_l, cv::Mat& out_img_r) const {
    CV_Assert(in_img_l.rows == in_img_r.rows && in_img_l.cols == in_img_r.cols && in_img_l.type() == in_img_r.type());
    CV_Assert(in_img_l.step == in_img_r.step);
    cv::Mat l(in_img_l.rows, in_img_l.cols, in_img_l.type()), r(in_img_r.rows, in_img_r.cols, in_img_r.type());
    rectify(in_img_l.data, in_img_r.data, in_img_l.rows, in_img_l.cols, in_img_l.step, adapters::mat_channels(in_img_l, 0), l.data, r.data, l.step);
    out_img_l = l; out_img_r = r;
}

}  // namespace openvslam
