// tests/cpp/test_adapters.cpp -- compiles include/openvslam_b200/adapters.hpp (the reference's own method signatures on the
// reference's data model) against the stand-in headers of tests/cpp/standin and, on a GPU box, runs one call of each:
//   orb_extractor::extract(cv::_InputArray, cv::_InputArray, std::vector<cv::KeyPoint>&, cv::_OutputArray)
//   match::robust::brute_force_match(data::frame&, data::keyframe*, matches)
//   match::projection::match_frame_and_landmarks(data::frame&, const std::vector<data::landmark*>&, margin)
//   optimize::pose_optimizer::optimize(data::frame&)
//   optimize::local_bundle_adjuster::optimize(data::keyframe*, bool* const)
// Exit codes: 0 ok, 2 no GPU (OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <vector>

#include "openvslam_b200/adapters.hpp"

using namespace openvslam;

namespace {
struct World {
    camera::perspective cam{camera::setup_type_t::Monocular, 640, 480, 500.0, 500.0, 320.0, 240.0, 0.0};
    std::vector<std::unique_ptr<data::landmark>> lms;
    std::vector<std::unique_ptr<data::keyframe>> kfs;
    std::vector<Vec3_t> true_pos;
    std::vector<Mat44_t> true_pose;
};

Mat44_t pose_at(double cx, double yaw) {
    Mat44_t T = Mat44_t::Identity();
    const double c = std::cos(yaw), s = std::sin(yaw);
    T(0, 0) = c; T(0, 2) = s; T(2, 0) = -s; T(2, 2) = c;            // R (world -> camera)
    const double C[3] = {cx, 0.0, 0.0};
    for (int r = 0; r < 3; ++r) T(r, 3) = -(T(r, 0) * C[0] + T(r, 1) * C[1] + T(r, 2) * C[2]);
    return T;
}
bool project(const camera::perspective& cam, const Mat44_t& T, const Vec3_t& p, float& u, float& v) {
    double pc[3];
    for (int r = 0; r < 3; ++r) pc[r] = T(r, 0) * p(0) + T(r, 1) * p(1) + T(r, 2) * p(2) + T(r, 3);
    if (pc[2] < 0.5) return false;
    u = static_cast<float>(cam.fx_ * pc[0] / pc[2] + cam.cx_); v = static_cast<float>(cam.fy_ * pc[1] / pc[2] + cam.cy_);
    return u >= 20 && u < 620 && v >= 20 && v < 460;
}
std::vector<float> sf8() { std::vector<float> s(8); for (int i = 0; i < 8; ++i) s[i] = std::pow(1.2f, (float)i); return s; }
std::vector<float> inv_sigma8() { std::vector<float> s = sf8(); for (float& v : s) v = 1.0f / (v * v); return s; }
}  // namespace

int main() {
    std::mt19937 rng(11);
    std::normal_distribution<double> gauss(0.0, 1.0);
    std::uniform_real_distribution<double> uni(0.0, 1.0);
    try {
        // ---- extract with the reference's cv:: signature
        feature::orb_extractor extractor(feature::orb_params(1000, 1.2f, 8, 20, 7));
        {
            cv::Mat img(480, 640, CV_8U);
            for (int i = 0; i < 480 * 640; ++i) img.data[i] = 110;
            for (int r = 0; r < 400; ++r) {
                const int x = rng() % 640, y = rng() % 480, w = 4 + rng() % 40, h = 4 + rng() % 40, v = 20 + rng() % 216;
                for (int yy = y; yy < std::min(480, y + h); ++yy) for (int xx = x; xx < std::min(640, x + w); ++xx) img.data[yy * 640 + xx] = (unsigned char)v;
            }
            std::vector<cv::KeyPoint> keypts; cv::Mat descriptors;
            extractor.extract(img, cv::noArray(), keypts, descriptors);
            std::printf("extract(cv::Mat): %zu keypoints, descriptors %d x %d\n", keypts.size(), descriptors.rows, descriptors.cols);
            if (keypts.size() < 500 || descriptors.rows != (int)keypts.size() || descriptors.cols != 32) return 1;
        }
        // ---- a small map: 6 keyframes on a line, 400 landmarks in front of them
        World w;
        const int NL = 400, NK = 6;
        std::vector<cv::Mat> lm_desc(NL);
        for (int l = 0; l < NL; ++l) {
            Vec3_t p; p(0) = -3 + 9 * uni(rng); p(1) = -2 + 4 * uni(rng); p(2) = 5 + 6 * uni(rng);
            w.true_pos.push_back(p);
            Vec3_t noisy = p; for (int k = 0; k < 3; ++k) noisy(k) += 0.008 * gauss(rng);
            w.lms.emplace_back(new data::landmark((unsigned)l, noisy));
            cv::Mat d(1, 32, CV_8U); for (int b = 0; b < 32; ++b) d.data[b] = (unsigned char)(rng() & 255);
            lm_desc[l] = d; w.lms.back()->set_descriptor(d);
        }
        for (int k = 0; k < NK; ++k) {
            const Mat44_t T = pose_at(0.6 * k, 0.02 * k);
            w.true_pose.push_back(T);
            w.kfs.emplace_back(new data::keyframe((unsigned)k, &w.cam));
            data::keyframe* kf = w.kfs.back().get();
            kf->scale_factors_ = sf8(); kf->inv_level_sigma_sq_ = inv_sigma8();
            std::vector<unsigned char> rows;
            for (int l = 0; l < NL; ++l) {
                float u, v;
                if (!project(w.cam, T, w.true_pos[l], u, v)) continue;
                cv::KeyPoint kp; kp.pt = cv::Point2f(u + (float)(0.5 * gauss(rng)), v + (float)(0.5 * gauss(rng))); kp.octave = 0; kp.angle = 0; kp.size = 31;
                if (uni(rng) < 0.04) { kp.pt.x += 25; kp.pt.y -= 18; }                          // a few gross outliers
                const unsigned idx = (unsigned)kf->undist_keypts_.size();
                kf->undist_keypts_.push_back(kp); kf->stereo_x_right_.push_back(-1.0f);
                kf->add_landmark(w.lms[l].get(), idx); w.lms[l]->add_observation(kf, idx);
                for (int b = 0; b < 32; ++b) rows.push_back(lm_desc[l].data[b]);
                rows[rows.size() - 32 + (rng() % 32)] ^= (unsigned char)(1u << (rng() % 8));
            }
            kf->num_keypts_ = (unsigned)kf->undist_keypts_.size();
            kf->descriptors_ = cv::Mat((int)kf->num_keypts_, 32, CV_8U);
            std::memcpy(kf->descriptors_.data, rows.data(), rows.size());
            Mat44_t noisy = T; noisy(0, 3) += (k ? 0.03 * gauss(rng) : 0.0); noisy(2, 3) += (k ? 0.03 * gauss(rng) : 0.0);
            kf->set_cam_pose(noisy);
        }
        data::keyframe* curr = w.kfs[NK - 1].get();
        for (int k = 0; k + 1 < NK; ++k) curr->graph_node_->covisibilities_.push_back(w.kfs[k].get());

        // ---- a tracked frame at the last keyframe's true pose: its keypoints carry no landmarks yet
        data::frame frm;
        frm.camera_ = &w.cam; frm.scale_factors_ = sf8(); frm.inv_level_sigma_sq_ = inv_sigma8(); frm.num_scale_levels_ = 8;
        const Mat44_t Tf = w.true_pose[NK - 1];
        std::vector<data::landmark*> local_lms;
        std::vector<unsigned char> rows;
        for (int l = 0; l < NL; ++l) {
            float u, v;
            data::landmark* lm = w.lms[l].get();
            local_lms.push_back(lm);
            if (!project(w.cam, Tf, w.true_pos[l], u, v)) { lm->is_observable_in_tracking_ = false; continue; }
            cv::KeyPoint kp; kp.pt = cv::Point2f(u + (float)(0.4 * gauss(rng)), v + (float)(0.4 * gauss(rng))); kp.octave = 0; kp.angle = 0;
            frm.undist_keypts_.push_back(kp); frm.stereo_x_right_.push_back(-1.0f);
            for (int b = 0; b < 32; ++b) rows.push_back(lm_desc[l].data[b]);
            lm->is_observable_in_tracking_ = true; lm->scale_level_in_tracking_ = 0; lm->x_right_in_tracking_ = -1.0f;
            lm->reproj_in_tracking_(0) = u; lm->reproj_in_tracking_(1) = v;
        }
        frm.num_keypts_ = (unsigned)frm.undist_keypts_.size();
        frm.keypts_ = frm.undist_keypts_;
        frm.descriptors_ = cv::Mat((int)frm.num_keypts_, 32, CV_8U);
        std::memcpy(frm.descriptors_.data, rows.data(), rows.size());
        frm.landmarks_.assign(frm.num_keypts_, nullptr);
        frm.outlier_flags_.assign(frm.num_keypts_, false);

        match::projection projection_matcher(0.8f, true);
        const unsigned n_proj = projection_matcher.match_frame_and_landmarks(frm, local_lms, 5.0f);
        unsigned assigned = 0;
        for (auto* lm : frm.landmarks_) assigned += lm != nullptr;
        std::printf("match_frame_and_landmarks(frame&, landmarks, 5): %u matches on %u keypoints (%u assigned)\n", n_proj, frm.num_keypts_, assigned);
        if (n_proj < 0.8 * frm.num_keypts_ || assigned != n_proj) return 1;

        match::robust robust_matcher(0.75f, true);
        std::vector<std::pair<int, int>> matches;
        const unsigned n_bf = robust_matcher.brute_force_match(frm, curr, matches);
        std::printf("brute_force_match(frame&, keyframe*): %u matches\n", n_bf);
        if (n_bf < 0.5 * frm.num_keypts_) return 1;

        // ---- pose_optimizer::optimize(frame&) from a perturbed pose
        Mat44_t start = Tf; start(0, 3) += 0.08; start(2, 3) -= 0.05;
        frm.set_cam_pose(start);
        optimize::pose_optimizer pose_optimizer;
        const unsigned n_inl = pose_optimizer.optimize(frm);
        const double err = std::fabs(frm.cam_pose_cw_(0, 3) - Tf(0, 3)) + std::fabs(frm.cam_pose_cw_(2, 3) - Tf(2, 3));
        std::printf("pose_optimizer::optimize(frame&): %u inliers, translation error %.4f (start 0.13)\n", n_inl, err);
        if (n_inl < 0.8 * n_proj || err > 0.02) return 1;

        // ---- local_bundle_adjuster::optimize(keyframe*, bool*)
        auto reproj_error = [&]() {
            double s = 0; int n = 0;
            for (auto& kf : w.kfs)
                for (unsigned i = 0; i < kf->num_keypts_; ++i) {
                    data::landmark* lm = kf->get_landmark(i);
                    if (!lm) continue;
                    float u, v;
                    if (!project(w.cam, kf->get_cam_pose(), lm->get_pos_in_world(), u, v)) continue;
                    const double du = u - kf->undist_keypts_[i].pt.x, dv = v - kf->undist_keypts_[i].pt.y;
                    s += du * du + dv * dv; ++n;
                }
            return std::sqrt(s / std::max(n, 1));
        };
        const double e0 = reproj_error();
        bool force_stop = false;
        optimize::local_bundle_adjuster local_ba;
        local_ba.optimize(curr, &force_stop);
        const double e1 = reproj_error();
        int erased = 0, updated = 0;
        for (auto& kf : w.kfs) erased += kf->num_erased_;
        for (auto& lm : w.lms) updated += lm->num_updates_ > 0;
        std::printf("local_bundle_adjuster::optimize(keyframe*, bool*): rms reprojection %.3f -> %.3f px, %d outlier observations erased, %d landmarks updated\n",
                    e0, e1, erased, updated);
        if (!(e1 < 0.5 * e0) || e1 > 1.5 || erased < 10 || updated < 300) return 1;
        // the origin keyframe (id 0) is fixed
        if (w.kfs[0]->get_cam_pose()(0, 3) != w.true_pose[0](0, 3)) return 1;
        std::printf("adapters ok\n");
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
}
