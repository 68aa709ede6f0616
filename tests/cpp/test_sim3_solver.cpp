// tests/cpp/test_sim3_solver.cpp -- openvslam::solve::sim3_solver through the adapter with the reference's own signature
// (include/openvslam_b200/adapters.hpp) against ground truth: two stand-in keyframes related by a known Sim3 (scale 1.3), 120
// matched landmark pairs of which 30 are wrong 3-D correspondences, plus pairs the constructor must drop (no match, an erased
// landmark, a landmark not observed in keyframe 2).  Then the batched class-layer call on two candidates.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "openvslam_b200/adapters.hpp"

int main() {
    using namespace openvslam;
    camera::perspective cam(camera::setup_type_t::Monocular, 640, 480, 500, 500, 320, 240, 0);
    // S_12: rotation of 0.2 rad about y, t = (0.3, -0.1, 0.2), s = 1.3; camera 1 at the world origin, camera 2 shifted
    const double c = std::cos(0.2), s = std::sin(0.2);
    const double S_true[13] = {c, 0, s, 0, 1, 0, -s, 0, c, 0.3, -0.1, 0.2, 1.3};
    data::keyframe kf1(7, &cam), kf2(9, &cam);
    Mat44_t T2 = Mat44_t::Identity();
    T2(0, 3) = 0.5; T2(2, 3) = -0.2;
    kf2.set_cam_pose(T2);
    // scale_factors_ as orb_params::calc_scale_factors forms them (scale factor 1.2); level_sigma_sq_ is their float square
    std::vector<float> sigma_sq;
    for (data::keyframe* k : {&kf1, &kf2}) {
        float sf = 1.0f;
        sigma_sq.clear();
        for (int l = 0; l < 8; ++l) { k->scale_factors_.push_back(sf); sigma_sq.push_back(sf * sf); sf = 1.2f * sf; }
    }
    for (int l = 0; l < 8; ++l)
        if (adapters::level_sigma_sq(&kf2, l) != sigma_sq[static_cast<std::size_t>(l)]) { std::printf("level_sigma_sq differs at level %d\n", l); return 1; }
    const int N = 130, num_wrong = 30;
    std::mt19937 rng(5);
    std::uniform_real_distribution<double> u(-1, 1);
    std::vector<std::unique_ptr<data::landmark>> lms;
    std::vector<data::landmark*> matched(N, nullptr);
    for (int i = 0; i < N; ++i) {
        const double p2[3] = {1.5 * u(rng), 1.0 * u(rng), 5 + 1.5 * u(rng)};   // camera-2 coordinates
        double p1[3];
        for (int r = 0; r < 3; ++r) p1[r] = S_true[12] * (S_true[3 * r] * p2[0] + S_true[3 * r + 1] * p2[1] + S_true[3 * r + 2] * p2[2]) + S_true[9 + r];
        if (i < num_wrong) { p1[0] += 0.8 * u(rng) + 1.0; p1[1] -= 0.6; }
        Vec3_t w1, w2;
        for (int r = 0; r < 3; ++r) { w1(r) = p1[r]; w2(r) = p2[r] - T2(r, 3); }
        lms.emplace_back(new data::landmark(2 * i, w1));
        lms.emplace_back(new data::landmark(2 * i + 1, w2));
        data::landmark* l1 = lms[lms.size() - 2].get();
        data::landmark* l2 = lms.back().get();
        cv::KeyPoint k1, k2;
        k1.octave = i % 8; k2.octave = (i / 8) % 8;
        kf1.undist_keypts_.push_back(k1); kf2.undist_keypts_.push_back(k2);
        kf1.add_landmark(l1, i); l1->add_observation(&kf1, i);
        if (i == N - 1) continue;                                     // not observed in keyframe 2: dropped
        kf2.add_landmark(l2, i); l2->add_observation(&kf2, i);
        if (i == N - 2) continue;                                     // not matched: dropped
        if (i == N - 3) l2->will_be_erased_ = true;                   // erased: dropped
        matched[i] = l2;
    }
    try {
        solve::sim3_solver solver(&kf1, &kf2, matched, false, 20);
        solver.find_via_ransac(200);
        const auto& sol = solver.best_solution();
        const Mat33_t R = solver.get_best_rotation_12();
        const Vec3_t t = solver.get_best_translation_12();
        // get_best_scale_12() is a float as in the reference: the double scale is checked to 1e-9, the float to its rounding
        if (std::fabs(solver.get_best_scale_12() - 1.3f) > 1e-6f) return 1;
        double err = std::fabs(sol.sim3_12[12] - 1.3);
        for (int r = 0; r < 3; ++r) {
            err = std::fmax(err, std::fabs(t(r) - S_true[9 + r]));
            for (int k = 0; k < 3; ++k) err = std::fmax(err, std::fabs(R(r, k) - S_true[3 * r + k]));
        }
        int wrong_kept = 0;
        for (int i = 0; i < num_wrong; ++i) wrong_kept += sol.is_inlier[i];
        std::printf("sim3 solver: valid %d, %u of %zu pairs inliers (hypothesis %d), %d wrong pairs kept, max |S - S_true| = %.2e\n",
                    solver.solution_is_valid() ? 1 : 0, sol.num_inliers, sol.is_inlier.size(), sol.best_iter, wrong_kept, err);
        if (!solver.solution_is_valid() || sol.is_inlier.size() != static_cast<std::size_t>(N - 3) || sol.num_inliers != N - 3 - num_wrong ||
            wrong_kept != 0 || err > 1e-9)
            return 1;
        // the same candidate twice in one batched call, once with a fixed scale solver
        std::vector<double> pw1, pw2;
        std::vector<float> s1, s2;
        for (int i = num_wrong; i < N - 3; ++i) {
            const Vec3_t a = kf1.get_landmark(i)->get_pos_in_world(), b = matched[i]->get_pos_in_world();
            for (int r = 0; r < 3; ++r) { pw1.push_back(a(r)); pw2.push_back(b(r)); }
            s1.push_back(1.0f); s2.push_back(1.0f);
        }
        double pose1[12], pose2[12];
        adapters::to_Rt(kf1.get_cam_pose(), pose1);
        adapters::to_Rt(kf2.get_cam_pose(), pose2);
        solve::sim3_solver::problem_view v;
        v.camera_1 = v.camera_2 = adapters::to_camera(&cam);
        v.cam_pose_1w = pose1; v.cam_pose_2w = pose2;
        v.num_pairs = static_cast<int>(s1.size());
        v.pos_w_1 = pw1.data(); v.level_sigma_sq_1 = s1.data(); v.pos_w_2 = pw2.data(); v.level_sigma_sq_2 = s2.data();
        solve::sim3_solver batch(false);
        std::vector<solve::sim3_solver::problem_view> probs{v, v};
        probs[1].seed = 3;
        const auto out = batch.find_via_ransac(probs, 50);
        for (const auto& o : out) {
            double e = std::fabs(o.sim3_12[12] - 1.3);
            for (int k = 0; k < 12; ++k) e = std::fmax(e, std::fabs(o.sim3_12[k] - S_true[k]));
            std::printf("batched: valid %d, %u inliers, max |S - S_true| = %.2e\n", o.valid ? 1 : 0, o.num_inliers, e);
            if (!o.valid || o.num_inliers != static_cast<unsigned>(v.num_pairs) || e > 1e-9) return 1;
        }
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("sim3 solver ok\n");
    return 0;
}
