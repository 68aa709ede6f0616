// tests/cpp/test_essential_solver.cpp -- openvslam::solve::essential_solver and match::robust::match_frame_and_keyframe through the
// adapters with the reference's own signatures (include/openvslam_b200/adapters.hpp) against ground truth: two views of 200 points
// at a known relative pose, noise-free bearings.  The solver must return E_21 = [t]x R (up to scale and sign) with every match an
// inlier; the matcher, on a frame whose keypoints carry the keyframe's descriptors in shuffled order, must hand every frame
// keypoint its own keyframe landmark.  Then a batch of 6 problems through the class layer against the per-problem calls.
// The stand-in data::frame / data::keyframe (tests/cpp/standin) declare no bearings_; the reference's do, so this program adds
// the member in derived types, which the adapter's template takes as it takes the reference's classes.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <numeric>
#include <random>
#include <string>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace {
struct frame_with_bearings : openvslam::data::frame {
    std::vector<openvslam::Vec3_t> bearings_;   // eigen_alloc_vector<bearing_t> in the reference
};
struct keyframe_with_bearings : openvslam::data::keyframe {
    using openvslam::data::keyframe::keyframe;
    std::vector<openvslam::Vec3_t> bearings_;
};
}  // namespace

int main() {
    using namespace openvslam;
    // p_2 = R p_1 + t: rotation of 0.2 rad about (2, -1, 2) / 3, t = (0.5, 0.1, -0.2)
    const double th = 0.2, ax[3] = {2.0 / 3, -1.0 / 3, 2.0 / 3}, c = std::cos(th), s = std::sin(th);
    const double K[9] = {0, -ax[2], ax[1], ax[2], 0, -ax[0], -ax[1], ax[0], 0};
    double R[9], t[3] = {0.5, 0.1, -0.2};
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) {
            double KK = 0;
            for (int m = 0; m < 3; ++m) KK += K[3 * r + m] * K[3 * m + k];
            R[3 * r + k] = (r == k ? 1.0 : 0.0) + s * K[3 * r + k] + (1 - c) * KK;
        }
    // E = [t]x R, scaled to unit Frobenius norm
    const double T[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    double E_true[9], nrm = 0;
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) {
            double v = 0;
            for (int m = 0; m < 3; ++m) v += T[3 * r + m] * R[3 * m + k];
            E_true[3 * r + k] = v;
            nrm += v * v;
        }
    for (double& v : E_true) v /= std::sqrt(nrm);
    auto E_error = [&](const double* E) {   // max |E / |E| -/+ E_true|, the better sign
        double n2 = 0, ep = 0, em = 0;
        for (int k = 0; k < 9; ++k) n2 += E[k] * E[k];
        for (int k = 0; k < 9; ++k) {
            ep = std::fmax(ep, std::fabs(E[k] / std::sqrt(n2) - E_true[k]));
            em = std::fmax(em, std::fabs(E[k] / std::sqrt(n2) + E_true[k]));
        }
        return std::fmin(ep, em);
    };
    const int N = 200;
    std::mt19937 rng(5);
    std::uniform_real_distribution<double> u(-1, 1);
    std::vector<Vec3_t> bear_1, bear_2;
    for (int i = 0; i < N; ++i) {
        const double z = 6.0 + 4.0 * u(rng);
        const double p1[3] = {0.9 * z * u(rng), 0.7 * z * u(rng), z};
        double p2[3];
        for (int r = 0; r < 3; ++r) p2[r] = R[3 * r] * p1[0] + R[3 * r + 1] * p1[1] + R[3 * r + 2] * p1[2] + t[r];
        const double L1 = std::sqrt(p1[0] * p1[0] + p1[1] * p1[1] + p1[2] * p1[2]), L2 = std::sqrt(p2[0] * p2[0] + p2[1] * p2[1] + p2[2] * p2[2]);
        Vec3_t b1, b2;
        for (int k = 0; k < 3; ++k) { b1(k) = p1[k] / L1; b2(k) = p2[k] / L2; }
        bear_1.push_back(b1); bear_2.push_back(b2);
    }
    try {
        // 1. the solver with the reference's constructor: match i = (i, perm[i])
        std::vector<int> perm(N);
        std::iota(perm.begin(), perm.end(), 0);
        std::shuffle(perm.begin(), perm.end(), rng);
        std::vector<Vec3_t> bear_2p(N);
        for (int i = 0; i < N; ++i) bear_2p[perm[i]] = bear_2[i];
        std::vector<std::pair<int, int>> matches_12;
        for (int i = 0; i < N; ++i) matches_12.emplace_back(i, perm[i]);
        solve::essential_solver solver(bear_1, bear_2p, matches_12);
        solver.find_via_ransac(50);
        const Mat33_t E = solver.get_best_E_21();
        double Ef[9];
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 3; ++k) Ef[3 * r + k] = E(r, k);
        const std::vector<bool> inl = solver.get_inlier_matches();
        const int num_in = static_cast<int>(std::count(inl.begin(), inl.end(), true));
        std::printf("essential solver: valid %d, %d of %d inliers (hypothesis %d), max |E - E_true| = %.2e\n", solver.solution_is_valid() ? 1 : 0,
                    num_in, N, solver.best_solution().best_iter, E_error(Ef));
        if (!solver.solution_is_valid() || inl.size() != static_cast<std::size_t>(N) || num_in != N || E_error(Ef) > 1e-9) return 1;

        // 2. robust::match_frame_and_keyframe: the keyframe (camera 2) holds the landmarks, the frame (camera 1) the same descriptors
        //    in the order perm
        camera::perspective cam{camera::setup_type_t::Monocular, 640, 480, 500.0, 500.0, 320.0, 240.0, 0.0};
        keyframe_with_bearings kf(7, &cam);
        frame_with_bearings frm;
        frm.camera_ = &cam;
        kf.num_keypts_ = frm.num_keypts_ = N;
        kf.descriptors_ = cv::Mat(N, 32, CV_8U);
        frm.descriptors_ = cv::Mat(N, 32, CV_8U);
        std::vector<std::unique_ptr<data::landmark>> lms;
        for (int j = 0; j < N; ++j) {
            for (int b = 0; b < 32; ++b) kf.descriptors_.ptr(j)[b] = static_cast<unsigned char>(rng() & 0xff);
            lms.emplace_back(new data::landmark(static_cast<unsigned>(j), Vec3_t{}));
            kf.add_landmark(lms.back().get(), static_cast<unsigned>(j));
        }
        kf.bearings_ = bear_2;
        frm.bearings_.resize(N);
        for (int j = 0; j < N; ++j) {   // frame keypoint perm[j] is keyframe keypoint j
            std::memcpy(frm.descriptors_.ptr(perm[j]), kf.descriptors_.ptr(j), 32);
            frm.bearings_[perm[j]] = bear_1[j];
        }
        match::robust matcher(0.8, false);
        std::vector<data::landmark*> matched;
        const unsigned int num = matcher.match_frame_and_keyframe(frm, &kf, matched);
        int right = 0;
        for (int j = 0; j < N; ++j) right += matched.at(perm[j]) == lms[j].get() ? 1 : 0;
        std::printf("robust match_frame_and_keyframe: %u inlier matches, %d of %d frame keypoints hold their own landmark\n", num, right, N);
        if (num != static_cast<unsigned int>(N) || right != N || matched.size() != static_cast<std::size_t>(N)) return 1;

        // 3. 6 problems (different lengths and seeds; problem 2 has 7 matches) in one batched call equal 6 single calls, bit for bit
        std::vector<double> f1, f2;
        for (int i = 0; i < N; ++i)
            for (int k = 0; k < 3; ++k) { f1.push_back(bear_1[i](k)); f2.push_back(bear_2[i](k)); }
        std::vector<solve::essential_solver::problem_view> probs(6);
        for (int b = 0; b < 6; ++b) {
            const int off = 9 * b, n = b == 2 ? 7 : N - 20 * b;
            probs[b].num_matches = n;
            probs[b].bearings_1 = f1.data() + 3 * off; probs[b].bearings_2 = f2.data() + 3 * off;
            probs[b].seed = 500 + b;
        }
        solve::essential_solver batch;
        const auto all = batch.find_via_ransac(probs, 50, true);
        for (int b = 0; b < 6; ++b) {
            const auto one = batch.find_via_ransac(std::vector<solve::essential_solver::problem_view>{probs[b]}, 50, true).front();
            const auto& o = all[b];
            std::printf("problem %d: valid %d, %u inliers, hypothesis %d\n", b, o.valid ? 1 : 0, o.num_inliers, o.best_iter);
            if (o.valid != one.valid || o.num_inliers != one.num_inliers || o.best_iter != one.best_iter || o.is_inlier != one.is_inlier ||
                std::memcmp(o.E_21, one.E_21, sizeof(o.E_21)) != 0 || std::memcmp(&o.best_score, &one.best_score, sizeof(double)) != 0)
                return 1;
            if ((b == 2) == o.valid) return 1;
        }
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("essential solver ok\n");
    return 0;
}
