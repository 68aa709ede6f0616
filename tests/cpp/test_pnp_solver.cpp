// tests/cpp/test_pnp_solver.cpp -- openvslam::solve::pnp_solver through the adapter with the reference's own signature
// (include/openvslam_b200/adapters.hpp) against ground truth: a synthetic frame at a known pose, 200 noise-free bearings of which
// 50 are matched to wrong landmarks.  Then a batch of 8 candidates through the class layer against the per-candidate calls.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "openvslam_b200/adapters.hpp"

int main() {
    using namespace openvslam;
    // cam_pose_cw: rotation of 0.3 rad about (1, 2, 2) / 3, t = (0.2, -0.4, 1.0)
    const double th = 0.3, ax[3] = {1.0 / 3, 2.0 / 3, 2.0 / 3}, c = std::cos(th), s = std::sin(th);
    double pose_true[12];
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) {
            const double K[9] = {0, -ax[2], ax[1], ax[2], 0, -ax[0], -ax[1], ax[0], 0};
            double KK = 0;
            for (int m = 0; m < 3; ++m) KK += K[3 * r + m] * K[3 * m + k];
            pose_true[3 * r + k] = (r == k ? 1.0 : 0.0) + s * K[3 * r + k] + (1 - c) * KK;
        }
    pose_true[9] = 0.2; pose_true[10] = -0.4; pose_true[11] = 1.0;
    std::vector<float> scale_factors;
    float sf = 1.0f;
    for (int l = 0; l < 8; ++l) { scale_factors.push_back(sf); sf *= 1.2f; }
    const int N = 200, num_wrong = 50;
    std::mt19937 rng(11);
    std::uniform_real_distribution<double> u(-1, 1);
    // the reference's eigen_alloc_vector<Vec3_t> is a std::vector with Eigen's aligned allocator; the stand-in Vec3_t needs none
    std::vector<Vec3_t> bearings, points;
    std::vector<cv::KeyPoint> keypts;
    for (int i = 0; i < N; ++i) {
        const double z = 4.0 + 2.0 * u(rng);
        double pc[3] = {0.8 * z * u(rng), 0.6 * z * u(rng), z};
        const double L = std::sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
        Vec3_t b, pw;
        for (int k = 0; k < 3; ++k) b(k) = pc[k] / L;
        // a wrong landmark: its camera-frame point moved sideways by 0.5 to 0.9 of its depth, far outside every bound
        if (i % 4 == 1) { pc[0] += (0.7 + 0.2 * u(rng)) * z * (pc[0] > 0 ? -1.0 : 1.0); pc[1] += 0.3 * z; }
        // p_w = R^T (p_c - t)
        for (int k = 0; k < 3; ++k) {
            double v = 0;
            for (int m = 0; m < 3; ++m) v += pose_true[3 * m + k] * (pc[m] - pose_true[9 + m]);
            pw(k) = v;
        }
        cv::KeyPoint kp;
        kp.octave = i % 8;
        bearings.push_back(b); points.push_back(pw); keypts.push_back(kp);
    }
    try {
        solve::pnp_solver solver(bearings, keypts, points, scale_factors, 10);
        solver.find_via_ransac(30);
        const Mat33_t R = solver.get_best_rotation();
        const Vec3_t t = solver.get_best_translation();
        const Mat44_t T = solver.get_best_cam_pose();
        const std::vector<bool> flags = solver.get_inlier_flags();
        double err = 0;
        for (int r = 0; r < 3; ++r) {
            err = std::fmax(err, std::fabs(t(r) - pose_true[9 + r]));
            err = std::fmax(err, std::fabs(T(r, 3) - pose_true[9 + r]));
            for (int k = 0; k < 3; ++k) err = std::fmax(err, std::fmax(std::fabs(R(r, k) - pose_true[3 * r + k]), std::fabs(T(r, k) - R(r, k))));
        }
        int wrong_kept = 0, right_kept = 0;
        for (int i = 0; i < N; ++i) (i % 4 == 1 ? wrong_kept : right_kept) += flags[i] ? 1 : 0;
        std::printf("pnp solver: valid %d, %u of %d inliers (hypothesis %d), %d wrong kept, max |pose - pose_true| = %.2e\n",
                    solver.solution_is_valid() ? 1 : 0, solver.best_solution().num_inliers, N, solver.best_solution().best_iter, wrong_kept, err);
        if (!solver.solution_is_valid() || flags.size() != static_cast<std::size_t>(N) || wrong_kept != 0 || right_kept != N - num_wrong ||
            err > 1e-9)
            return 1;
        // 8 candidates (different lengths and seeds) in one batched call equal 8 single calls, bit for bit
        std::vector<double> bflat, pflat;
        std::vector<float> sflat;
        for (int i = 0; i < N; ++i) {
            for (int k = 0; k < 3; ++k) { bflat.push_back(bearings[i](k)); pflat.push_back(points[i](k)); }
            sflat.push_back(scale_factors[static_cast<std::size_t>(keypts[i].octave)]);
        }
        std::vector<solve::pnp_solver::problem_view> probs(8);
        for (int b = 0; b < 8; ++b) {
            const int off = 7 * b, n = b == 3 ? 5 : N - 9 * b;       // candidate 3 is too small to run
            probs[b].num_corrs = n;
            probs[b].bearings = bflat.data() + 3 * off; probs[b].pos_w = pflat.data() + 3 * off; probs[b].scale_factor = sflat.data() + off;
            probs[b].seed = 1000 + b;
        }
        solve::pnp_solver batch(10);
        const auto all = batch.find_via_ransac(probs, 30, true);
        for (int b = 0; b < 8; ++b) {
            const auto one = batch.find_via_ransac(std::vector<solve::pnp_solver::problem_view>{probs[b]}, 30, true).front();
            const auto& o = all[b];
            std::printf("candidate %d: valid %d, %u inliers, hypothesis %d\n", b, o.valid ? 1 : 0, o.num_inliers, o.best_iter);
            if (o.valid != one.valid || o.num_inliers != one.num_inliers || o.best_iter != one.best_iter || o.is_inlier != one.is_inlier ||
                std::memcmp(o.pose_cw, one.pose_cw, sizeof(o.pose_cw)) != 0)
                return 1;
            if ((b == 3) == o.valid) return 1;
        }
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("pnp solver ok\n");
    return 0;
}
