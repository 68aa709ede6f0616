// tests/cpp/test_transform_optimizer.cpp -- openvslam::optimize::transform_optimizer of the C++ class layer against ground
// truth: two keyframes related by a known Sim3 (scale 1.4), 200 correspondences of which 20 are wrong, a perturbed start.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "openvslam_b200/openvslam_b200.hpp"

int main() {
    using namespace openvslam;
    const ovs_camera cam{OVS_CAMERA_PERSPECTIVE, 500, 500, 320, 240, 0, 640, 480};
    // S_12: rotation of 0.1 rad about y, t = (0.3, -0.1, 0.2), s = 1.4
    const double c = std::cos(0.1), s = std::sin(0.1);
    const double S_true[13] = {c, 0, s, 0, 1, 0, -s, 0, c, 0.3, -0.1, 0.2, 1.4};
    const double pose_1w[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    const double pose_2w[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0.5, 0, -0.2};
    const int N = 200, num_wrong = 20;
    std::mt19937 rng(11);
    std::uniform_real_distribution<double> u(-1, 1);
    std::vector<double> pw1(3 * N), pw2(3 * N);
    std::vector<float> xy1(2 * N), xy2(2 * N), w1(N, 1.0f), w2(N, 1.0f);
    for (int i = 0; i < N; ++i) {
        const double p2[3] = {1.5 * u(rng), 1.0 * u(rng), 5 + 1.5 * u(rng)};   // camera-2 coordinates
        double p1[3];
        for (int r = 0; r < 3; ++r) p1[r] = S_true[12] * (S_true[3 * r] * p2[0] + S_true[3 * r + 1] * p2[1] + S_true[3 * r + 2] * p2[2]) + S_true[9 + r];
        for (int r = 0; r < 3; ++r) { pw1[3 * i + r] = p1[r] - pose_1w[9 + r]; pw2[3 * i + r] = p2[r] - pose_2w[9 + r]; }
        xy1[2 * i] = static_cast<float>(500 * p1[0] / p1[2] + 320 + 0.3 * u(rng));
        xy1[2 * i + 1] = static_cast<float>(500 * p1[1] / p1[2] + 240 + 0.3 * u(rng));
        xy2[2 * i] = static_cast<float>(500 * p2[0] / p2[2] + 320 + 0.3 * u(rng));
        xy2[2 * i + 1] = static_cast<float>(500 * p2[1] / p2[2] + 240 + 0.3 * u(rng));
        if (i < num_wrong) { xy1[2 * i] += 40.0f; xy1[2 * i + 1] -= 30.0f; }
    }
    double S[13];
    for (int k = 0; k < 13; ++k) S[k] = S_true[k];
    S[9] += 0.03; S[10] -= 0.02; S[12] *= 1.03;
    try {
        optimize::transform_optimizer opt(false);
        std::vector<std::uint8_t> inlier;
        const unsigned n = opt.optimize(cam, cam, pose_1w, pose_2w, N, pw1.data(), xy1.data(), w1.data(), pw2.data(), xy2.data(), w2.data(), S,
                                        10.0f, inlier);
        int wrong_kept = 0;
        for (int i = 0; i < num_wrong; ++i) wrong_kept += inlier[i];
        double dt = 0;
        for (int k = 0; k < 3; ++k) dt = std::fmax(dt, std::fabs(S[9 + k] - S_true[9 + k]));
        std::printf("transform optimiser: %u inliers, %d wrong pairs kept, s = %.5f, |dt| = %.2e\n", n, wrong_kept, S[12], dt);
        if (n < 170 || n > static_cast<unsigned>(N - num_wrong) || wrong_kept != 0 || std::fabs(S[12] - 1.4) > 5e-3 || dt > 5e-3) return 1;
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("transform optimizer ok\n");
    return 0;
}
