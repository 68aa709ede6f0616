// tests/cpp/test_class_layer.cpp -- compiles the C++ class layer (include/openvslam_b200/openvslam_b200.hpp)
// against libovs_b200.so and, when a GPU is present, runs extract -> brute_force_match ->
// pose_optimizer -> local_bundle_adjuster through the reference's class names.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "openvslam_b200/openvslam_b200.hpp"

int main() {
    using namespace openvslam;
    // synthetic 640x480 image: random rectangles
    const int W = 640, H = 480;
    std::vector<std::uint8_t> img(static_cast<size_t>(W) * H, 110), img2;
    std::mt19937 rng(7);
    for (int r = 0; r < 400; ++r) {
        const int x = rng() % W, y = rng() % H, w = 4 + rng() % 40, h = 4 + rng() % 40, v = 20 + rng() % 216;
        for (int yy = y; yy < std::min(H, y + h); ++yy)
            for (int xx = x; xx < std::min(W, x + w); ++xx) img[static_cast<size_t>(yy) * W + xx] = static_cast<std::uint8_t>(v);
    }
    img2 = img;  // second frame: shifted by 3 px
    for (int y = 0; y < H; ++y)
        for (int x = 3; x < W; ++x) img2[static_cast<size_t>(y) * W + x] = img[static_cast<size_t>(y) * W + x - 3];
    try {
        feature::orb_extractor extractor(feature::orb_params(1000, 1.2f, 8, 20, 7));
        std::vector<ovs_keypoint> kps1, kps2;
        std::vector<std::uint8_t> d1, d2;
        extractor.extract(img.data(), H, W, W, nullptr, 0, kps1, d1);
        extractor.extract(img2.data(), H, W, W, nullptr, 0, kps2, d2);
        std::printf("keypoints: %zu / %zu\n", kps1.size(), kps2.size());
        if (kps1.size() < 500 || d1.size() != kps1.size() * 32) return 1;

        match::robust robust_matcher(0.75f, true);
        std::vector<std::pair<int, int>> matches;
        const unsigned nm = robust_matcher.brute_force_match(d2.data(), static_cast<int>(kps2.size()), d1.data(), static_cast<int>(kps1.size()), nullptr, matches);
        int consistent = 0;
        for (const auto& m : matches) consistent += std::fabs((kps2[m.first].x - kps1[m.second].x) - 3.0f) < 2.5f;
        std::printf("brute-force matches: %u, consistent with the 3 px shift: %d\n", nm, consistent);
        if (nm < 200 || consistent < static_cast<int>(0.7 * nm)) return 1;

        // colour input: util::convert_to_grayscale fused in front of extract -- a BGR image whose channels all equal the
        // gray image converts back to it exactly ((3735 + 19235 + 9798) v + 16384) >> 15 == v
        {
            std::vector<std::uint8_t> bgr(static_cast<size_t>(W) * H * 3);
            for (size_t i = 0; i < img.size(); ++i) bgr[3 * i] = bgr[3 * i + 1] = bgr[3 * i + 2] = img[i];
            std::vector<ovs_keypoint> kc; std::vector<std::uint8_t> dc;
            extractor.extract_color(bgr.data(), H, W, static_cast<size_t>(W) * 3, 3, OVS_COLOR_ORDER_BGR, nullptr, 0, kc, dc);
            std::printf("colour extract: %zu keypoints\n", kc.size());
            if (kc.size() != kps1.size() || dc != d1) return 1;
        }

        // frame index + projection::match_keyframes_mutually: frame 2 is frame 1 shifted by 3 px
        {
            auto view = [&](const std::vector<ovs_keypoint>& k, const std::vector<std::uint8_t>& d, std::vector<float>& x, std::vector<float>& y,
                            std::vector<std::int32_t>& o, std::vector<float>& a) {
                for (const auto& p : k) { x.push_back(p.x); y.push_back(p.y); o.push_back(p.octave); a.push_back(p.angle); }
                match::frame_view v{};
                v.num_keypts = static_cast<int>(k.size()); v.x = x.data(); v.y = y.data(); v.octave = o.data(); v.angle = a.data();
                v.stereo_x_right = nullptr; v.descriptors = d.data();
                v.grid = ovs_grid{0.0f, 0.0f, 64.0f / W, 48.0f / H, 64, 48};
                return v;
            };
            std::vector<float> x1, y1, a1, x2, y2, a2; std::vector<std::int32_t> o1, o2;
            match::projection proj(0.6f, true);
            const match::frame_view v1 = view(kps1, d1, x1, y1, o1, a1), v2 = view(kps2, d2, x2, y2, o2, a2);
            match::frame_index f1(proj, v1), f2(proj, v2);
            std::vector<float> sf(8); sf[0] = 1.0f; for (int l = 1; l < 8; ++l) sf[l] = sf[l - 1] * 1.2f;
            std::vector<float> r12, r21;
            for (const auto& p : kps1) { r12.push_back(p.x + 3.0f); r12.push_back(p.y); }
            for (const auto& p : kps2) { r21.push_back(p.x - 3.0f); r21.push_back(p.y); }
            std::vector<std::int32_t> mutual;
            const unsigned nmut = proj.match_keyframes_mutually(f1, f2, sf, nullptr, r12.data(), o1.data(), d1.data(), nullptr, r21.data(), o2.data(),
                                                                d2.data(), mutual, 7.5f);
            int ok = 0;
            for (size_t i = 0; i < mutual.size(); ++i)
                if (mutual[i] >= 0) ok += std::fabs(kps2[mutual[i]].x - kps1[i].x - 3.0f) < 2.5f;
            std::printf("mutual projection matches: %u, consistent: %d\n", nmut, ok);
            if (nmut < 150 || ok < static_cast<int>(0.8 * nmut)) return 1;
        }

        // pose optimiser: perspective camera, 300 points in front of it, perturbed pose
        ovs_camera cam{OVS_CAMERA_PERSPECTIVE, 500, 500, 320, 240, 0, 640, 480};
        const int N = 300;
        std::vector<double> pw(3 * N); std::vector<float> xy(2 * N), w(N, 1.0f);
        std::uniform_real_distribution<double> u(-1, 1);
        for (int i = 0; i < N; ++i) {
            pw[3 * i] = 2 * u(rng); pw[3 * i + 1] = 1.5 * u(rng); pw[3 * i + 2] = 6 + 2 * u(rng);
            xy[2 * i] = static_cast<float>(500 * pw[3 * i] / pw[3 * i + 2] + 320 + 0.3 * u(rng));
            xy[2 * i + 1] = static_cast<float>(500 * pw[3 * i + 1] / pw[3 * i + 2] + 240 + 0.3 * u(rng));
        }
        double pose[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0.05, -0.03, 0.04};
        optimize::pose_optimizer pose_opt;
        std::vector<std::uint8_t> outliers;
        const unsigned ninl = pose_opt.optimize(cam, true, N, pw.data(), xy.data(), nullptr, w.data(), pose, outliers);
        std::printf("pose optimiser inliers: %u, t = (%.4f %.4f %.4f)\n", ninl, pose[9], pose[10], pose[11]);
        if (ninl < 280 || std::fabs(pose[9]) > 5e-3 || std::fabs(pose[11]) > 5e-3) return 1;

        // local BA: 3 keyframes (1 fixed), same points, noisy initial points
        const int K = 3;
        std::vector<double> poses(12 * K, 0.0), pts = pw;
        std::vector<std::uint8_t> fixed = {0, 0, 1};
        for (int k = 0; k < K; ++k) { poses[12 * k] = poses[12 * k + 4] = poses[12 * k + 8] = 1; poses[12 * k + 9] = -0.3 * k; }
        std::vector<std::int32_t> okf, olm; std::vector<float> oxy, ow;
        for (int i = 0; i < N; ++i)
            for (int k = 0; k < K; ++k) {
                const double x = pw[3 * i] - 0.3 * k, y = pw[3 * i + 1], z = pw[3 * i + 2];
                okf.push_back(k); olm.push_back(i); ow.push_back(1.0f);
                oxy.push_back(static_cast<float>(500 * x / z + 320 + 0.3 * u(rng))); oxy.push_back(static_cast<float>(500 * y / z + 240 + 0.3 * u(rng)));
            }
        for (auto& v : pts) v += 0.05 * u(rng);
        poses[9] += 0.02; poses[12 + 10] -= 0.02;
        auto rms = [&]() {
            double s2 = 0;
            for (size_t o = 0; o < okf.size(); ++o) {
                const double* P = &poses[12 * okf[o]]; const double* X = &pts[3 * olm[o]];
                const double x = P[0] * X[0] + P[1] * X[1] + P[2] * X[2] + P[9], y = P[3] * X[0] + P[4] * X[1] + P[5] * X[2] + P[10],
                             z = P[6] * X[0] + P[7] * X[1] + P[8] * X[2] + P[11];
                const double ex = oxy[2 * o] - (500 * x / z + 320), ey = oxy[2 * o + 1] - (500 * y / z + 240);
                s2 += ex * ex + ey * ey;
            }
            return std::sqrt(s2 / okf.size());
        };
        const double rms0 = rms();
        optimize::local_bundle_adjuster ba;
        std::vector<std::uint8_t> outl;
        bool stop = false;
        ba.optimize(cam, true, K, poses.data(), fixed.data(), N, pts.data(), static_cast<int>(okf.size()), okf.data(), olm.data(), oxy.data(), nullptr,
                    ow.data(), &stop, outl);
        const double rms1 = rms();
        std::printf("local BA: reprojection rms %.3f px -> %.3f px, fixed keyframe tx %.4f\n", rms0, rms1, poses[24 + 9]);
        if (!(rms1 < 0.5 && rms1 < 0.2 * rms0) || poses[24 + 9] != -0.6) return 1;
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("class layer ok\n");
    return 0;
}
