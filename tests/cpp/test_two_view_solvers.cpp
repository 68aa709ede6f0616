// tests/cpp/test_two_view_solvers.cpp -- openvslam::solve::homography_solver and solve::fundamental_solver through the adapters with
// the reference's own signatures (include/openvslam_b200/adapters.hpp) against ground truth: two views (K = 500 px, 640 x 480) of
// 200 noise-free points at a known relative pose, on a plane for H and at depths 4..10 m for F, with 100 unmatched keypoints per
// view.  Each solver must return the true model (up to scale and sign) with every match an inlier.  Then a batch of 6 problems of
// each model through the class layer against the per-problem calls.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <random>
#include <string>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace {
void mul3(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// max |M / |M| -/+ T / |T||, the better sign
double model_error(const double* M, const double* T) {
    double nm = 0, nt = 0, ep = 0, em = 0;
    for (int k = 0; k < 9; ++k) { nm += M[k] * M[k]; nt += T[k] * T[k]; }
    for (int k = 0; k < 9; ++k) {
        ep = std::fmax(ep, std::fabs(M[k] / std::sqrt(nm) - T[k] / std::sqrt(nt)));
        em = std::fmax(em, std::fabs(M[k] / std::sqrt(nm) + T[k] / std::sqrt(nt)));
    }
    return std::fmin(ep, em);
}
}  // namespace

int main() {
    using namespace openvslam;
    const double th = 0.1, ax[3] = {2.0 / 3, -1.0 / 3, 2.0 / 3}, c = std::cos(th), s = std::sin(th);
    const double Kx[9] = {0, -ax[2], ax[1], ax[2], 0, -ax[0], -ax[1], ax[0], 0};
    double R[9], t[3] = {0.3, 0.05, -0.1};
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) {
            double KK = 0;
            for (int m = 0; m < 3; ++m) KK += Kx[3 * r + m] * Kx[3 * m + k];
            R[3 * r + k] = (r == k ? 1.0 : 0.0) + s * Kx[3 * r + k] + (1 - c) * KK;
        }
    const double K[9] = {500, 0, 320, 0, 500, 240, 0, 0, 1}, KI[9] = {1.0 / 500, 0, -320.0 / 500, 0, 1.0 / 500, -240.0 / 500, 0, 0, 1};
    // plane n^T p = d with n = (0, 0, 1), d = 6: H = K (R + t n^T / d) K^-1; F = K^-T [t]x R K^-1
    double A[9], H_true[9], F_true[9], tmp[9];
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) A[3 * r + k] = R[3 * r + k] + (k == 2 ? t[r] / 6.0 : 0.0);
    mul3(K, A, tmp); mul3(tmp, KI, H_true);
    const double T[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0}, KIt[9] = {KI[0], KI[3], KI[6], KI[1], KI[4], KI[7], KI[2], KI[5], KI[8]};
    mul3(T, R, A); mul3(KIt, A, tmp); mul3(tmp, KI, F_true);

    const int N = 200, X = 100;
    std::mt19937 rng(7);
    std::uniform_real_distribution<double> ux(20, 620), uy(20, 460), uz(4, 10);
    auto views = [&](bool planar, std::vector<cv::KeyPoint>& k1, std::vector<cv::KeyPoint>& k2, std::vector<std::pair<int, int>>& m) {
        k1.assign(N + X, cv::KeyPoint{}); k2.assign(N + X, cv::KeyPoint{});
        std::vector<int> perm(N + X);
        std::iota(perm.begin(), perm.end(), 0);
        std::shuffle(perm.begin(), perm.end(), rng);
        m.clear();
        for (int i = 0; i < N + X; ++i) {
            k1[i].pt = cv::Point2f(static_cast<float>(ux(rng)), static_cast<float>(uy(rng)));
            k2[i].pt = cv::Point2f(static_cast<float>(ux(rng)), static_cast<float>(uy(rng)));
        }
        for (int i = 0; i < N; ++i) {
            const double u = ux(rng), v = uy(rng), z = planar ? 6.0 : uz(rng);
            const double p1[3] = {(u - 320) / 500 * z, (v - 240) / 500 * z, z};
            double p2[3];
            for (int r = 0; r < 3; ++r) p2[r] = R[3 * r] * p1[0] + R[3 * r + 1] * p1[1] + R[3 * r + 2] * p1[2] + t[r];
            k1[i].pt = cv::Point2f(static_cast<float>(u), static_cast<float>(v));
            k2[perm[i]].pt = cv::Point2f(static_cast<float>(500 * p2[0] / p2[2] + 320), static_cast<float>(500 * p2[1] / p2[2] + 240));
            m.emplace_back(i, perm[i]);
        }
    };
    try {
        std::vector<cv::KeyPoint> k1, k2;
        std::vector<std::pair<int, int>> m;
        // 1. the reference's constructors
        views(true, k1, k2, m);
        solve::homography_solver hs(k1, k2, m, 1.0f);
        hs.find_via_ransac(100, true);
        const Mat33_t H = hs.get_best_H_21();
        double Hf[9];
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 3; ++k) Hf[3 * r + k] = H(r, k);
        std::vector<bool> inl = hs.get_inlier_matches();
        int num_in = static_cast<int>(std::count(inl.begin(), inl.end(), true));
        std::printf("homography solver: valid %d, %d of %d inliers, score %.3f, max |H - H_true| = %.2e\n", hs.solution_is_valid() ? 1 : 0,
                    num_in, N, hs.get_best_score(), model_error(Hf, H_true));
        if (!hs.solution_is_valid() || num_in != N || model_error(Hf, H_true) > 1e-5 || !(hs.get_best_score() > 0)) return 1;

        views(false, k1, k2, m);
        solve::fundamental_solver fs(k1, k2, m, 1.0f);
        fs.find_via_ransac(100, true);
        const Mat33_t F = fs.get_best_F_21();
        double Ff[9];
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 3; ++k) Ff[3 * r + k] = F(r, k);
        inl = fs.get_inlier_matches();
        num_in = static_cast<int>(std::count(inl.begin(), inl.end(), true));
        std::printf("fundamental solver: valid %d, %d of %d inliers, score %.3f, max |F - F_true| = %.2e\n", fs.solution_is_valid() ? 1 : 0,
                    num_in, N, fs.get_best_score(), model_error(Ff, F_true));
        if (!fs.solution_is_valid() || num_in != N || model_error(Ff, F_true) > 1e-5) return 1;

        // 2. 6 problems per model (different match counts and seeds; problem 2 has 7 matches) in one batched call equal 6 single calls
        std::vector<ovs_keypoint> o1(k1.size()), o2(k2.size());
        std::memcpy(o1.data(), k1.data(), sizeof(ovs_keypoint) * k1.size());
        std::memcpy(o2.data(), k2.data(), sizeof(ovs_keypoint) * k2.size());
        std::vector<std::int32_t> flat;
        for (const auto& p : m) { flat.push_back(p.first); flat.push_back(p.second); }
        std::vector<solve::two_view_solver_base::problem_view> probs(6);
        for (int b = 0; b < 6; ++b) {
            probs[b].num_keypts_1 = static_cast<int>(o1.size()); probs[b].keypts_1 = o1.data();
            probs[b].num_keypts_2 = static_cast<int>(o2.size()) - b; probs[b].keypts_2 = o2.data();
            probs[b].num_matches = b == 2 ? 7 : N - 30 * b;
            probs[b].matches_12 = flat.data() + 18 * b;
            probs[b].seed = 700 + b;
            for (int i = 0; i < probs[b].num_matches; ++i)   // keep every idx_2 inside the shortened view 2
                if (probs[b].matches_12[2 * i + 1] >= probs[b].num_keypts_2) probs[b].num_matches = i;
        }
        solve::homography_solver hb;
        solve::fundamental_solver fb;
        for (int model = 0; model < 2; ++model) {
            const solve::two_view_solver_base& sv = model == 0 ? static_cast<const solve::two_view_solver_base&>(hb) : fb;
            const auto all = sv.find_via_ransac(probs, 100, true);
            for (int b = 0; b < 6; ++b) {
                const auto one = sv.find_via_ransac(std::vector<solve::two_view_solver_base::problem_view>{probs[b]}, 100, true).front();
                const auto& o = all[b];
                std::printf("%s problem %d: %d matches, valid %d, %u inliers, hypothesis %d\n", model == 0 ? "H" : "F", b, probs[b].num_matches,
                            o.valid ? 1 : 0, o.num_inliers, o.best_iter);
                if (o.valid != one.valid || o.num_inliers != one.num_inliers || o.best_iter != one.best_iter || o.is_inlier != one.is_inlier ||
                    std::memcmp(o.M_21, one.M_21, sizeof(o.M_21)) != 0 || std::memcmp(&o.best_score, &one.best_score, sizeof(double)) != 0)
                    return 1;
                if (probs[b].num_matches < 8 && o.valid) return 1;
            }
        }
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("two-view solvers ok\n");
    return 0;
}
