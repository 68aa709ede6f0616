// tests/cpp/test_graph_optimizer.cpp -- openvslam::optimize::graph_optimizer of the C++ class layer against ground truth: 24
// keyframes on a circle, exact relative Sim3 measurements (parents, covisibilities, the loop edge), a start with a drifted
// rotation, translation and scale.  The optimised vertices must return to the truth.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "openvslam_b200/openvslam_b200.hpp"

namespace {
// S = {R about y by a, t, s}
void make(double a, const double* t, double s, double* S) {
    const double c = std::cos(a), sn = std::sin(a);
    const double R[9] = {c, 0, sn, 0, 1, 0, -sn, 0, c};
    for (int k = 0; k < 9; ++k) S[k] = R[k];
    for (int k = 0; k < 3; ++k) S[9 + k] = t[k];
    S[12] = s;
}
void compose(const double* A, const double* B, double* O) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
    for (int i = 0; i < 3; ++i) O[9 + i] = A[12] * (A[3 * i] * B[9] + A[3 * i + 1] * B[10] + A[3 * i + 2] * B[11]) + A[9 + i];
    O[12] = A[12] * B[12];
}
void inverse(const double* S, double* O) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O[3 * i + j] = S[3 * j + i];
    for (int k = 0; k < 3; ++k) O[9 + k] = -(S[k] * S[9] + S[3 + k] * S[10] + S[6 + k] * S[11]) / S[12];
    O[12] = 1.0 / S[12];
}
}  // namespace

int main() {
    using namespace openvslam;
    const int K = 24;
    std::vector<double> truth(13 * K), start(13 * K);
    for (int k = 0; k < K; ++k) {
        const double a = 2 * M_PI * k / K;
        const double t[3] = {5 * std::cos(a), 0.1 * k, 5 * std::sin(a)};
        make(a, t, 1.0, &truth[13 * k]);
    }
    for (int q = 0; q < 13; ++q) start[q] = truth[q];   // keyframe 0 (fixed) is exact
    for (int k = 1; k < K; ++k) {
        const double a = 2 * M_PI * k / K;
        const double t[3] = {5 * std::cos(a) + 0.02 * k, 0.1 * k - 0.01 * k, 5 * std::sin(a) + 0.015 * k};
        make(a + 0.004 * k, t, 1.0 + 0.01 * k, &start[13 * k]);
    }
    std::vector<std::int32_t> ei, ej;
    for (int k = 0; k + 1 < K; ++k) { ei.push_back(k); ej.push_back(k + 1); }
    for (int k = 0; k + 2 < K; ++k) { ei.push_back(k + 2); ej.push_back(k); }
    ei.push_back(K - 1); ej.push_back(0);
    const int E = static_cast<int>(ei.size());
    std::vector<double> meas(13 * E);
    for (int e = 0; e < E; ++e) {
        double inv_i[13];
        inverse(&truth[13 * ei[e]], inv_i);
        compose(&truth[13 * ej[e]], inv_i, &meas[13 * e]);   // S_ji = S_j S_i^-1
    }
    std::vector<std::uint8_t> fixed(K, 0);
    fixed[0] = 1;
    std::vector<double> pose(12 * K);
    try {
        optimize::graph_optimizer opt(false);
        opt.optimize(K, start.data(), fixed.data(), E, ei.data(), ej.data(), meas.data(), 0, nullptr, nullptr, pose.data());
        double err = 0;
        for (int k = 0; k < 13 * K; ++k) err = std::fmax(err, std::fabs(start[k] - truth[k]));
        std::printf("graph optimiser: max |S - S_true| = %.2e\n", err);
        if (!(err < 1e-8)) return 1;
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return std::string(e.what()).find("no CPU fallback") != std::string::npos || std::string(e.what()).find("sm_90a") != std::string::npos ? 2 : 1;
    }
    std::printf("graph optimizer ok\n");
    return 0;
}
