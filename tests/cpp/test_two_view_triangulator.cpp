// tests/cpp/test_two_view_triangulator.cpp -- openvslam::module::two_view_triangulator through the class layer and through the
// create_new_landmarks adapter on keyframes of the reference's data model (include/openvslam_b200/adapters.hpp).  The keyframe type
// below carries the members the adapter reads, with the reference's names (the adapter is a template deduced from its arguments).
// Scene: 900 points at depths 4..20 m seen by keyframe 1 and five neighbours (perspective, K = 500 px, 640 x 480, half the keypoints
// stereo with a 0.5 m baseline), keypoints noise-free up to float rounding, one descriptor and one vocabulary node per point.
// Checks: every record pairs the two views of one point and lies within 1e-3 (relative) of it; no keyframe-1 keypoint gets two
// landmarks; the adapter equals the class layer on views flattened here; the records of the first two neighbours are the prefix of
// the five-neighbour call; a batch of triangulate problems equals the per-problem calls of the reference-shaped object.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace tvt {
using namespace openvslam;

// the members of data::keyframe the adapter reads (data/keyframe.h, names as recalled)
struct keyframe {
    camera::base* camera_ = nullptr;
    unsigned int num_keypts_ = 0;
    std::vector<cv::KeyPoint> undist_keypts_;
    std::vector<Vec3_t> bearings_;
    std::vector<float> stereo_x_right_, depths_;
    cv::Mat descriptors_;
    float scale_factor_ = 1.2f;
    std::vector<float> scale_factors_, level_sigma_sq_;
    std::map<unsigned int, std::vector<unsigned int>> bow_feat_vec_;   // DBoW2::FeatureVector
    Mat44_t pose_ = Mat44_t::Identity();
    std::vector<data::landmark*> landmarks_;
    std::vector<int> point_of_keypt;                                    // test bookkeeping
    Mat44_t get_cam_pose() const { return pose_; }
    std::vector<data::landmark*> get_landmarks() const { return landmarks_; }
};

int fail(const char* what) { std::printf("FAIL: %s\n", what); return 1; }
}  // namespace tvt

int main() {
    using namespace openvslam;
    using tvt::fail;
    {
        ovs_matcher* probe = nullptr;
        const int rc = ovs_matcher_create(0, &probe);
        if (rc == OVS_ERR_NO_DEVICE) { std::printf("no GPU\n"); return 2; }
        if (rc != OVS_OK) return fail("matcher");
        ovs_matcher_destroy(probe);
    }
    const double fx = 500, cx = 320, cy = 240, base_m = 0.5;
    camera::perspective cam(camera::setup_type_t::Stereo, 640, 480, fx, fx, cx, cy, fx * base_m);
    std::mt19937 rng(11);
    std::uniform_real_distribution<double> ux(-8, 8), uy(-5, 5), uz(4, 20), un(0, 1);
    const int N = 900;
    std::vector<std::array<double, 3>> X(N);
    for (auto& p : X) p = {ux(rng), uy(rng), uz(rng)};
    std::vector<std::array<unsigned char, 32>> desc(N);
    for (auto& d : desc) for (auto& c : d) c = static_cast<unsigned char>(rng() & 0xff);
    std::vector<float> sf(8), sig(8);
    sf[0] = 1.0f;
    for (int l = 1; l < 8; ++l) sf[l] = sf[l - 1] * 1.2f;
    for (int l = 0; l < 8; ++l) sig[l] = sf[l] * sf[l];
    data::landmark* some_landmark = reinterpret_cast<data::landmark*>(&cam);   // only compared with nullptr

    auto make = [&](double cx_m, double yaw, bool with_landmarks) {
        tvt::keyframe k;
        k.camera_ = &cam;
        k.scale_factors_ = sf; k.level_sigma_sq_ = sig;
        const double c = std::cos(yaw), s = std::sin(yaw);
        const double R[9] = {c, 0, s, 0, 1, 0, -s, 0, c};
        const double C[3] = {cx_m, 0.02 * cx_m, 0.05 * cx_m};
        for (int r = 0; r < 3; ++r) {
            for (int q = 0; q < 3; ++q) k.pose_(r, q) = R[3 * r + q];
            k.pose_(r, 3) = -(R[3 * r] * C[0] + R[3 * r + 1] * C[1] + R[3 * r + 2] * C[2]);
        }
        std::vector<int> pts;
        for (int i = 0; i < N; ++i) if (un(rng) < 0.9) pts.push_back(i);
        std::shuffle(pts.begin(), pts.end(), rng);
        for (const int i : pts) {
            double pc[3];
            for (int r = 0; r < 3; ++r) pc[r] = R[3 * r] * X[i][0] + R[3 * r + 1] * X[i][1] + R[3 * r + 2] * X[i][2] + k.pose_(r, 3);
            if (pc[2] < 1.0) continue;
            const float u = static_cast<float>(fx * pc[0] / pc[2] + cx), v = static_cast<float>(fx * pc[1] / pc[2] + cy);
            if (u < 0 || u >= 640 || v < 0 || v >= 480) continue;
            cv::KeyPoint kp;
            kp.pt.x = u; kp.pt.y = v; kp.octave = 0; kp.angle = static_cast<float>(i % 360);
            k.undist_keypts_.push_back(kp);
            Vec3_t b;
            const double bx = (u - cx) / fx, by = (v - cy) / fx, nrm = std::sqrt(bx * bx + by * by + 1.0);
            b(0) = bx / nrm; b(1) = by / nrm; b(2) = 1.0 / nrm;
            k.bearings_.push_back(b);
            const bool st = un(rng) < 0.5;
            k.depths_.push_back(st ? static_cast<float>(pc[2]) : -1.0f);
            k.stereo_x_right_.push_back(st ? static_cast<float>(u - fx * base_m / pc[2]) : -1.0f);
            k.point_of_keypt.push_back(i);
        }
        const int n = static_cast<int>(k.undist_keypts_.size());
        k.num_keypts_ = static_cast<unsigned int>(n);
        k.descriptors_ = cv::Mat(n, 32, CV_8U);
        for (int j = 0; j < n; ++j) {
            std::memcpy(k.descriptors_.ptr(j), desc[k.point_of_keypt[j]].data(), 32);
            k.bow_feat_vec_[static_cast<unsigned int>(k.point_of_keypt[j] % 16)].push_back(static_cast<unsigned int>(j));
        }
        k.landmarks_.assign(static_cast<std::size_t>(n), nullptr);
        if (with_landmarks)
            for (int j = 0; j < n; ++j) if (un(rng) < 0.1) k.landmarks_[j] = some_landmark;
        return k;
    };
    try {
        tvt::keyframe kf1 = make(0.0, 0.0, true);
        std::vector<tvt::keyframe> nb;
        for (int b = 0; b < 5; ++b) nb.push_back(make(0.35 * (b + 1) * (b % 2 ? -1 : 1), 0.02 * (b - 2), false));
        std::vector<tvt::keyframe*> nbp;
        for (auto& k : nb) nbp.push_back(&k);

        module::two_view_triangulator tri(1.0f);
        const std::vector<ovs_new_landmark> rec = tri.create_new_landmarks(&kf1, nbp, false);
        std::vector<int> taken(kf1.num_keypts_, 0);
        int eligible = 0;
        for (unsigned int j = 0; j < kf1.num_keypts_; ++j) eligible += kf1.landmarks_[j] == nullptr;
        for (const auto& r : rec) {
            const int p1 = kf1.point_of_keypt.at(r.idx_1), p2 = nb.at(r.neighbour).point_of_keypt.at(r.idx_2);
            if (p1 != p2) return fail("a record pairs two different points");
            if (kf1.landmarks_[r.idx_1] || taken[r.idx_1]++) return fail("a keyframe-1 keypoint got a second landmark");
            double e = 0, nx = 0;
            for (int c = 0; c < 3; ++c) { e += (r.pos_w[c] - X[p1][c]) * (r.pos_w[c] - X[p1][c]); nx += X[p1][c] * X[p1][c]; }
            if (!(std::sqrt(e / nx) < 1e-3)) return fail("a record's point is off its true position");
        }
        if (static_cast<int>(rec.size()) < eligible / 2) return fail("too few records");

        // the class layer on views flattened here (plain loops, not the adapter's code)
        std::vector<std::vector<ovs_keypoint>> kp(6);
        std::vector<std::vector<double>> bear(6);
        std::vector<std::vector<std::uint8_t>> dsc(6), lm(6);
        std::vector<std::vector<std::int32_t>> node(6);
        std::vector<ovs_keyframe_view> views(6);
        std::vector<tvt::keyframe*> all{&kf1};
        for (auto* k : nbp) all.push_back(k);
        for (int v = 0; v < 6; ++v) {
            tvt::keyframe& k = *all[v];
            const int n = static_cast<int>(k.num_keypts_);
            kp[v].resize(n); bear[v].resize(3 * n); dsc[v].resize(32 * n); lm[v].resize(n); node[v].assign(n, -1);
            for (int j = 0; j < n; ++j) {
                kp[v][j] = ovs_keypoint{k.undist_keypts_[j].pt.x, k.undist_keypts_[j].pt.y, 0, k.undist_keypts_[j].angle, 0, 0, -1};
                for (int c = 0; c < 3; ++c) bear[v][3 * j + c] = k.bearings_[j](c);
                std::memcpy(&dsc[v][32 * j], k.descriptors_.ptr(j), 32);
                lm[v][j] = k.landmarks_[j] != nullptr;
                node[v][j] = k.point_of_keypt[j] % 16;
            }
            ovs_keyframe_view& w = views[v];
            w = ovs_keyframe_view{};
            for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) w.pose_cw[3 * r + c] = k.pose_(r, c); w.pose_cw[9 + r] = k.pose_(r, 3); }
            w.camera = ovs_camera{OVS_CAMERA_PERSPECTIVE, fx, fx, cx, cy, fx * base_m, 640, 480};
            w.true_baseline = fx * base_m / fx; w.scale_factor = 1.2f;
            w.num_scale_levels = 8; w.scale_factors = sf.data(); w.level_sigma_sq = sig.data();
            w.num_keypts = n; w.undist_keypts = kp[v].data(); w.bearings = bear[v].data();
            w.stereo_x_right = k.stereo_x_right_.data(); w.depths = k.depths_.data();
            w.descriptors = dsc[v].data(); w.has_landmark = lm[v].data(); w.bow_node = node[v].data();
        }
        std::vector<std::array<double, 9>> E(5);
        std::vector<std::array<double, 3>> ep(5);
        for (int b = 0; b < 5; ++b) adapters::e12_and_epipole(views[0].pose_cw, views[b + 1].pose_cw, E[b], ep[b]);
        const std::vector<ovs_keyframe_view> nviews(views.begin() + 1, views.end());
        const std::vector<ovs_new_landmark> rec2 = tri.create_new_landmarks(views[0], nviews, E, ep, false);
        if (rec2.size() != rec.size() || (!rec.empty() && std::memcmp(rec.data(), rec2.data(), sizeof(ovs_new_landmark) * rec.size())))
            return fail("the adapter differs from the class layer");

        // prefix rule
        const std::vector<tvt::keyframe*> first2(nbp.begin(), nbp.begin() + 2);
        const std::vector<ovs_new_landmark> rec3 = tri.create_new_landmarks(&kf1, first2, false);
        std::size_t k2 = 0;
        while (k2 < rec.size() && rec[k2].neighbour < 2) ++k2;
        if (rec3.size() != k2 || (k2 && std::memcmp(rec.data(), rec3.data(), sizeof(ovs_new_landmark) * k2)))
            return fail("the first two neighbours' records are not the prefix");

        // a batch of triangulate problems against the reference-shaped per-problem objects
        std::vector<module::two_view_triangulator::problem> probs;
        for (int b = 0; b < 5; ++b) {
            std::map<int, unsigned int> idx2;
            for (unsigned int j = 0; j < nb[b].num_keypts_; ++j) idx2[nb[b].point_of_keypt[j]] = j;
            module::two_view_triangulator::problem pr{&views[0], &views[b + 1], {}};
            for (unsigned int j = 0; j < kf1.num_keypts_; ++j) {
                const auto it = idx2.find(kf1.point_of_keypt[j]);
                if (it != idx2.end()) pr.pairs.emplace_back(j, it->second);
            }
            probs.push_back(pr);
        }
        std::vector<std::vector<std::uint8_t>> valid;
        std::vector<std::vector<double>> pos;
        tri.triangulate(probs, valid, pos);
        int nvalid = 0;
        for (int b = 0; b < 5; ++b) {
            module::two_view_triangulator one(views[0], views[b + 1], 1.0f);
            std::vector<std::uint8_t> v;
            std::vector<double> p;
            one.triangulate(probs[b].pairs, v, p);
            if (v != valid[b] || p.size() != pos[b].size() || (!p.empty() && std::memcmp(p.data(), pos[b].data(), 8 * p.size())))
                return fail("a batch differs from its single calls");
            for (auto x : v) nvalid += x;
        }
        if (nvalid < 1000) return fail("too few valid pairs");
        std::printf("two-view triangulator ok: %zu records, %d valid of the batched pairs\n", rec.size(), nvalid);
    } catch (const std::exception& e) {
        std::printf("FAIL: %s\n", e.what());
        return 1;
    }
    return 0;
}
