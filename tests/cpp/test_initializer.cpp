// tests/cpp/test_initializer.cpp -- openvslam::initialize::perspective and initialize::bearing_vector through the class layer and
// through the data::frame adapter (include/openvslam_b200/adapters.hpp).  The frame type below carries the members the adapter
// reads, with the reference's names (the adapter is a template deduced from its arguments).
// Scenes: 600 points at depths 4..10 m, seen from the reference camera (the origin) and a current camera at (R, t), |t| = 0.5 m;
// perspective (K = 500 px, 640 x 480) and equirectangular (1920 x 960); 40 extra unmatched keypoints per view; keypoints
// noise-free up to float rounding, bearings formed from the keypoints.
// Checks: through the adapter both initialisers succeed and recover R within 1e-6, t / |t| within 1e-5 and the triangulated points
// (scaled by 1 / |t|) within 1e-3 relative; the adapter equals the class layer on views flattened here, bit for bit; the batched
// form equals its single calls.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace tin {
using namespace openvslam;

// the members of data::frame the adapter reads (data/frame.h, names as recalled)
struct frame {
    camera::base* camera_ = nullptr;
    std::vector<cv::KeyPoint> undist_keypts_;
    std::vector<Vec3_t> bearings_;
};

struct scene {
    frame ref, cur;
    std::vector<int> ref_matches_with_cur;
    double R[9], t[3];
    std::vector<std::array<double, 3>> X;   // per reference keypoint (zero when unmatched)
};

int fail(const char* what) { std::printf("FAIL: %s\n", what); return 1; }

void rotation(double ax, double ay, double az, double* R) {
    const double th = std::sqrt(ax * ax + ay * ay + az * az), x = ax / th, y = ay / th, z = az / th, c = std::cos(th), s = std::sin(th), C = 1 - c;
    const double M[9] = {c + x * x * C, x * y * C - z * s, x * z * C + y * s, y * x * C + z * s, c + y * y * C, y * z * C - x * s,
                         z * x * C - y * s, z * y * C + x * s, c + z * z * C};
    std::memcpy(R, M, sizeof(M));
}

// keypoint <-> bearing of a camera
void project(const camera::base* cam, const double* p, float* uv) {
    if (cam->model_type_ == camera::model_type_t::Equirectangular) {
        const double L = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
        const double lat = -std::asin(p[1] / L), lon = std::atan2(p[0] / L, p[2] / L);
        uv[0] = (float)(cam->cols_ * (0.5 + lon / (2 * M_PI))); uv[1] = (float)(cam->rows_ * (0.5 - lat / M_PI));
        return;
    }
    auto c = static_cast<const camera::perspective*>(cam);
    uv[0] = (float)(c->fx_ * p[0] / p[2] + c->cx_); uv[1] = (float)(c->fy_ * p[1] / p[2] + c->cy_);
}
Vec3_t bearing(const camera::base* cam, const float* uv) {
    Vec3_t b;
    if (cam->model_type_ == camera::model_type_t::Equirectangular) {
        const double lon = (uv[0] / cam->cols_ - 0.5) * 2 * M_PI, lat = -(uv[1] / cam->rows_ - 0.5) * M_PI;
        b(0) = std::cos(lat) * std::sin(lon); b(1) = -std::sin(lat); b(2) = std::cos(lat) * std::cos(lon);
        return b;
    }
    auto c = static_cast<const camera::perspective*>(cam);
    const double x = (uv[0] - c->cx_) / c->fx_, y = (uv[1] - c->cy_) / c->fy_, n = std::sqrt(x * x + y * y + 1.0);
    b(0) = x / n; b(1) = y / n; b(2) = 1.0 / n;
    return b;
}

scene make_scene(camera::base* cam, unsigned seed) {
    std::mt19937 rng(seed);
    std::uniform_real_distribution<double> u(-1, 1), depth(4, 10), uu(0, 1);
    std::normal_distribution<double> g(0, 1);
    scene s;
    rotation(0.05 + 0.02 * u(rng), -0.04 + 0.02 * u(rng), 0.03, s.R);
    double t[3] = {0.3 + 0.1 * u(rng), -0.2 + 0.1 * u(rng), 0.1 * u(rng)};
    const double tn = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    for (int k = 0; k < 3; ++k) s.t[k] = 0.5 * t[k] / tn;
    const bool equi = cam->model_type_ == camera::model_type_t::Equirectangular;
    const int N = 600, extra = 40;
    s.ref.camera_ = s.cur.camera_ = cam;
    std::vector<std::array<float, 2>> kr, kc;
    std::vector<std::array<double, 3>> X;
    while ((int)X.size() < N) {
        double ray[3];
        if (equi) { for (double& v : ray) v = g(rng); }
        else { ray[0] = 0.55 * u(rng); ray[1] = 0.4 * u(rng); ray[2] = 1.0; }
        const double rn = std::sqrt(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2]), z = depth(rng);
        std::array<double, 3> p{ray[0] / rn * z, ray[1] / rn * z, ray[2] / rn * z};
        double q[3];
        for (int r = 0; r < 3; ++r) q[r] = s.R[3 * r] * p[0] + s.R[3 * r + 1] * p[1] + s.R[3 * r + 2] * p[2] + s.t[r];
        if (!equi && q[2] <= 0.5) continue;
        std::array<float, 2> a, b;
        project(cam, p.data(), a.data()); project(cam, q, b.data());
        if (!equi && (b[0] < 0 || b[0] > 640 || b[1] < 0 || b[1] > 480)) continue;
        X.push_back(p); kr.push_back(a); kc.push_back(b);
    }
    for (int e = 0; e < extra; ++e) {
        kr.push_back({(float)(uu(rng) * cam->cols_), (float)(uu(rng) * cam->rows_)});
        kc.push_back({(float)(uu(rng) * cam->cols_), (float)(uu(rng) * cam->rows_)});
    }
    // the current view lists its keypoints in reverse order, so that the matches are not the identity
    const int n = N + extra;
    s.ref.undist_keypts_.resize(n); s.cur.undist_keypts_.resize(n);
    s.ref.bearings_.resize(n); s.cur.bearings_.resize(n);
    s.ref_matches_with_cur.assign(n, -1); s.X.assign(n, {0, 0, 0});
    for (int i = 0; i < n; ++i) {
        const int j = n - 1 - i;
        s.ref.undist_keypts_[i].pt.x = kr[i][0]; s.ref.undist_keypts_[i].pt.y = kr[i][1];
        s.cur.undist_keypts_[j].pt.x = kc[i][0]; s.cur.undist_keypts_[j].pt.y = kc[i][1];
        s.ref.bearings_[i] = bearing(cam, kr[i].data()); s.cur.bearings_[j] = bearing(cam, kc[i].data());
        if (i < N) { s.ref_matches_with_cur[i] = j; s.X[i] = X[i]; }
    }
    return s;
}

// the adapter recovers the truth, equals the class layer on hand-flattened views, and the batched form equals its single calls
template <class Init>
int check(camera::base* cam, const char* name) {
    const scene s = make_scene(cam, 7);
    Init init(s.ref, 100, 50, 1.0f, 4.0f);
    if (!init.initialize(s.cur, s.ref_matches_with_cur)) { std::printf("%s: status %d\n", name, init.last_result().status); return fail("initialize"); }
    const Mat33_t R = init.get_rotation_ref_to_cur();
    const Vec3_t t = init.get_translation_ref_to_cur();
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c)
            if (std::fabs(R(r, c) - s.R[3 * r + c]) > 1e-6) return fail("rotation");
        if (std::fabs(t(r) - s.t[r] / 0.5) > 1e-5) return fail("translation");
    }
    const std::vector<Vec3_t> pts = init.get_triangulated_pts();
    const std::vector<bool> flags = init.get_triangulated_flags();
    int n_tri = 0;
    for (std::size_t i = 0; i < flags.size(); ++i) {
        if (!flags[i]) continue;
        if (s.ref_matches_with_cur[i] < 0) return fail("an unmatched keypoint triangulated");
        ++n_tri;
        double e = 0, nx = 0;
        for (int r = 0; r < 3; ++r) { const double x = s.X[i][r] / 0.5; e += (pts[i](r) - x) * (pts[i](r) - x); nx += x * x; }
        if (std::sqrt(e / nx) > 1e-3) return fail("point");
    }
    if (n_tri < 540) return fail("too few triangulated points");

    // the class layer on views flattened here, with the adapter's seed
    std::vector<ovs_keypoint> kr(s.ref.undist_keypts_.size()), kc(s.cur.undist_keypts_.size());
    std::vector<double> br, bc;
    for (std::size_t i = 0; i < kr.size(); ++i) { kr[i].x = s.ref.undist_keypts_[i].pt.x; kr[i].y = s.ref.undist_keypts_[i].pt.y; }
    for (std::size_t i = 0; i < kc.size(); ++i) { kc[i].x = s.cur.undist_keypts_[i].pt.x; kc[i].y = s.cur.undist_keypts_[i].pt.y; }
    for (const auto& b : s.ref.bearings_) for (int k = 0; k < 3; ++k) br.push_back(b(k));
    for (const auto& b : s.cur.bearings_) for (int k = 0; k < 3; ++k) bc.push_back(b(k));
    const ovs_init_view vr{adapters::to_camera(cam), (std::int32_t)kr.size(), kr.data(), br.data()};
    const ovs_init_view vc{adapters::to_camera(cam), (std::int32_t)kc.size(), kc.data(), bc.data()};
    Init flat(vr, 100, 50, 1.0f, 4.0f);
    const std::uint64_t seed = adapters::init_seed(vr, vc, s.ref_matches_with_cur);
    if (!flat.initialize(vc, s.ref_matches_with_cur, seed)) return fail("class layer");
    if (std::memcmp(&flat.last_result(), &init.last_result(), sizeof(ovs_init_result)) != 0) return fail("class layer != adapter (record)");
    if (flat.triangulated_pts() != init.triangulated_pts() || flat.triangulated_flags() != init.triangulated_flags())
        return fail("class layer != adapter (points)");

    // the batched form against single calls: the scene, a second scene and the scene with half its matches
    const scene s2 = make_scene(cam, 8);
    std::vector<ovs_keypoint> kr2(s2.ref.undist_keypts_.size()), kc2(s2.cur.undist_keypts_.size());
    std::vector<double> br2, bc2;
    for (std::size_t i = 0; i < kr2.size(); ++i) { kr2[i].x = s2.ref.undist_keypts_[i].pt.x; kr2[i].y = s2.ref.undist_keypts_[i].pt.y; }
    for (std::size_t i = 0; i < kc2.size(); ++i) { kc2[i].x = s2.cur.undist_keypts_[i].pt.x; kc2[i].y = s2.cur.undist_keypts_[i].pt.y; }
    for (const auto& b : s2.ref.bearings_) for (int k = 0; k < 3; ++k) br2.push_back(b(k));
    for (const auto& b : s2.cur.bearings_) for (int k = 0; k < 3; ++k) bc2.push_back(b(k));
    const ovs_init_view vr2{adapters::to_camera(cam), (std::int32_t)kr2.size(), kr2.data(), br2.data()};
    const ovs_init_view vc2{adapters::to_camera(cam), (std::int32_t)kc2.size(), kc2.data(), bc2.data()};
    std::vector<int> half = s.ref_matches_with_cur;
    for (std::size_t i = 0; i < half.size(); i += 2) half[i] = -1;
    const std::vector<initialize::base::problem> probs{{&vr, &vc, s.ref_matches_with_cur, 3}, {&vr2, &vc2, s2.ref_matches_with_cur, 4},
                                                      {&vr, &vc, half, 5}};
    std::vector<initialize::base::result> batch;
    flat.initialize(probs, batch);
    for (std::size_t b = 0; b < probs.size(); ++b) {
        std::vector<initialize::base::result> one;
        flat.initialize(std::vector<initialize::base::problem>{probs[b]}, one);
        if (std::memcmp(&one[0].record, &batch[b].record, sizeof(ovs_init_result)) != 0 ||
            one[0].is_triangulated != batch[b].is_triangulated || one[0].triangulated_pts != batch[b].triangulated_pts)
            return fail("batch != single calls");
        if (batch[b].record.status != OVS_INIT_OK) return fail("batch problem not initialised");
    }
    std::printf("%s ok: model %d, %d points triangulated\n", name, init.last_result().model, n_tri);
    return 0;
}
}  // namespace tin

int main() {
    using namespace openvslam;
    {
        ovs_matcher* probe = nullptr;
        const int rc = ovs_matcher_create(0, &probe);
        if (rc == OVS_ERR_NO_DEVICE) { std::printf("no GPU\n"); return 2; }
        if (rc != OVS_OK) return tin::fail("matcher");
        ovs_matcher_destroy(probe);
    }
    camera::perspective persp(camera::setup_type_t::Monocular, 640, 480, 500, 500, 320, 240, 0.0);
    camera::equirectangular equi(1920, 960);
    int rc = tin::check<initialize::perspective>(&persp, "perspective");
    if (rc == 0) rc = tin::check<initialize::bearing_vector>(&equi, "bearing_vector");
    return rc;
}
