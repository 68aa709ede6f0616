// tests/cpp/test_tracking_search.cpp -- the tracker's two projection searches through the adapters of
// include/openvslam_b200/adapters.hpp, against the class layer on arrays flattened here.  The frame and landmark types below carry
// the members the adapters read, with the reference's names (the adapters are templates deduced from their arguments); the camera
// is the stand-in camera::perspective of tests/cpp/standin.
// Scene: 3000 landmarks at 2..25 m in front of a 640 x 480 stereo camera (K = 500 px, 0.1 m baseline); the local-map search runs
// on a frame 5 cm along the optical axis, the motion model on a last frame at the origin and a current frame 25 cm forward.  Each frame has a keypoint near the reprojection of
// most landmarks it can observe, at the predicted level, with a few descriptor bits flipped, plus clutter.  Some current-frame
// keypoints already hold a landmark; some last-frame landmarks are outliers.
// Checks: search_local_landmarks writes the same tracking fields and matches as projection::search_local_landmarks on hand-flattened
// arrays and makes the num_observable increments of a hand-written loop; match_current_and_last_frames(curr, last, margin) equals
// the array-view call; at least 95 % of the matches of each are the true correspondences.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace tts {
using namespace openvslam;

int fail(const char* what) { std::printf("FAIL: %s\n", what); return 1; }

// the members of data::landmark the tracking adapters read and write (data/landmark.h, names as recalled); the unscaled valid
// distances are the one accessor INTEGRATION.md adds to the reference
class landmark {
public:
    landmark(const unsigned id, const Vec3_t& pos_w) : id_(id), pos_w_(pos_w) {}
    unsigned id_;
    Vec2_t reproj_in_tracking_;
    float x_right_in_tracking_ = -1.0f;
    bool is_observable_in_tracking_ = false;
    int scale_level_in_tracking_ = 0;
    unsigned int identifier_in_local_lm_search_ = 0;
    bool will_be_erased_ = false;
    Vec3_t get_pos_in_world() const { return pos_w_; }
    Vec3_t get_obs_mean_normal() const { return mean_normal_; }
    std::pair<float, float> get_unscaled_valid_distances() const { return {min_valid_dist_, max_valid_dist_}; }
    cv::Mat get_descriptor() const { return descriptor_.clone(); }
    bool has_observation() const { return true; }
    bool will_be_erased() const { return will_be_erased_; }
    void increase_num_observable(const unsigned int num_observable = 1) { num_observable_ += num_observable; }
    unsigned int get_num_observable() const { return num_observable_; }
    // test set-up (update_normal_and_depth and compute_descriptor in the reference)
    void set_normal_and_depth(const Vec3_t& n, const float min_d, const float max_d) { mean_normal_ = n; min_valid_dist_ = min_d; max_valid_dist_ = max_d; }
    void set_descriptor(const cv::Mat& d) { descriptor_ = d.clone(); }
private:
    Vec3_t pos_w_, mean_normal_;
    float min_valid_dist_ = 0.0f, max_valid_dist_ = 0.0f;
    cv::Mat descriptor_;
    unsigned int num_observable_ = 1;
};

// the members of data::frame the tracking adapters read and write (data/frame.h)
struct frame {
    unsigned int id_ = 0;
    camera::base* camera_ = nullptr;
    unsigned int num_keypts_ = 0;
    std::vector<cv::KeyPoint> undist_keypts_;
    std::vector<float> stereo_x_right_;
    cv::Mat descriptors_;
    std::vector<landmark*> landmarks_;
    std::vector<bool> outlier_flags_;
    std::vector<float> scale_factors_;
    unsigned int num_scale_levels_ = 0;
    float log_scale_factor_ = 0.0f;
    Mat44_t cam_pose_cw_ = Mat44_t::Identity();
    void set_cam_pose(const Mat44_t& T) {
        cam_pose_cw_ = T;
        for (int i = 0; i < 3; ++i) cam_center_(i) = -(T(0, i) * T(0, 3) + T(1, i) * T(1, 3) + T(2, i) * T(2, 3));
    }
    Vec3_t get_cam_center() const { return cam_center_; }
private:
    Vec3_t cam_center_;
};

Mat44_t pose_at(const double z) {
    Mat44_t T = Mat44_t::Identity();
    T(2, 3) = -z;                                  // camera centre at (0, 0, z)
    return T;
}

}  // namespace tts

int main() {
    using namespace openvslam;
    using tts::fail;
    {
        ovs_matcher* probe = nullptr;
        const int rc = ovs_matcher_create(0, &probe);
        if (rc == OVS_ERR_NO_DEVICE) { std::printf("no GPU\n"); return 2; }
        if (rc != OVS_OK) return fail("matcher");
        ovs_matcher_destroy(probe);
    }
    const double fx = 500, cx = 320, cy = 240, base_m = 0.1;
    camera::perspective cam(camera::setup_type_t::Stereo, 640, 480, fx, fx, cx, cy, fx * base_m);
    const double true_baseline = cam.focal_x_baseline_ / fx;   // as the reference's camera constructors store it
    const int L = 8;
    std::vector<float> sf(L);
    sf[0] = 1.0f;
    for (int l = 1; l < L; ++l) sf[l] = sf[l - 1] * 1.2f;
    std::mt19937 rng(7);
    std::uniform_real_distribution<double> ux(-1, 1), uz(2, 25), un(0, 1);
    std::normal_distribution<double> noise(0.0, 0.7);

    const int N = 3000;
    std::vector<std::unique_ptr<tts::landmark>> lms;
    std::vector<tts::landmark*> local;
    for (int i = 0; i < N; ++i) {
        const double z = uz(rng);
        Vec3_t p;
        p(0) = ux(rng) * 0.6 * z; p(1) = ux(rng) * 0.45 * z; p(2) = z;
        lms.emplace_back(new tts::landmark(static_cast<unsigned>(i), p));
        tts::landmark* lm = lms.back().get();
        const double d = std::sqrt(p(0) * p(0) + p(1) * p(1) + p(2) * p(2));
        Vec3_t n;
        for (int k = 0; k < 3; ++k) n(k) = p(k) / d;
        const float max_d = static_cast<float>(d * (0.8 + 2.5 * un(rng)));
        lm->set_normal_and_depth(n, max_d / std::pow(1.2f, 7.0f), max_d);
        cv::Mat desc(1, 32, CV_8U);
        for (int c = 0; c < 32; ++c) desc.ptr(0)[c] = static_cast<unsigned char>(rng() & 0xff);
        lm->set_descriptor(desc);
        if (i % 97 == 0) lm->will_be_erased_ = true;
        local.push_back(lm);
    }

    auto flat = [&](std::vector<double>& pos, std::vector<double>& nrm, std::vector<float>& lo, std::vector<float>& hi, std::vector<std::uint8_t>& desc) {
        pos.assign(3 * N, 0.0); nrm.assign(3 * N, 0.0); lo.assign(N, 0.0f); hi.assign(N, 0.0f); desc.assign(32 * N, 0);
        for (int i = 0; i < N; ++i) {
            const Vec3_t p = local[i]->get_pos_in_world(), n = local[i]->get_obs_mean_normal();
            for (int k = 0; k < 3; ++k) { pos[3 * i + k] = p(k); nrm[3 * i + k] = n(k); }
            const std::pair<float, float> d = local[i]->get_unscaled_valid_distances();
            lo[i] = d.first; hi[i] = d.second;
            std::memcpy(&desc[32 * i], local[i]->get_descriptor().data, 32);
        }
    };
    std::vector<double> pos, nrm;
    std::vector<float> lo, hi;
    std::vector<std::uint8_t> ldesc;
    flat(pos, nrm, lo, hi, ldesc);

    try {
        match::projection matcher(0.8);
        // a frame at camera centre (0, 0, z): keypoints near the landmarks it can observe (device can_observe), plus clutter
        auto make_frame = [&](const unsigned id, const double z, std::vector<int>& truth) {
            tts::frame f;
            f.id_ = id; f.camera_ = &cam;
            f.scale_factors_ = sf; f.num_scale_levels_ = L; f.log_scale_factor_ = std::log(1.2f);
            f.set_cam_pose(tts::pose_at(z));
            const ovs_frame_geometry g = adapters::frame_geometry(f);
            std::vector<std::uint8_t> ok(N);
            std::vector<float> uv(2 * N), xr(N);
            std::vector<std::int32_t> lvl(N);
            matcher.can_observe(g, N, nullptr, pos.data(), nrm.data(), lo.data(), hi.data(), 0.5f, ok.data(), uv.data(), xr.data(), lvl.data());
            truth.clear();
            for (int i = 0; i < N; ++i) {
                if (!ok[i] || un(rng) > 0.8) continue;
                cv::KeyPoint kp;
                kp.pt.x = static_cast<float>(std::min(639.0, std::max(0.0, uv[2 * i] + noise(rng))));
                kp.pt.y = static_cast<float>(std::min(479.0, std::max(0.0, uv[2 * i + 1] + noise(rng))));
                kp.octave = lvl[i]; kp.angle = static_cast<float>(i % 360);
                f.undist_keypts_.push_back(kp);
                f.stereo_x_right_.push_back(un(rng) < 0.5 ? static_cast<float>(xr[i] + 0.3 * noise(rng)) : -1.0f);
                truth.push_back(i);
            }
            for (int c = 0; c < 300; ++c) {
                cv::KeyPoint kp;
                kp.pt.x = static_cast<float>(320 + 319 * ux(rng)); kp.pt.y = static_cast<float>(240 + 239 * ux(rng));
                kp.octave = static_cast<int>(rng() % L); kp.angle = 0;
                f.undist_keypts_.push_back(kp);
                f.stereo_x_right_.push_back(-1.0f);
                truth.push_back(-1);
            }
            const int n = static_cast<int>(f.undist_keypts_.size());
            f.num_keypts_ = static_cast<unsigned>(n);
            f.descriptors_ = cv::Mat(n, 32, CV_8U);
            for (int j = 0; j < n; ++j) {
                unsigned char* d = f.descriptors_.ptr(j);
                if (truth[j] >= 0) std::memcpy(d, &ldesc[32 * truth[j]], 32);
                else for (int c = 0; c < 32; ++c) d[c] = static_cast<unsigned char>(rng() & 0xff);
                for (int b = 0; b < 5; ++b) { const unsigned bit = rng() % 256; d[bit / 8] ^= static_cast<unsigned char>(1u << (bit % 8)); }
            }
            f.landmarks_.assign(n, nullptr);
            f.outlier_flags_.assign(n, false);
            return f;
        };

        // ---------------------------------------------------------------- search_local_landmarks
        std::vector<int> truth;
        tts::frame curr = make_frame(42, 0.05, truth);
        const int n = static_cast<int>(curr.num_keypts_);
        for (int j = 0; j < n; j += 20) if (truth[j] >= 0) curr.landmarks_[j] = local[truth[j]];   // already tracked in this frame
        // the hand-flattened reference: the skip rule, then the class layer's composed call
        std::vector<std::uint8_t> usable(N), has(n, 0), observable(N);
        std::vector<unsigned> tracked(N, 0);
        for (int j = 0; j < n; ++j) if (curr.landmarks_[j]) { has[j] = 1; if (!curr.landmarks_[j]->will_be_erased()) tracked[curr.landmarks_[j]->id_] = 1; }
        for (int i = 0; i < N; ++i) usable[i] = !tracked[i] && !local[i]->will_be_erased();
        std::vector<float> uv(2 * N), xr(N);
        std::vector<std::int32_t> lvl(N), matched;
        const adapters::frame_arrays arrays(curr);
        unsigned num_ref;
        {
            const match::frame_index idx(matcher, arrays.view);
            num_ref = matcher.search_local_landmarks(idx, adapters::frame_geometry(curr), sf, N, usable.data(), pos.data(), nrm.data(), lo.data(), hi.data(),
                                                     ldesc.data(), has.data(), observable.data(), uv.data(), xr.data(), lvl.data(), matched, 5.0f);
        }
        std::vector<unsigned> before(N);
        for (int i = 0; i < N; ++i) before[i] = local[i]->get_num_observable();
        std::vector<tts::landmark*> lm_before = curr.landmarks_;
        const bool found = adapters::search_local_landmarks(matcher, curr, local, 5.0f);
        unsigned num_obs = 0;
        for (int i = 0; i < N; ++i) {
            const tts::landmark* lm = local[i];
            const unsigned want = before[i] + (tracked[i] ? 1u : 0u) + (usable[i] && observable[i] ? 1u : 0u);
            if (lm->get_num_observable() != want) return fail("num_observable increments");
            if (tracked[i] && (lm->is_observable_in_tracking_ || lm->identifier_in_local_lm_search_ != 42)) return fail("frame's own landmark fields");
            if (!usable[i]) continue;
            if (lm->is_observable_in_tracking_ != (observable[i] != 0)) return fail("is_observable_in_tracking_");
            if (!observable[i]) continue;
            ++num_obs;
            if (lm->reproj_in_tracking_(0) != uv[2 * i] || lm->reproj_in_tracking_(1) != uv[2 * i + 1] || lm->x_right_in_tracking_ != xr[i] ||
                lm->scale_level_in_tracking_ != lvl[i])
                return fail("tracking fields");
        }
        if (!found || num_obs == 0) return fail("found_proj_candidate");
        unsigned num_adapter = 0, correct = 0;
        for (int j = 0; j < n; ++j) {
            tts::landmark* want = matched[j] >= 0 ? local[matched[j]] : lm_before[j];
            if (curr.landmarks_[j] != want) return fail("adapter matches differ from the class layer");
            if (matched[j] >= 0) { ++num_adapter; correct += truth[j] == matched[j] ? 1u : 0u; }
        }
        if (num_adapter != num_ref || num_ref < 500) return fail("match count");
        if (correct < 0.95 * num_ref) return fail("fewer than 95 % true local-map matches");
        std::printf("search_local_landmarks: %u observable, %u matches, %u true\n", num_obs, num_ref, correct);

        // ---------------------------------------------------------------- match_current_and_last_frames
        std::vector<int> truth_last, truth_curr;
        tts::frame last = make_frame(41, 0.0, truth_last);
        const int nl = static_cast<int>(last.num_keypts_);
        for (int j = 0; j < nl; ++j) {
            if (truth_last[j] >= 0 && un(rng) < 0.95) last.landmarks_[j] = local[truth_last[j]];
            last.outlier_flags_[j] = un(rng) < 0.05;
        }
        tts::frame curr2 = make_frame(43, 0.25, truth_curr);     // 0.25 m forward of the last frame: more than the 0.1 m baseline
        const int nc = static_cast<int>(curr2.num_keypts_);
        std::vector<std::uint8_t> lu(nl), has2(nc, 0), lds(32 * nl, 0);
        std::vector<double> lpos(3 * nl, 0.0);
        std::vector<std::int32_t> loct(nl);
        std::vector<float> lang(nl);
        for (int j = 0; j < nl; ++j) {
            lu[j] = last.landmarks_[j] && !last.outlier_flags_[j];
            loct[j] = last.undist_keypts_[j].octave; lang[j] = last.undist_keypts_[j].angle;
            if (!lu[j]) continue;
            const Vec3_t p = last.landmarks_[j]->get_pos_in_world();
            for (int k = 0; k < 3; ++k) lpos[3 * j + k] = p(k);
            std::memcpy(&lds[32 * j], last.landmarks_[j]->get_descriptor().data, 32);
        }
        double last_pose[12];
        adapters::to_Rt(last.cam_pose_cw_, last_pose);
        std::vector<std::int32_t> matched2;
        unsigned num2_ref;
        {
            const adapters::frame_arrays arrays2(curr2);
            const match::frame_index idx(matcher, arrays2.view);
            num2_ref = matcher.match_current_and_last_frames_reproject(idx, adapters::frame_geometry(curr2), false, true_baseline, last_pose, sf, nl,
                                                                       lu.data(), lpos.data(), loct.data(), lang.data(), lds.data(), has2.data(),
                                                                       matched2, 20.0f);
        }
        const unsigned num2 = matcher.match_current_and_last_frames(curr2, last, 20.0f);
        if (num2 != num2_ref || num2_ref < 300) return fail("motion-model match count");
        unsigned correct2 = 0;
        for (int j = 0; j < nc; ++j) {
            tts::landmark* want = matched2[j] >= 0 ? last.landmarks_[matched2[j]] : nullptr;
            if (curr2.landmarks_[j] != want) return fail("motion-model adapter differs from the class layer");
            if (want && static_cast<int>(want->id_) == truth_curr[j]) ++correct2;
        }
        if (correct2 < 0.95 * num2) return fail("fewer than 95 % true motion-model matches");
        std::printf("match_current_and_last_frames: %u matches, %u true\n", num2, correct2);
        // the three-argument form makes the reference's own matcher, match::projection(0.8), for the call
        tts::frame curr3 = make_frame(44, 0.05, truth);
        if (!adapters::search_local_landmarks(curr3, local, 5.0f)) return fail("found_proj_candidate (reference's matcher)");
        unsigned num3 = 0, correct3 = 0;
        for (unsigned j = 0; j < curr3.num_keypts_; ++j)
            if (curr3.landmarks_[j]) { ++num3; correct3 += static_cast<int>(curr3.landmarks_[j]->id_) == truth[j] ? 1u : 0u; }
        if (num3 < 500 || correct3 < 0.95 * num3) return fail("matches with the reference's matcher");
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return 1;
    }
    std::printf("tracking search ok\n");
    return 0;
}
