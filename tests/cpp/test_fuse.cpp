// tests/cpp/test_fuse.cpp -- mapping_module::fuse_landmark_duplication and match::fuse::replace_duplication through the adapters of
// include/openvslam_b200/adapters.hpp, against a sequential restatement of replace_duplication on the same types that makes one
// single-query library call per landmark with its live descriptor.  The keyframe and landmark types below carry the members the
// adapters read and write, with the reference's names; landmark::replace and compute_descriptor are written as recalled.
// Scene: 240 points 3..15 m in front of a 640 x 480 monocular camera (K = 500 px), seen by the current keyframe and five targets
// within 0.3 m of it.  Each keyframe has a keypoint near the reprojection of the points it sees (a few descriptor bits flipped) and
// clutter.  The points come in six kinds, so that the fusion reaches: a target's duplicate replaced by a current landmark that is
// then queried in later targets (re-queries); a current landmark replaced by another current landmark that a target holds; two
// current landmarks taking the same keypoint of a target; erased and already-observed landmarks; a backward fusion into the
// current keyframe; and a forward replace that removes a backward candidate.
// Both sides run on the same objects at the same addresses (the scene is rebuilt in place), so that the std::unordered_set of the
// backward candidates iterates in the same order.  A scene without duplicates makes exactly 2 library calls.
// Exit codes: 0 ok, 2 no GPU (library reported OVS_ERR_NO_DEVICE), 1 failure.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <unordered_set>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace tfu {
using namespace openvslam;

int fail(const char* what) { std::printf("FAIL: %s\n", what); return 1; }

class keyframe;

// the members of data::landmark that replace_duplication reads and writes (data/landmark.h, names as recalled)
class landmark {
public:
    unsigned id_ = 0;
    bool will_be_erased_ = false;
    std::map<keyframe*, unsigned int> observations_;
    Vec3_t get_pos_in_world() const { return pos_w_; }
    Vec3_t get_obs_mean_normal() const { return mean_normal_; }
    std::pair<float, float> get_unscaled_valid_distances() const { return {min_valid_dist_, max_valid_dist_}; }
    cv::Mat get_descriptor() const { return descriptor_.clone(); }
    bool will_be_erased() const { return will_be_erased_; }
    bool is_observed_in_keyframe(keyframe* kf) const { return observations_.count(kf) != 0; }
    unsigned int num_observations() const { return static_cast<unsigned int>(observations_.size()); }
    void add_observation(keyframe* kf, const unsigned int idx) { observations_[kf] = idx; }
    inline void replace(landmark* lm);
    inline void compute_descriptor();
    // test set-up
    void reset(const unsigned id, const Vec3_t& p, const Vec3_t& n, const float lo, const float hi, const cv::Mat& d) {
        id_ = id; will_be_erased_ = false; observations_.clear(); pos_w_ = p; mean_normal_ = n; min_valid_dist_ = lo; max_valid_dist_ = hi;
        descriptor_ = d.clone();
    }
    cv::Mat descriptor_;
private:
    Vec3_t pos_w_, mean_normal_;
    float min_valid_dist_ = 0.0f, max_valid_dist_ = 0.0f;
};

// the members of data::keyframe that replace_duplication reads and writes (data/keyframe.h)
class keyframe {
public:
    unsigned id_ = 0;
    camera::base* camera_ = nullptr;
    std::vector<cv::KeyPoint> undist_keypts_;
    std::vector<float> stereo_x_right_;
    cv::Mat descriptors_;
    std::vector<float> scale_factors_, inv_level_sigma_sq_;
    unsigned int num_scale_levels_ = 0;
    float log_scale_factor_ = 0.0f;
    std::vector<landmark*> landmarks_;
    Mat44_t cam_pose_cw_ = Mat44_t::Identity();
    Mat44_t get_cam_pose() const { return cam_pose_cw_; }
    Vec3_t get_cam_center() const {
        Vec3_t c;
        for (int i = 0; i < 3; ++i) c(i) = -(cam_pose_cw_(0, i) * cam_pose_cw_(0, 3) + cam_pose_cw_(1, i) * cam_pose_cw_(1, 3) + cam_pose_cw_(2, i) * cam_pose_cw_(2, 3));
        return c;
    }
    std::vector<landmark*> get_landmarks() const { return landmarks_; }
    landmark* get_landmark(const unsigned int idx) const { return landmarks_.at(idx); }
    void add_landmark(landmark* lm, const unsigned int idx) { landmarks_.at(idx) = lm; }
    void replace_landmark(landmark* lm, const unsigned int idx) { landmarks_.at(idx) = lm; }
    void erase_landmark_with_index(const unsigned int idx) { landmarks_.at(idx) = nullptr; }
    bool will_be_erased() const { return false; }
};

// landmark::replace(lm): this is erased; each of its observations moves to lm, or is erased from a keyframe that already observes lm;
// then lm->compute_descriptor()
void landmark::replace(landmark* lm) {
    if (lm->id_ == id_) return;
    const std::map<keyframe*, unsigned int> observations = observations_;
    will_be_erased_ = true;
    observations_.clear();
    for (const auto& kf_idx : observations) {
        keyframe* kf = kf_idx.first;
        if (!lm->is_observed_in_keyframe(kf)) {
            kf->replace_landmark(lm, kf_idx.second);
            lm->add_observation(kf, kf_idx.second);
        } else {
            kf->erase_landmark_with_index(kf_idx.second);
        }
    }
    lm->compute_descriptor();
}

// landmark::compute_descriptor: of the descriptors of its observations, the one with the smallest median Hamming distance to the
// others (first on ties)
void landmark::compute_descriptor() {
    if (will_be_erased_) return;
    std::vector<const unsigned char*> descs;
    for (const auto& kf_idx : observations_) descs.push_back(kf_idx.first->descriptors_.ptr(static_cast<int>(kf_idx.second)));
    if (descs.empty()) return;
    const std::size_t n = descs.size();
    unsigned best_median = ~0u; std::size_t best = 0;
    for (std::size_t i = 0; i < n; ++i) {
        std::vector<unsigned> d(n);
        for (std::size_t j = 0; j < n; ++j) {
            unsigned s = 0;
            for (int b = 0; b < 32; ++b) s += static_cast<unsigned>(__builtin_popcount(descs[i][b] ^ descs[j][b]));
            d[j] = s;
        }
        std::sort(d.begin(), d.end());
        const unsigned median = d[(n - 1) / 2];
        if (median < best_median) { best_median = median; best = i; }
    }
    descriptor_ = cv::Mat(1, 32, CV_8U);
    std::memcpy(descriptor_.data, descs[best], 32);
}

// ------------------------------------------------------------------------------------------------------------- scene
constexpr int kPoints = 240, kTargets = 5, kKeyframes = kTargets + 1;
constexpr int kLandmarks = 2 * kPoints;

struct scene {
    camera::perspective cam{camera::setup_type_t::Monocular, 640, 480, 500.0, 500.0, 320.0, 240.0, 0.0};
    std::vector<landmark> lms = std::vector<landmark>(kLandmarks);   // fixed storage: rebuilt in place, same addresses
    std::vector<keyframe> kfs = std::vector<keyframe>(kKeyframes);   // kfs[0] is the current keyframe
    std::vector<keyframe*> targets;

    // duplicates = false: every point has one landmark (kinds 0, 4 and 5 only)
    void build(const bool duplicates) {
        std::mt19937 rng(11);
        std::uniform_real_distribution<double> u(-1.0, 1.0), uz(3.0, 15.0);
        std::normal_distribution<double> jitter(0.0, 0.3);
        const int L = 8;
        std::vector<float> sf(L), isf(L);
        sf[0] = 1.0f;
        for (int l = 1; l < L; ++l) sf[l] = sf[l - 1] * 1.2f;
        for (int l = 0; l < L; ++l) isf[l] = 1.0f / (sf[l] * sf[l]);
        targets.clear();
        std::vector<std::vector<cv::KeyPoint>> kps(kKeyframes);
        std::vector<std::vector<std::vector<unsigned char>>> kdesc(kKeyframes);
        std::vector<std::vector<landmark*>> slot(kKeyframes);
        for (int k = 0; k < kKeyframes; ++k) {
            keyframe& kf = kfs[k];
            kf.id_ = static_cast<unsigned>(k); kf.camera_ = &cam; kf.num_scale_levels_ = L; kf.log_scale_factor_ = std::log(1.2f);
            kf.scale_factors_ = sf; kf.inv_level_sigma_sq_ = isf;
            kf.cam_pose_cw_ = Mat44_t::Identity();
            if (k > 0) { kf.cam_pose_cw_(0, 3) = -0.06 * k; kf.cam_pose_cw_(1, 3) = 0.02 * k; targets.push_back(&kf); }
        }
        int nl = 0;
        auto new_landmark = [&](const Vec3_t& p, const std::vector<unsigned char>& base) {
            landmark* lm = &lms[static_cast<std::size_t>(nl)];
            const double d = std::sqrt(p(0) * p(0) + p(1) * p(1) + p(2) * p(2));
            Vec3_t n;
            for (int c = 0; c < 3; ++c) n(c) = p(c) / d;
            cv::Mat desc(1, 32, CV_8U);
            std::memcpy(desc.data, base.data(), 32);
            desc.data[rng() % 32] ^= static_cast<unsigned char>(1u << (rng() % 8));
            lm->reset(static_cast<unsigned>(nl), p, n, static_cast<float>(d * 2.0 / std::pow(1.2, 7.0)), static_cast<float>(d * 2.0), desc);
            ++nl;
            return lm;
        };
        // a keypoint of keyframe k near the reprojection of p (nullptr landmark: an empty slot); returns its index
        auto keypoint = [&](const int k, const Vec3_t& p, const std::vector<unsigned char>& base, landmark* lm) {
            const Mat44_t& T = kfs[k].cam_pose_cw_;
            Vec3_t pc;
            for (int r = 0; r < 3; ++r) pc(r) = T(r, 0) * p(0) + T(r, 1) * p(1) + T(r, 2) * p(2) + T(r, 3);
            cv::KeyPoint kp;
            kp.pt.x = static_cast<float>(500.0 * pc(0) / pc(2) + 320.0 + jitter(rng));
            kp.pt.y = static_cast<float>(500.0 * pc(1) / pc(2) + 240.0 + jitter(rng));
            const double d = std::sqrt(pc(0) * pc(0) + pc(1) * pc(1) + pc(2) * pc(2));
            kp.octave = std::max(0, std::min(7, static_cast<int>(std::ceil(std::log(2.0 * std::sqrt(p(0) * p(0) + p(1) * p(1) + p(2) * p(2)) / d) / std::log(1.2)))));
            std::vector<unsigned char> desc = base;
            for (int f = 0; f < 3; ++f) desc[rng() % 32] ^= static_cast<unsigned char>(1u << (rng() % 8));
            kps[k].push_back(kp); kdesc[k].push_back(desc); slot[k].push_back(lm);
            const unsigned idx = static_cast<unsigned>(kps[k].size() - 1);
            if (lm) lm->add_observation(&kfs[k], idx);
            return idx;
        };
        for (int i = 0; i < kPoints; ++i) {
            const double z = uz(rng);
            Vec3_t p;
            p(0) = u(rng) * 0.45 * z; p(1) = u(rng) * 0.35 * z; p(2) = z;
            std::vector<unsigned char> base(32);
            for (auto& b : base) b = static_cast<unsigned char>(rng() & 0xff);
            const int kind = duplicates ? i % 6 : (i % 3 == 0 ? 0 : i % 3 == 1 ? 4 : 5);
            switch (kind) {
                case 0: {   // one landmark in the current keyframe and targets 1, 2 (already observed there); the others see it too
                    landmark* a = new_landmark(p, base);
                    keypoint(0, p, base, a); keypoint(1, p, base, a); keypoint(2, p, base, a);
                    for (int k = 3; k < kKeyframes; ++k) keypoint(k, p, base, nullptr);
                    break;
                }
                case 1: {   // a current landmark and its duplicate in target 1 (equal counts: the duplicate is replaced)
                    landmark* a = new_landmark(p, base);
                    landmark* b = new_landmark(p, base);
                    keypoint(0, p, base, a); keypoint(1, p, base, b);
                    for (int k = 2; k < kKeyframes; ++k) keypoint(k, p, base, nullptr);
                    break;
                }
                case 2: {   // two current landmarks on two keypoints; the second is also in target 2 and replaces the first there
                    landmark* a = new_landmark(p, base);
                    landmark* c = new_landmark(p, base);
                    keypoint(0, p, base, a); keypoint(0, p, base, c); keypoint(2, p, base, c);
                    break;
                }
                case 3: {   // two current landmarks take the same empty keypoint of target 3
                    landmark* a = new_landmark(p, base);
                    landmark* b = new_landmark(p, base);
                    keypoint(0, p, base, a); keypoint(0, p, base, b); keypoint(3, p, base, nullptr);
                    break;
                }
                case 4: {   // a landmark of target 4 only, fused backwards into the current keyframe
                    landmark* a = new_landmark(p, base);
                    keypoint(0, p, base, nullptr); keypoint(4, p, base, a);
                    break;
                }
                default: {  // an erased current landmark
                    landmark* a = new_landmark(p, base);
                    keypoint(0, p, base, a); keypoint(5, p, base, nullptr);
                    a->will_be_erased_ = true;
                    break;
                }
            }
        }
        for (int i = nl; i < kLandmarks; ++i) lms[static_cast<std::size_t>(i)].reset(static_cast<unsigned>(i), Vec3_t(), Vec3_t(), 0, 0, cv::Mat(1, 32, CV_8U));
        for (int k = 0; k < kKeyframes; ++k) {   // clutter
            for (int c = 0; c < 150; ++c) {
                cv::KeyPoint kp;
                kp.pt.x = static_cast<float>(320.0 + 319.0 * u(rng)); kp.pt.y = static_cast<float>(240.0 + 239.0 * u(rng)); kp.octave = static_cast<int>(rng() % 8);
                std::vector<unsigned char> d(32);
                for (auto& b : d) b = static_cast<unsigned char>(rng() & 0xff);
                kps[k].push_back(kp); kdesc[k].push_back(d); slot[k].push_back(nullptr);
            }
            keyframe& kf = kfs[k];
            kf.undist_keypts_ = kps[k];
            kf.stereo_x_right_.clear();
            kf.descriptors_ = cv::Mat(static_cast<int>(kps[k].size()), 32, CV_8U);
            for (std::size_t r = 0; r < kps[k].size(); ++r) std::memcpy(kf.descriptors_.ptr(static_cast<int>(r)), kdesc[k][r].data(), 32);
            kf.landmarks_ = slot[k];
        }
        for (int i = 0; i < nl; ++i) lms[static_cast<std::size_t>(i)].compute_descriptor();
    }

    // every keyframe's landmark array, every landmark's observations, erased flag and descriptor
    std::vector<long long> state() const {
        std::vector<long long> s;
        for (const keyframe& kf : kfs) {
            s.push_back(-7);
            for (const landmark* lm : kf.landmarks_) s.push_back(lm ? static_cast<long long>(lm->id_) : -1);
        }
        for (const landmark& lm : lms) {
            s.push_back(-8); s.push_back(lm.will_be_erased_);
            for (const auto& o : lm.observations_) { s.push_back(o.first->id_); s.push_back(o.second); }
            for (int b = 0; b < 32; ++b) s.push_back(lm.descriptor_.data[b]);
        }
        return s;
    }
};

// What the restatement saw, to show that the scene reaches every branch.
struct reached {
    int survivor_queried_later = 0, replaced_by_current = 0, same_keypoint = 0, erased_skips = 0, observed_skips = 0;
    int removed_candidates = 0;
};

// match::fuse::replace_duplication(keyfrm, landmarks_to_check, margin), one landmark after the other, each with its own library call
template <class Container>
unsigned int replace_duplication_sequential(const match::fuse& fz, keyframe* keyfrm, const Container& landmarks_to_check, const float margin,
                                            reached& R, const std::vector<landmark*>& current, std::vector<landmark*>* survivors) {
    const adapters::fuse_target_arrays tgt(*keyfrm);
    const std::vector<ovs_fuse_target> targets(1, tgt.target);
    std::unordered_set<landmark*> added_here;
    unsigned int num_fused = 0;
    for (landmark* lm : landmarks_to_check) {
        if (!lm) continue;
        if (lm->will_be_erased()) { ++R.erased_skips; continue; }
        if (lm->is_observed_in_keyframe(keyfrm)) { ++R.observed_skips; continue; }
        adapters::fuse_landmark_rows<landmark> row;
        row.add(lm);
        std::vector<std::int32_t> best;
        fz.replace_duplication(targets, row.table(), {0, 1}, {0}, margin, best);
        if (best[0] < 0) continue;
        landmark* lm_in_keyfrm = keyfrm->get_landmark(static_cast<unsigned int>(best[0]));
        if (lm_in_keyfrm) {
            if (!lm_in_keyfrm->will_be_erased()) {
                if (added_here.count(lm_in_keyfrm)) ++R.same_keypoint;
                if (lm->num_observations() < lm_in_keyfrm->num_observations()) {
                    if (std::find(current.begin(), current.end(), lm_in_keyfrm) != current.end()) ++R.replaced_by_current;
                    lm->replace(lm_in_keyfrm);
                } else {
                    lm_in_keyfrm->replace(lm);
                    if (survivors) survivors->push_back(lm);
                }
            }
        } else {
            lm->add_observation(keyfrm, static_cast<unsigned int>(best[0]));
            keyfrm->add_landmark(lm, static_cast<unsigned int>(best[0]));
            added_here.insert(lm);
        }
        ++num_fused;
    }
    return num_fused;
}

void fuse_landmark_duplication_sequential(const match::fuse& fz, keyframe* cur, const std::vector<keyframe*>& targets, const float margin,
                                          reached& R) {
    const std::vector<landmark*> cur_landmarks = cur->get_landmarks();
    std::unordered_set<landmark*> in_targets_before;
    for (keyframe* t : targets) for (landmark* lm : t->get_landmarks()) if (lm && !lm->will_be_erased()) in_targets_before.insert(lm);
    for (std::size_t t = 0; t < targets.size(); ++t) {
        std::vector<landmark*> survivors;
        replace_duplication_sequential(fz, targets[t], cur_landmarks, margin, R, cur_landmarks, &survivors);
        for (landmark* s : survivors)
            for (std::size_t u = t + 1; u < targets.size(); ++u)
                if (!s->will_be_erased() && !s->is_observed_in_keyframe(targets[u])) { ++R.survivor_queried_later; break; }
    }
    std::unordered_set<landmark*> candidates;
    for (keyframe* t : targets)
        for (landmark* lm : t->get_landmarks()) {
            if (!lm || lm->will_be_erased()) continue;
            candidates.insert(lm);
        }
    for (landmark* lm : in_targets_before) R.removed_candidates += lm->will_be_erased() ? 1 : 0;
    replace_duplication_sequential(fz, cur, candidates, margin, R, cur_landmarks, nullptr);
}

}  // namespace tfu

int main() {
    using namespace openvslam;
    using tfu::fail;
    {
        ovs_matcher* probe = nullptr;
        const int rc = ovs_matcher_create(0, &probe);
        if (rc == OVS_ERR_NO_DEVICE) { std::printf("no GPU\n"); return 2; }
        if (rc != OVS_OK) return fail("matcher");
        ovs_matcher_destroy(probe);
    }
    static tfu::scene S;
    const float margin = 3.0f;

    // 1. fuse_landmark_duplication: adapter against the sequential restatement
    S.build(true);
    const std::vector<long long> start = S.state();
    const match::fuse fz(0.6);
    adapters::fuse_landmark_duplication(fz, &S.kfs[0], S.targets, margin);
    const std::vector<long long> got = S.state();
    const unsigned calls = fz.num_device_calls(), requeries = fz.num_requery_calls();
    S.build(true);
    if (S.state() != start) return fail("the scene is not rebuilt identically");
    const match::fuse seq(0.6);
    tfu::reached R;
    tfu::fuse_landmark_duplication_sequential(seq, &S.kfs[0], S.targets, margin, R);
    if (S.state() != got) return fail("fuse_landmark_duplication: end states differ from the sequential restatement");
    if (got == start) return fail("nothing was fused");
    std::printf("fuse_landmark_duplication: %u library calls (%u re-queries) vs %u sequential; reached: survivor queried later %d, replaced by a "
                "current landmark %d, same keypoint %d, erased skips %d, observed skips %d, removed backward candidates %d\n",
                calls, requeries, seq.num_device_calls(), R.survivor_queried_later, R.replaced_by_current, R.same_keypoint, R.erased_skips,
                R.observed_skips, R.removed_candidates);
    if (requeries == 0 || calls != 2 + requeries) return fail("re-query count");
    if (!(R.survivor_queried_later > 0 && R.replaced_by_current > 0 && R.same_keypoint > 0 && R.erased_skips > 0 && R.observed_skips > 0 &&
          R.removed_candidates > 0))
        return fail("the scene does not reach every branch");

    // 2. replace_duplication(keyfrm, landmarks, margin) on its own: return value and end state, with a vector container
    for (int t = 1; t <= 3; ++t) {
        S.build(true);
        const std::vector<tfu::landmark*> cur = S.kfs[0].get_landmarks();
        const match::fuse one(0.6);
        const unsigned n_adapter = one.replace_duplication(&S.kfs[t], cur, margin);
        const std::vector<long long> a = S.state();
        S.build(true);
        tfu::reached R2;
        const unsigned n_seq = tfu::replace_duplication_sequential(seq, &S.kfs[t], cur, margin, R2, cur, nullptr);
        if (n_adapter != n_seq || S.state() != a) return fail("replace_duplication differs from the sequential restatement");
        if (one.num_device_calls() != 1) return fail("replace_duplication: one library call");
        std::printf("replace_duplication into target %d: %u fused\n", t, n_adapter);
    }

    // 3. a scene without duplicates: no replace, so exactly the forward and the backward call
    S.build(false);
    const std::vector<long long> start2 = S.state();
    const match::fuse fz2(0.6);
    adapters::fuse_landmark_duplication(fz2, &S.kfs[0], S.targets, margin);
    const std::vector<long long> got2 = S.state();
    S.build(false);
    tfu::reached R3;
    tfu::fuse_landmark_duplication_sequential(seq, &S.kfs[0], S.targets, margin, R3);
    if (S.state() != got2 || got2 == start2) return fail("scene without duplicates");
    if (fz2.num_device_calls() != 2 || fz2.num_requery_calls() != 0) return fail("a scene without replaces makes 2 library calls");
    std::printf("fuse ok\n");
    return 0;
}
