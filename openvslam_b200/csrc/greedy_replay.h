// greedy_replay.h -- the host replay of the reference's sequential "a keypoint goes to its first taker" matchers
// (match::projection, match::area, match::bow_tree, match::robust).  Host code only.
//
// The device returns, per query, its K best candidates as sorted keys (distance << 16 | visiting order, 0xffffffff where
// the list ends), computed before any query has claimed anything.  The host walks the queries in the reference's order
// and decides each one from its list; the candidates claimed by earlier queries are skipped.  Where the list cannot
// decide (its valid entries ran out before the decision was certain), the matcher asks the device again for this one
// query with the claimed candidates excluded ("re-query") and decides on the fresh list for good.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/ovs_b200.h"

namespace ovs {

constexpr unsigned kNoKey = 0xffffffffu;

inline int key_dist(unsigned key) { return key == kNoKey ? OVS_MAX_HAMMING_DIST : (int)(key >> 16); }

// A candidate farther than d_star(lowe_ratio) can neither be an acceptable best (> HAMMING_DIST_THR_LOW) nor make the
// ratio test fail (lowe_ratio * d_star >= THR_LOW >= best): for a matcher with that threshold and an unconditional ratio
// test, a list whose unlisted candidates are all >= d_star is complete for every decision the reference takes.
inline int d_star(float lowe_ratio) {
    int d = OVS_HAMMING_DIST_THR_LOW + 1;
    while (d < OVS_MAX_HAMMING_DIST && lowe_ratio * (float)(unsigned)d < (float)OVS_HAMMING_DIST_THR_LOW) ++d;
    return d + 1;
}

// complete_at for the matchers without the d_star shortcut: no lower bound reaches it
constexpr int kNeverComplete = OVS_MAX_HAMMING_DIST + 1;

// One query's list after the claimed candidates are dropped.
template <int K>
struct ReplayList {
    int r = 0;                               // valid entries
    int dist[K], id[K], pos[K];              // in list order; pos = the entry's place in the key list
    bool exhausted = false;                  // the list ended before K entries: nothing exists beyond it
    int lower_bound = OVS_MAX_HAMMING_DIST;  // every unlisted candidate has distance >= this
};

template <int K, class Decode, class Valid>
ReplayList<K> resolve(const unsigned* keys, Decode&& decode, Valid&& valid) {
    ReplayList<K> L;
    for (int k = 0; k < K; ++k) {
        if (keys[k] == kNoKey) { L.exhausted = true; break; }
        const int id = decode(keys[k]), d = key_dist(keys[k]);
        if (valid(id, d)) { L.dist[L.r] = d; L.id[L.r] = id; L.pos[L.r] = k; ++L.r; }
    }
    L.lower_bound = L.exhausted ? OVS_MAX_HAMMING_DIST : key_dist(keys[K - 1]);
    return L;
}

// What the ratio test of entry 0 is compared against: the second listed entry, the lower bound of the unlisted
// candidates, or nothing (second = OVS_MAX_HAMMING_DIST).  The matchers' tests treat these differently.
enum class Second { listed, bound, none };

enum class Outcome { accept, reject, requery };

// The decision on one resolved list.  ratio(L, second, kind) is true when entry 0 passes the ratio test.
//   r >= 2, or complete (exhausted, lower_bound >= complete_at, or after a re-query):
//       accept entry 0 iff r >= 1, its distance <= thr and it passes against entry 1 (or against none if r < 2)
//   r == 1: re-query iff its distance <= thr and it fails against the lower bound (only the true second can decide);
//       otherwise as above with the lower bound as the second
//   r == 0: re-query iff an unlisted candidate could be within thr (lower_bound <= thr); otherwise reject
template <int K, class Ratio>
Outcome decide(const ReplayList<K>& L, int thr, int complete_at, Ratio&& ratio, bool after_requery) {
    if (L.r >= 2 || L.exhausted || L.lower_bound >= complete_at || after_requery) {
        if (L.r == 0 || L.dist[0] > thr) return Outcome::reject;
        const bool pass = L.r >= 2 ? ratio(L, L.dist[1], Second::listed) : ratio(L, OVS_MAX_HAMMING_DIST, Second::none);
        return pass ? Outcome::accept : Outcome::reject;
    }
    if (L.r == 1) {
        if (L.dist[0] > thr) return Outcome::reject;
        return ratio(L, L.lower_bound, Second::bound) ? Outcome::accept : Outcome::requery;
    }
    return L.lower_bound <= thr ? Outcome::requery : Outcome::reject;
}

// The matchers without a ratio test
constexpr auto no_ratio_test = [](const auto&, int, Second) { return true; };

struct ReplayPick {
    int id = -1;             // the accepted candidate, -1 when the query is rejected
    int dist = 0, pos = -1;  // its distance and its place in the list it came from
    bool requeried = false;  // that list is the re-query's
};

// One query: decide on `keys` (K entries); if that asks for it, requery(fresh) fills fresh[K] with the query's list over
// the unclaimed candidates (and counts the re-query), and the fresh list decides.  Returns requery's error, else OVS_OK.
template <int K, class Decode, class Valid, class Ratio, class Requery>
int replay_query(const unsigned* keys, int thr, int complete_at, Decode&& decode, Valid&& valid, Ratio&& ratio, Requery&& requery,
                 ReplayPick* pick) {
    unsigned fresh[K];
    ReplayList<K> L = resolve<K>(keys, decode, valid);
    Outcome o = decide(L, thr, complete_at, ratio, false);
    const bool requeried = o == Outcome::requery;
    if (requeried) {
        const int rc = requery(fresh);
        if (rc != OVS_OK) return rc;
        L = resolve<K>(fresh, decode, valid);
        o = decide(L, thr, complete_at, ratio, true);
    }
    *pick = ReplayPick{};
    if (o == Outcome::accept) *pick = ReplayPick{L.id[0], L.dist[0], L.pos[0], requeried};
    return OVS_OK;
}

// match::angle_checker<int>(30, 3)::get_invalid_matches over (delta_angle, tag) pairs
inline void angle_checker_invalid(const std::vector<float>& deltas, std::vector<uint8_t>& invalid) {
    const int H = 30, keepn = 3;
    const float inv_len = 1.0f / H;
    std::vector<int> bin(deltas.size()), count(H, 0), order(H);
    for (size_t i = 0; i < deltas.size(); ++i) {
        float d = deltas[i];
        if (d < 0.0) d += 360.0;
        if (360.0 <= d) d -= 360.0;
        bin[i] = (int)((unsigned)lrintf(d * inv_len) % (unsigned)H);
        count[bin[i]]++;
    }
    for (int b = 0; b < H; ++b) order[b] = b;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return count[a] > count[b]; });
    std::vector<uint8_t> keep(H, 0);
    const int top = count[order[0]];
    for (int r = 0; r < keepn; ++r) {
        if (r > 0 && (float)count[order[r]] < 0.1f * (float)top) break;
        keep[order[r]] = 1;
    }
    invalid.resize(deltas.size());
    for (size_t i = 0; i < deltas.size(); ++i) invalid[i] = !keep[bin[i]];
}

// The orientation check of a matcher: add() each accepted match's angle difference and a tag naming the match, then
// unset_invalid(unset) calls unset(tag) for every match outside the dominant rotation bins.
struct OrientationCheck {
    std::vector<float> deltas;
    std::vector<int> tags;
    void add(float delta, int tag) { deltas.push_back(delta); tags.push_back(tag); }
    template <class Unset>
    void unset_invalid(Unset&& unset) const {
        if (deltas.empty()) return;
        std::vector<uint8_t> invalid;
        angle_checker_invalid(deltas, invalid);
        for (size_t k = 0; k < deltas.size(); ++k) if (invalid[k]) unset(tags[k]);
    }
};

}  // namespace ovs
