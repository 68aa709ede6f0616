// Host-compiled shim over csrc/greedy_replay.h for tests/test_greedy_replay.py.  A problem is nq queries over nc candidates:
// dist[q * nc + c] is candidate c's distance to query q (< 0: c is no candidate of q), level[c] its pyramid level, and
// claimed[c] is set when c is unavailable from the start.  The shim's "device" lists a query's exact top-K keys
// (distance << 16 | c, ascending) over its unclaimed candidates: the first lists see only the initial claims, a re-query
// also the candidates taken by earlier queries.
#include <vector>

#include "../../openvslam_b200/csrc/greedy_replay.h"

namespace {

// the matchers' ratio tests: none (match_best, triangulation); unconditional, no second = OVS_MAX_HAMMING_DIST (bow_tree,
// robust, area); only between equal levels against a listed second (match_frame_and_landmarks)
enum { kNoRatio = 0, kRatio = 1, kLevelRatio = 2 };

template <int K>
void top_k(const int* dist, int nc, const std::vector<uint8_t>& claimed, unsigned* keys) {
    for (int k = 0; k < K; ++k) keys[k] = ovs::kNoKey;
    for (int c = 0; c < nc; ++c) {
        if (dist[c] < 0 || claimed[c]) continue;
        unsigned key = ((unsigned)dist[c] << 16) | (unsigned)c;
        for (int k = 0; k < K; ++k)
            if (key < keys[k]) { const unsigned t = keys[k]; keys[k] = key; key = t; }
    }
}

template <int K>
int replay(int nq, int nc, const int* dist, const int* level, const uint8_t* claimed_0, int mode, int thr, int complete_at,
           float lowe_ratio, int* match, int* num_requeries) {
    std::vector<uint8_t> claimed(claimed_0, claimed_0 + nc);
    std::vector<unsigned> keys((size_t)nq * K);
    for (int q = 0; q < nq; ++q) top_k<K>(dist + (size_t)q * nc, nc, claimed, &keys[(size_t)q * K]);
    const auto decode = [](unsigned key) { return (int)(key & 0xffffu); };
    const auto unclaimed = [&](int c, int) { return !claimed[c]; };
    const auto ratio = [&](const ovs::ReplayList<K>& L, int second, ovs::Second kind) {
        if (mode == kNoRatio) return true;
        if (mode == kRatio) return !(lowe_ratio * (float)(unsigned)second < (float)L.dist[0]);
        if (kind == ovs::Second::bound) return !((float)L.dist[0] > lowe_ratio * (float)second);
        const int second_level = kind == ovs::Second::listed ? level[L.id[1]] : -1;
        return !(level[L.id[0]] == second_level && (float)L.dist[0] > lowe_ratio * (float)second);
    };
    *num_requeries = 0;
    for (int q = 0; q < nq; ++q) {
        const auto requery = [&](unsigned* fresh) {
            ++*num_requeries;
            top_k<K>(dist + (size_t)q * nc, nc, claimed, fresh);
            return OVS_OK;
        };
        ovs::ReplayPick p;
        const int rc = ovs::replay_query<K>(&keys[(size_t)q * K], thr, complete_at, decode, unclaimed, ratio, requery, &p);
        if (rc != OVS_OK) return rc;
        match[q] = p.id;
        if (p.id >= 0) claimed[p.id] = 1;
    }
    return OVS_OK;
}

}  // namespace

extern "C" {

// complete_at < 0: ovs::kNeverComplete.  match[q]: the candidate query q took, or -1.
int rc_replay(int K, int nq, int nc, const int* dist, const int* level, const uint8_t* claimed, int mode, int thr, int complete_at,
              float lowe_ratio, int* match, int* num_requeries) {
    if (complete_at < 0) complete_at = ovs::kNeverComplete;
    if (K == 4) return replay<4>(nq, nc, dist, level, claimed, mode, thr, complete_at, lowe_ratio, match, num_requeries);
    if (K == 8) return replay<8>(nq, nc, dist, level, claimed, mode, thr, complete_at, lowe_ratio, match, num_requeries);
    return OVS_ERR_INVALID_ARG;
}

int rc_d_star(float lowe_ratio) { return ovs::d_star(lowe_ratio); }

}  // extern "C"
