"""CPU checks of csrc/greedy_replay.h, the host replay of the sequential first-taker matchers: a g++ shim (tests/replaycheck)
runs the replay over seeded candidate sets, with exact top-K lists as its "device", and its matches must equal a direct
sequential loop over the full candidate sets.  No device is needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
THR_LOW, THR_HIGH, MAX_DIST = 50, 100, 256
NO_RATIO, RATIO, LEVEL_RATIO = 0, 1, 2
F32 = np.float32


@pytest.fixture(scope="module")
def rc(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("replaycheck") / "libreplaycheck.so")
    subprocess.check_call(["g++", "-O1", "-fPIC", "-std=c++17", "-shared", "-o", so, os.path.join(HERE, "replaycheck", "replaycheck.cpp")])
    lib = C.CDLL(so)
    lib.rc_replay.restype = C.c_int
    lib.rc_replay.argtypes = [C.c_int] * 3 + [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_float, C.c_void_p, C.c_void_p]
    lib.rc_d_star.restype = C.c_int
    lib.rc_d_star.argtypes = [C.c_float]
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def replay(rc, K, dist, level, claimed, mode, thr, complete_at, lowe_ratio):
    nq, nc = dist.shape
    dist = np.ascontiguousarray(dist, np.int32)
    match = np.full(nq, -2, np.int32)
    nreq = C.c_int(-1)
    assert rc.rc_replay(K, nq, nc, _ptr(dist), _ptr(level), _ptr(claimed), mode, thr, complete_at, lowe_ratio, _ptr(match),
                        C.byref(nreq)) == 0
    return match, nreq.value


def sequential(dist, level, claimed, mode, thr, lowe_ratio):
    """The reference's loop: every query scans its unclaimed candidates in index order for the best and second best
    (strict '<', so the first wins ties), then applies the threshold and the ratio test; a match claims its candidate."""
    claimed = claimed.astype(bool)
    match = np.full(dist.shape[0], -1, np.int32)
    lowe = F32(lowe_ratio)
    for q, row in enumerate(dist.tolist()):
        best, second, best_c, best_level, second_level = MAX_DIST, MAX_DIST, -1, -1, -1
        for c, d in enumerate(row):
            if d < 0 or claimed[c]:
                continue
            if d < best:
                second, second_level = best, best_level
                best, best_level, best_c = d, int(level[c]), c
            elif d < second:
                second, second_level = d, int(level[c])
        if best_c < 0 or best > thr:
            continue
        if mode == RATIO and lowe * F32(second) < F32(best):
            continue
        if mode == LEVEL_RATIO and best_level == second_level and F32(best) > lowe * F32(second):
            continue
        match[q] = best_c
        claimed[best_c] = True
    return match


def problem(seed, d_star):
    """Queries that contend for few candidates (so that earlier takers empty later lists), distances drawn around the
    thresholds and d_star with many ties, duplicate rows, and some candidates claimed from the start."""
    rng = np.random.default_rng(seed)
    nq, nc = int(rng.integers(1, 120)), int(rng.integers(1, 40))
    marks = np.array([THR_LOW, THR_HIGH, d_star], np.int64)
    near = (marks[:, None] + np.arange(-2, 3)[None, :]).ravel()
    pool = np.concatenate([near, rng.integers(0, 256, 16), rng.integers(30, 70, 16), [0, 255]])
    dist = rng.choice(pool, (nq, nc)).astype(np.int32)
    dist[rng.random((nq, nc)) < rng.uniform(0.0, 0.7)] = -1          # not a candidate of this query
    dup = rng.random(nq) < 0.2                                        # a query repeating an earlier one's candidate set
    for q in np.flatnonzero(dup):
        if q > 0:
            dist[q] = dist[int(rng.integers(0, q))]
    level = rng.integers(0, int(rng.integers(1, 4)), nc).astype(np.int32)
    claimed = (rng.random(nc) < rng.uniform(0.0, 0.3)).astype(np.uint8)
    return dist, level, claimed


LOWE = (0.6, 0.7, 0.75, 0.8, 0.9, 1.0)
CASES = [(K, mode, complete) for K in (4, 8) for mode in (NO_RATIO, RATIO, LEVEL_RATIO) for complete in (False, True)]


@pytest.mark.parametrize("K,mode,complete", CASES,
                         ids=["K%d-%s-%s" % (K, ("no_ratio", "ratio", "level_ratio")[m], "d_star" if c else "never") for K, m, c in CASES])
def test_replay_equals_sequential_loop(rc, K, mode, complete):
    # the d_star shortcut holds for the threshold HAMMING_DIST_THR_LOW only (bow_tree, robust); the window and
    # triangulation replays run without it at their own thresholds
    thresholds = (THR_LOW,) if complete else (THR_LOW, THR_HIGH, MAX_DIST)
    requeries = 0
    for seed in range(40):
        lowe = LOWE[seed % len(LOWE)]
        d_star = rc.rc_d_star(lowe)
        dist, level, claimed = problem(1000 * K + 100 * mode + seed, d_star)
        for thr in thresholds:
            want = sequential(dist, level, claimed, mode, thr, lowe)
            got, n = replay(rc, K, dist, level, claimed, mode, thr, d_star if complete else -1, lowe)
            np.testing.assert_array_equal(got, want, err_msg="seed %d thr %d lowe %g" % (seed, thr, lowe))
            requeries += n
            if complete:
                # at HAMMING_DIST_THR_LOW a list whose lower bound reaches d_star passes the ratio test against that bound
                # and needs no re-query anyway: the shortcut changes neither a decision nor the re-query count
                got_never, n_never = replay(rc, K, dist, level, claimed, mode, thr, -1, lowe)
                np.testing.assert_array_equal(got_never, want)
                assert n_never == n
    assert requeries > 0, "no list needed a re-query: the cases do not reach the replay's re-query branches"

