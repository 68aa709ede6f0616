"""CPU checks of tests/candidate_lists_reference.py, the numpy reference the device candidate lists are compared with
(tests/test_candidate_lists_gpu.py): against the oracle's brute force (best and second best), against a direct Python loop on
small cases, and -- through its sequential first-taker loop over its lists -- against the oracle's match_for_triangulation."""
import numpy as np
import pytest

import candidate_lists_reference as ref
from openvslam_b200 import synth


def _loop_topk(dist, tie, valid):
    """the K smallest (distance, tie) pairs of one row by sorting Python tuples"""
    pairs = sorted((int(d), int(t)) for d, t, v in zip(dist, tie, valid) if v)[:ref.K]
    return [(d << 16) | t for d, t in pairs] + [ref.EMPTY] * (ref.K - len(pairs))


def _loop_hamming(a, b):
    return sum(bin(int(x) ^ int(y)).count("1") for x, y in zip(a, b))


@pytest.mark.parametrize("nq,nt,seed", [(1, 1, 0), (7, 5, 1), (40, 300, 2), (300, 40, 3)])
def test_bruteforce_topk_equals_the_oracle(oracle, nq, nt, seed):
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = np.concatenate([q, rng.integers(0, 256, (nt, 32), dtype=np.uint8)])[rng.permutation(nq + nt)][:nt]
    t[rng.integers(0, nt, nt // 4)] = t[0]                  # equal distances
    keys = ref.bruteforce_topk(q, t)
    bi, bd, sd = oracle.bruteforce(q, t)
    k0, k1 = keys[:, 0].astype(np.int64), keys[:, 1].astype(np.int64)
    assert np.array_equal(np.where(k0 == ref.EMPTY, -1, k0 & 0xFFFF), bi)
    assert np.array_equal(np.where(k0 == ref.EMPTY, 256, k0 >> 16), bd)
    assert np.array_equal(np.where(k1 == ref.EMPTY, 256, k1 >> 16), sd)


def test_hamming_equals_a_bit_loop():
    rng = np.random.default_rng(4)
    q = rng.integers(0, 256, (5, 32), dtype=np.uint8); t = rng.integers(0, 256, (9, 32), dtype=np.uint8)
    t[0] = q[0]; t[1] = ~q[1]
    d = ref.hamming(q, t)
    assert d[0, 0] == 0 and d[1, 1] == 256
    assert d.tolist() == [[_loop_hamming(a, b) for b in t] for a in q]


def test_topk_keys_equal_a_python_loop():
    rng = np.random.default_rng(5)
    for m in (0, 1, 3, 8, 9, 40):
        dist = rng.integers(0, 6, (20, m))                     # many equal distances
        tie = rng.permutation(0x10000)[:m]
        valid = rng.random((20, m)) < 0.7
        got = ref.topk_keys(dist, tie, valid)
        assert got.dtype == np.uint32 and got.shape == (20, ref.K)
        for r in range(20):
            assert got[r].tolist() == _loop_topk(dist[r], tie, valid[r]), (m, r)


def test_hamming_one_and_node_topk_equal_a_python_loop():
    rng = np.random.default_rng(6)
    base = rng.integers(0, 256, (3, 32), dtype=np.uint8)
    t = base[rng.integers(0, 3, 300)] ^ (rng.random((300, 32)) < 0.02).astype(np.uint8)
    q = base[rng.integers(0, 3, 12)]
    words = rng.integers(0, 2 ** 32, (300 + 31) // 32, dtype=np.uint64).astype(np.uint32)
    excl = [(int(words[j >> 5]) >> (j & 31)) & 1 for j in range(300)]
    for i in range(len(q)):
        want = _loop_topk([_loop_hamming(q[i], x) for x in t], range(300), [not e for e in excl])
        assert ref.hamming_one(q[i], t, words).tolist() == want
    seg = np.array([[0, 0], [0, 1], [5, 14], [5, 14], [20, 300], [299, 300]] * 2)
    taken = rng.random(300) < 0.4
    for tk in (None, taken):
        got = ref.node_topk(q, seg, t, tk)
        for i, (b, e) in enumerate(seg):
            want = _loop_topk([_loop_hamming(q[i], t[c]) for c in range(b, e)], range(b, e),
                              [tk is None or not tk[c] for c in range(b, e)])
            assert got[i].tolist() == want, (i, b, e)


def test_node_order_and_segments_equal_a_python_loop():
    rng = np.random.default_rng(8)
    node = rng.integers(-1, 6, 200).astype(np.int32)
    keep = rng.random(200) < 0.7
    got = ref.node_order(node, keep)
    assert got.tolist() == sorted((i for i in range(200) if keep[i] and node[i] >= 0), key=lambda i: (node[i], i))
    seg = ref.node_segments(np.array([-1, 0, 3, 5, 9]), node[got])
    for (b, e), q in zip(seg, [-1, 0, 3, 5, 9]):
        assert [int(x) for x in node[got][b:e]] == [q] * int(sum(node[got] == q))


@pytest.mark.parametrize("n,seed,nodes,dup", [(300, 1, 20, False), (400, 2, 3, False), (300, 7, 2, True)])
def test_triangulation_lists_replay_to_the_oracle(oracle, n, seed, nodes, dup):
    """The reference's gates (distance, epipole, epipolar plane) and its tie rule (last of equal distances), replayed by the
    sequential first-taker loop, give the oracle's match_for_triangulation without the orientation check."""
    p = synth.triangulation_problem(n, seed, n_nodes=nodes, stereo_frac=0.3)
    if dup:           # few distinct descriptors: ties everywhere and exhausted lists
        rng = np.random.default_rng(seed)
        base = rng.integers(0, 256, (3, 32), dtype=np.uint8)
        p["desc_1"] = base[rng.integers(0, 3, len(p["desc_1"]))]
        p["desc_2"] = base[rng.integers(0, 3, len(p["desc_2"]))]
    sf = oracle.scale_factors(1.2, 8)
    keys = ("desc_1", "bearing_1", "octave_1", "angle_1", "has_lm_1", "is_stereo_1", "bow_node_1",
            "desc_2", "bearing_2", "angle_2", "has_lm_2", "is_stereo_2", "bow_node_2", "E_12", "epipole_in_2")
    onum, om = oracle.robust_match_for_triangulation(*[p[k] for k in keys], sf, False)
    got, requeries = ref.match_for_triangulation(p, np.asarray(sf, np.float32))
    assert np.array_equal(got, om) and onum > 20
    if dup:
        assert requeries > 0
