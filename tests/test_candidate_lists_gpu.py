"""The matchers' device candidate lists, key for key, against the numpy top-K of tests/candidate_lists_reference.py.

The greedy replays (csrc/greedy_replay.h) trust every entry of a list and take its last distance as the bound on every unlisted
candidate, so a list is only right when all 8 keys are: the brute force (k_hamming_topk + k_topk_merge) at the shapes that reach
each branch of launch_topk's geometry, and the kernels of the re-queries (k_hamming_one with its exclusion mask, k_node_topk and
k_triangulation_topk with taken flags, q0 and the spare output row) through their test hooks.  Equal distances are placed on
both sides of the chunk and tile boundaries, where a lost or duplicated key would show."""
import ctypes as C

import numpy as np
import pytest

import candidate_lists_reference as ref
from openvslam_b200 import _lib, match

pytestmark = pytest.mark.gpu

EMPTY = ref.EMPTY
TILE = 128            # match_bruteforce.cu: train descriptors per shared-memory tile, queries per block
NODE_CHUNK = 256      # match_window.cu: candidates a warp walks per chunk (32 lanes x 8)
SEGMENTS = (0, 1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 511, 512, 513, 4000)
SCALE_FACTORS = (1.2 ** np.arange(8)).astype(np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def mt():
    m = match.robust()
    yield m
    m.close()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def bf_geometry(nq, nt, sms):
    """launch_topk's (nchunks, chunk): enough (query block, train chunk) pairs for 8 blocks per SM, chunks a multiple of the tile"""
    qblocks = (nq + TILE - 1) // TILE
    nchunks = max(1, (8 * sms + qblocks - 1) // qblocks)
    nchunks = min(nchunks, max(1, (nt + TILE - 1) // TILE))
    chunk = (nt + nchunks - 1) // nchunks
    chunk = max(TILE, (chunk + TILE - 1) // TILE * TILE)
    return max(1, (nt + chunk - 1) // chunk), chunk


def _flip(rng, d, nbits):
    """d with nbits random bits flipped per row"""
    out = d.copy()
    for i in range(len(out)):
        for b in rng.choice(256, nbits, replace=False):
            out[i, b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def _bf_problem(rng, nq, nt, chunk, nhot=24):
    """Random train descriptors with hot descriptors planted as exact copies: in pairs straddling every chunk and tile
    boundary, and up to 10 inside one chunk; queries are near copies of the hot descriptors (and some random ones) drawn from a
    pool of at most 300 distinct rows, so that every list ends inside a run of equal distances."""
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    hot = rng.integers(0, 256, (nhot, 32), dtype=np.uint8)
    bounds = sorted({b for s in (chunk, TILE) for b in range(s, nt, s)})
    for i, b in enumerate(bounds[:4000]):
        t[b - 1] = t[b] = hot[i % nhot]
    if nt >= 16:
        c0 = int(rng.integers(0, (nt - 1) // chunk + 1)) * chunk
        pos = c0 + rng.choice(min(chunk, nt - c0), min(10, nt - c0), replace=False)
        t[pos] = hot[0]
    pool = np.concatenate([_flip(rng, hot[rng.integers(0, nhot, 200)], 3), rng.integers(0, 256, (100, 32), dtype=np.uint8), hot[:4]])
    return pool[rng.integers(0, len(pool), nq)], t


def _bf_reference(q, t):
    u, inv = np.unique(q, axis=0, return_inverse=True)
    return ref.bruteforce_topk(u, t)[inv.reshape(-1)]


def _bf_cases(sms):
    """(name, nq, nt) and the geometry each one is there for"""
    nq_one = 8 * sms * TILE                                   # qblocks == 8 SMs: one chunk whatever nt
    q_tile = 4000
    n_tile = -(-8 * sms // -(-q_tile // TILE))                # chunks of exactly one tile
    nt_part = next(nt for nt in range(20000, 22000)
                   if (lambda nc, ch: 0 < nt - (nc - 1) * ch < ch and (nt - (nc - 1) * ch) % TILE and nt - (nc - 1) * ch > TILE)(*bf_geometry(2000, nt, sms)))
    return [("one_chunk_by_train", 1000, 100), ("one_chunk_by_queries", nq_one, 300), ("chunk_is_one_tile", q_tile, n_tile * TILE),
            ("partial_last_tile_and_chunk", 2000, nt_part), ("nq127", 127, 1000), ("nq128", 128, 1000), ("nq129", 129, 1000),
            ("nt1", 300, 1), ("nt5", 300, 5), ("nt7", 300, 7), ("nq1_nt65535", 1, 65535)]


CASE_NAMES = ["one_chunk_by_train", "one_chunk_by_queries", "chunk_is_one_tile", "partial_last_tile_and_chunk", "nq127", "nq128", "nq129",
              "nt1", "nt5", "nt7", "nq1_nt65535"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_bruteforce_lists_at_every_launch_geometry(mt, sms, name):
    _, nq, nt = next(c for c in _bf_cases(sms) if c[0] == name)
    nchunks, chunk = bf_geometry(nq, nt, sms)
    last = nt - (nchunks - 1) * chunk
    if name.startswith("one_chunk"):
        assert nchunks == 1 and (nt <= TILE or (nq + TILE - 1) // TILE >= 8 * sms)
    elif name == "chunk_is_one_tile":
        assert nchunks > 1 and chunk == TILE and last == TILE
    elif name == "partial_last_tile_and_chunk":
        assert nchunks > 1 and chunk > TILE and TILE < last < chunk and last % TILE
    elif name == "nq1_nt65535":
        assert nchunks >= 256 and nt == 65535
    elif name.startswith("nt"):
        assert nt < ref.K
    rng = np.random.default_rng(nq * 7 + nt)
    q, t = _bf_problem(rng, nq, nt, chunk)
    if name == "nq1_nt65535":
        t[65534] = t[chunk - 1] = t[chunk] = q[0]               # distance 0 at the last 16-bit index and across a boundary
    want = _bf_reference(q, t)
    got = mt.brute_force_topk(q, t)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, (name, nchunks, chunk, bad[:5], got[bad[:2]], want[bad[:2]])
    if nt >= ref.K:
        assert (want != EMPTY).all()
    else:
        assert (want[:, nt:] == EMPTY).all() and (want[:, :nt] != EMPTY).all()


def test_bruteforce_lists_of_identical_and_complementary_descriptors(mt, sms):
    rng = np.random.default_rng(11)
    q = rng.integers(0, 256, (300, 32), dtype=np.uint8)
    same = np.repeat(q[:1], 3000, axis=0)                      # every distance equal: the 8 lowest indices
    for t in (same, ~same):
        got, want = mt.brute_force_topk(q, t), _bf_reference(q, t)
        assert np.array_equal(got, want)
        assert np.array_equal(got[0] & 0xFFFF, np.arange(8)) and (got[0] >> 16 == (0 if t is same else 256)).all()
    t = np.repeat(~q[:1], 2000, axis=0)                        # distance 256 everywhere except three copies at distance 0
    t[[127, 128, 1999]] = q[0]
    got, want = mt.brute_force_topk(q, t), _bf_reference(q, t)
    assert np.array_equal(got, want) and (got[0, :3] == [127, 128, 1999]).all() and got[0, 3] == (256 << 16 | 0)


def test_bruteforce_device_entry_equals_the_host_entry():
    import torch
    rng = np.random.default_rng(12)
    nchunks, chunk = bf_geometry(3000, 5000, 132)
    q, t = _bf_problem(rng, 3000, 5000, chunk)
    dev = torch.device("cuda", 0)
    tq, tt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
    keys = torch.full((3000, 8), 7, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    m = match.robust()
    m.brute_force_topk_device(tq.data_ptr(), 3000, tt.data_ptr(), 5000, keys.data_ptr())
    got = keys.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, m.brute_force_topk(q, t)) and np.array_equal(got, _bf_reference(q, t))
    # no query: no launch, nothing written
    before = _lib.launch_count()
    m.brute_force_topk_device(tq.data_ptr(), 0, tt.data_ptr(), 5000, keys.data_ptr())
    assert _lib.launch_count() == before
    # descriptors that are not 16-byte aligned are refused before any launch
    raw = torch.zeros(32 * 101, dtype=torch.uint8, device=dev)
    for dq, dt in ((raw.data_ptr() + 8, tt.data_ptr()), (tq.data_ptr(), raw.data_ptr() + 4)):
        with pytest.raises(_lib.OvsError) as e:
            m.brute_force_topk_device(dq, 100, dt, 100, keys.data_ptr())
        assert e.value.code == -1 and _lib.launch_count() == before
    m.close()


# ----------------------------------------------------------------------------------------------- k_hamming_one
def _mask(kind, nt, rng, want_free):
    """exclusion bitmask words (bit j & 31 of word j >> 5 excludes train descriptor j)"""
    words = (nt + 31) // 32
    j = np.arange(nt)
    if kind == "none":
        ex = np.zeros(nt, bool)
    elif kind == "all":
        ex = np.ones(nt, bool)
    elif kind.startswith("all_but_"):
        ex = np.ones(nt, bool)
        ex[want_free[:int(kind[8:])]] = False
    elif kind == "alternate_words":
        ex = (j >> 5) % 2 == 0
    elif kind == "one_thread_stride":
        ex = j % 256 == 37
    elif kind == "word_edges":
        ex = (j % 32 == 0) | (j % 32 == 31)
    else:
        ex = rng.random(nt) < 0.5
    bits = np.zeros(words * 32, np.uint8)
    bits[:nt] = ex
    return np.packbits(bits, bitorder="little").view("<u4").copy()


MASKS = ("none", "all", "all_but_1", "all_but_3", "all_but_7", "alternate_words", "one_thread_stride", "word_edges", "random")


@pytest.mark.parametrize("nt", (1, 255, 256, 257, 4000, 65535))
def test_hamming_one_lists_with_exclusion_masks(mt, nt):
    rng = np.random.default_rng(nt)
    q = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    # equal near copies of the query on both sides of the 32-bit words, of the 256-thread stride and at the end
    pos = np.unique([p for p in (0, 1, 15, 16, 31, 32, 33, 37, 63, 64, 255, 256, 257, 293, 511, 512, nt - 1) if p < nt])
    t[pos] = _flip(rng, q, 4)[0]
    t[pos[::3]] = q[0]
    want_free = rng.permutation(pos)
    for kind in MASKS:
        words = _mask(kind, nt, rng, want_free)
        assert np.array_equal(ref.mask_bits(words, nt), _mask_bits_loop(words, nt))
        keys = _hamming_one(mt, q, t, words)
        want = ref.hamming_one(q[0], t, words)
        assert np.array_equal(keys, want), (kind, keys, want)
        if kind == "all":
            assert (keys == EMPTY).all()
        if kind.startswith("all_but_"):
            n_free = min(int(kind[8:]), len(pos))
            assert (keys[:n_free] != EMPTY).all() and (keys[n_free:] == EMPTY).all()


def _hamming_one(mt, q, t, words):
    keys = np.zeros(8, np.uint32)
    _lib.check(_lib.lib().ovs_debug_hamming_one(mt._h, _p(q), _p(t), len(t), _p(words), _p(keys)))
    return keys


def _mask_bits_loop(words, nt):
    return np.array([(int(words[j >> 5]) >> (j & 31)) & 1 for j in range(nt)], bool)


# ------------------------------------------------------------------------------------------------- k_node_topk
def _segment_problem(rng, lengths, per_segment=4, shared=(4000, 200), R_total=None):
    """Candidates laid out segment after segment (rank order); in each segment near copies of a hot descriptor, with
    exact duplicates on both sides of every 256-candidate chunk boundary; queries near copies of their segment's hot
    descriptor, `shared[1]` of them on the segment of length shared[0]."""
    starts = np.concatenate([[0], np.cumsum(lengths)])
    R = int(starts[-1]) if R_total is None else R_total
    t = rng.integers(0, 256, (R, 32), dtype=np.uint8)
    hot = rng.integers(0, 256, (len(lengths), 32), dtype=np.uint8)
    qd, qs = [], []
    off = 0 if R_total is None else R_total - int(starts[-1])
    for s, L in enumerate(lengths):
        b = off + int(starts[s])
        if L:
            t[b:b + L] = _flip(rng, np.repeat(hot[s:s + 1], L, axis=0), 6)
            k = rng.integers(0, 12, L)
            t[b:b + L][k < 3] = _flip(rng, hot[s:s + 1], 2)[0]                # a run of equal distances
            t[b:b + L][k == 10] = _flip(rng, hot[s:s + 1].repeat((k == 10).sum(), axis=0), int(rng.integers(44, 54)))   # around 50
            t[b:b + L][k == 11] = rng.integers(0, 256, ((k == 11).sum(), 32), dtype=np.uint8)
            for c in range(NODE_CHUNK, L, NODE_CHUNK):
                t[b + c - 1] = t[b + c] = hot[s]
        n = shared[1] if L == shared[0] else per_segment
        qd.append(_flip(rng, np.repeat(hot[s:s + 1], n, axis=0), 3)); qs += [(b, b + L)] * n
    return np.concatenate(qd), np.array(qs, np.int32), t


def _node(mt, qdesc, qseg, tdesc, taken=None, q0=-1):
    nq = len(qdesc)
    keys = np.zeros((nq + (q0 >= 0), 8), np.uint32)
    _lib.check(_lib.lib().ovs_debug_node_topk(mt._h, nq, _p(np.ascontiguousarray(qdesc)), _p(np.ascontiguousarray(qseg, np.int32)), len(tdesc),
                                              _p(np.ascontiguousarray(tdesc)), _p(taken), int(q0), _p(keys)))
    return keys


def _taken_kinds(rng, R, listed_ranks):
    """random and adversarial taken flags: sparse, dense, every listed candidate, the chunk edges and the listed ones"""
    listed = np.zeros(R, np.uint8)
    listed[listed_ranks] = 1
    edges = np.zeros(R, np.uint8)
    r = np.arange(R)
    edges[(r % NODE_CHUNK == 0) | (r % NODE_CHUNK == NODE_CHUNK - 1)] = 1
    return {"sparse": (rng.random(R) < 0.3).astype(np.uint8), "dense": (rng.random(R) < 0.95).astype(np.uint8), "listed": listed,
            "chunk_edges": edges | listed}


def test_node_lists_over_every_segment_shape(mt):
    rng = np.random.default_rng(21)
    qdesc, qseg, tdesc = _segment_problem(rng, SEGMENTS)
    want = ref.node_topk(qdesc, qseg, tdesc)
    got = _node(mt, qdesc, qseg, tdesc)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, (bad[:5], qseg[bad[:5]], got[bad[:1]], want[bad[:1]])
    L = qseg[:, 1] - qseg[:, 0]
    assert ((want != EMPTY).sum(axis=1) == np.minimum(L, 8)).all()
    # with taken flags on every query at once
    for name, taken in _taken_kinds(rng, len(tdesc), want[want != EMPTY].astype(np.int64) & 0xFFFF).items():
        assert np.array_equal(_node(mt, qdesc, qseg, tdesc, taken), ref.node_topk(qdesc, qseg, tdesc, taken)), name


def test_node_requery_writes_the_spare_row_only(mt):
    rng = np.random.default_rng(22)
    qdesc, qseg, tdesc = _segment_problem(rng, SEGMENTS, per_segment=2, shared=(4000, 20))
    full = ref.node_topk(qdesc, qseg, tdesc)
    kinds = _taken_kinds(rng, len(tdesc), full[full != EMPTY].astype(np.int64) & 0xFFFF)
    for q0 in [0] + [int(np.flatnonzero(qseg[:, 1] - qseg[:, 0] == L)[0]) for L in SEGMENTS[1:]] + [len(qdesc) - 1]:
        kinds["listed"] = np.zeros(len(tdesc), np.uint8)
        kinds["listed"][full[q0][full[q0] != EMPTY].astype(np.int64) & 0xFFFF] = 1     # the replay's case: its list used up
        for name, taken in kinds.items():
            got = _node(mt, qdesc, qseg, tdesc, taken, q0)
            assert np.array_equal(got[:-1], full), (q0, name)
            assert np.array_equal(got[-1], ref.node_topk(qdesc[q0:q0 + 1], qseg[q0:q0 + 1], tdesc, taken)[0]), (q0, name)


def test_node_lists_at_the_16_bit_rank_limit(mt):
    rng = np.random.default_rng(23)
    R = 65535
    qdesc, qseg, tdesc = _segment_problem(rng, (513, 256, 1), per_segment=3, shared=(0, 0), R_total=R)
    qseg = np.concatenate([qseg, [[0, R], [0, R]]]).astype(np.int32)          # and the whole of it
    qdesc = np.concatenate([qdesc, qdesc[:1], tdesc[R - 1:R]])
    assert qseg[:, 1].max() == R
    want = ref.node_topk(qdesc, qseg, tdesc)
    assert np.array_equal(_node(mt, qdesc, qseg, tdesc), want)
    assert want[-1, 0] == R - 1                                                 # distance 0 at rank 65534


# ---------------------------------------------------------------------------------------- k_triangulation_topk
def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _essential(rng):
    a = rng.normal(size=3); th = np.linalg.norm(a); k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    Rm = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = _unit(rng.normal(size=3))
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    return (tx @ Rm).reshape(9), t


def _tri_problem(rng, lengths, per_segment=4, shared=(4000, 100)):
    qdesc, qseg, tdesc = _segment_problem(rng, lengths, per_segment, shared)
    nq, R = len(qdesc), len(tdesc)
    E, epipole = _essential(rng)
    # keyframe-2 bearings: random, a quarter of them within a few degrees of the epipole; keyframe-1 bearings: random, so that
    # about half of the pairs pass the one-sided epipolar test
    tb = _unit(rng.normal(size=(R, 3)))
    near = rng.random(R) < 0.25
    tb[near] = _unit(epipole + rng.normal(scale=0.06, size=(near.sum(), 3)))
    qb = _unit(rng.normal(size=(nq, 3)))
    qscale = SCALE_FACTORS[rng.integers(0, 8, nq)]
    q8 = (rng.random(nq) < 0.3).astype(np.uint8); t8 = (rng.random(R) < 0.3).astype(np.uint8)
    return dict(qdesc=qdesc, qbearing=qb, qscale=qscale, qstereo=q8, qseg=qseg, tdesc=tdesc, tbearing=tb, tstereo=t8, E=E, epipole=epipole)


def _tri(mt, P, taken=None, q0=-1, batched=False):
    nq = len(P["qseg"])
    qpp = P.get("queries_per_prob", nq)
    E = np.ascontiguousarray(np.reshape(P["E"], -1), np.float64); ep = np.ascontiguousarray(np.reshape(P["epipole"], -1), np.float64)
    nprob = len(ep) // 3
    tbase = np.ascontiguousarray(P.get("tbase", np.zeros(1)), np.int32)
    keys = np.zeros((nq + (q0 >= 0), 8), np.uint32)
    a = {k: np.ascontiguousarray(P[k], dt) for k, dt in (("qdesc", np.uint8), ("qbearing", np.float64), ("qscale", np.float32), ("qstereo", np.uint8),
                                                         ("qseg", np.int32), ("tdesc", np.uint8), ("tbearing", np.float64), ("tstereo", np.uint8))}
    _lib.check(_lib.lib().ovs_debug_triangulation_topk(
        mt._h, int(batched), nq, qpp, _p(a["qdesc"]), _p(a["qbearing"]), _p(a["qscale"]), _p(a["qstereo"]), _p(a["qseg"]),
        len(a["tdesc"]), _p(a["tdesc"]), _p(a["tbearing"]), _p(a["tstereo"]), nprob, _p(E), _p(ep), _p(tbase), _p(taken), int(q0), _p(keys)))
    return keys


def _tri_ref(P, taken=None, rows=None):
    s = slice(None) if rows is None else rows
    return ref.triangulation_topk(P["qdesc"][s], P["qbearing"][s], P["qscale"][s], P["qstereo"][s], P["qseg"][s], P["tdesc"], P["tbearing"],
                                  P["tstereo"], P["E"], P["epipole"], taken, with_margin=True)


def test_triangulation_lists_over_every_segment_shape(mt):
    rng = np.random.default_rng(31)
    P = _tri_problem(rng, SEGMENTS)
    want, margin = _tri_ref(P)
    assert margin > 1e-9, "a candidate within 1e-9 of a gate: the device's acos may decide it either way"
    listed = (want != EMPTY).sum(axis=1)
    assert listed.max() == 8 and (listed[(P["qseg"][:, 1] - P["qseg"][:, 0]) > 0] < 8).any()     # full and short lists
    got = _tri(mt, P)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, (bad[:5], P["qseg"][bad[:5]], got[bad[:1]], want[bad[:1]])
    for name, taken in _taken_kinds(rng, len(P["tdesc"]), 0xFFFF - (want[want != EMPTY].astype(np.int64) & 0xFFFF)).items():
        assert np.array_equal(_tri(mt, P, taken), _tri_ref(P, taken)[0]), name


def test_triangulation_gates_and_stereo_flags_matter(mt):
    """the same problem with every keypoint monocular, every one stereo, and stereo on one side only: each gate removes
    candidates somewhere, and the device agrees in every setting"""
    rng = np.random.default_rng(32)
    P = _tri_problem(rng, (300, 600, 4000), per_segment=20, shared=(0, 0))
    lists = {}
    for q8, t8 in ((0, 0), (1, 1), (1, 0), (0, 1)):
        Q = dict(P, qstereo=np.full(len(P["qseg"]), q8, np.uint8), tstereo=np.full(len(P["tdesc"]), t8, np.uint8))
        want, margin = _tri_ref(Q)
        assert margin > 1e-9
        assert np.array_equal(_tri(mt, Q), want), (q8, t8)
        lists[q8, t8] = want
    assert not np.array_equal(lists[0, 0], lists[1, 1])            # the epipole test removed candidates of the monocular pairs
    assert np.array_equal(lists[1, 1], lists[1, 0]) and np.array_equal(lists[1, 1], lists[0, 1])


def test_triangulation_requery_writes_the_spare_row_only(mt):
    rng = np.random.default_rng(33)
    P = _tri_problem(rng, SEGMENTS, per_segment=2, shared=(4000, 10))
    full, _ = _tri_ref(P)
    R = len(P["tdesc"])
    for q0 in (0, 9, 17, 25, len(P["qseg"]) - 1):
        listed = np.zeros(R, np.uint8)
        k = full[q0][full[q0] != EMPTY].astype(np.int64)
        listed[0xFFFF - (k & 0xFFFF)] = 1
        for taken in (listed, (rng.random(R) < 0.5).astype(np.uint8) | listed):
            got = _tri(mt, P, taken, q0)
            assert np.array_equal(got[:-1], full), q0
            assert np.array_equal(got[-1], _tri_ref(P, taken, slice(q0, q0 + 1))[0][0]), q0


def _batched_problem(rng, sizes, Q):
    """problems with keyframe-2 sets of the given sizes one after the other (prob_tbase), one query set of Q keypoints shared by
    all problems, each query's segment drawn inside its problem (empty for an empty problem), a different E_12 and epipole each"""
    parts = [_tri_problem(rng, (max(n, 1),), per_segment=Q, shared=(0, 0)) for n in sizes]
    base = parts[0]
    tbase = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int32)
    td = np.concatenate([p["tdesc"][:n] for p, n in zip(parts, sizes)])
    tb = np.concatenate([p["tbearing"][:n] for p, n in zip(parts, sizes)])
    t8 = np.concatenate([p["tstereo"][:n] for p, n in zip(parts, sizes)])
    seg = []
    for n in sizes:
        b = rng.integers(0, n + 1, Q); e = np.minimum(n, b + rng.choice([1, 8, 9, 256, 257, 600, 4000], Q))
        b[::5] = 0; e[::5] = n                                      # whole problem
        seg.append(np.stack([b, np.maximum(b, e)], 1))
    return dict(qdesc=base["qdesc"], qbearing=base["qbearing"], qscale=base["qscale"], qstereo=base["qstereo"], qseg=np.concatenate(seg).astype(np.int32),
                tdesc=td, tbearing=tb, tstereo=t8, E=np.stack([p["E"] for p in parts]), epipole=np.stack([p["epipole"] for p in parts]),
                tbase=tbase, queries_per_prob=Q)


def _tri_batched_ref(P, taken=None):
    return ref.triangulation_topk_batched(P["qdesc"], P["qbearing"], P["qscale"], P["qstereo"], P["qseg"], P["tdesc"], P["tbearing"], P["tstereo"],
                                          P["E"], P["epipole"], P["tbase"], P["queries_per_prob"], taken, with_margin=True)


def test_batched_triangulation_lists(mt):
    rng = np.random.default_rng(34)
    Q = 30
    P = _batched_problem(rng, (700, 0, 4100, 40, 1), Q)
    # the batch's queries are near copies of problem 0's candidates: give every problem some of them
    for p, b in enumerate(P["tbase"]):
        n = (list(P["tbase"][1:]) + [len(P["tdesc"])])[p] - b
        if n:
            P["tdesc"][b + rng.integers(0, n, min(n, 200))] = _flip(rng, P["qdesc"][rng.integers(0, Q, min(n, 200))], 3)
    want, margin = _tri_batched_ref(P)
    assert margin > 1e-9
    assert (want[Q:2 * Q] == EMPTY).all() and (want[2 * Q:3 * Q] != EMPTY).any() and (want != EMPTY).sum(axis=1).max() == 8
    got = _tri(mt, P, batched=True)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, (bad[:5], got[bad[:1]], want[bad[:1]])
    R = len(P["tdesc"])
    taken = (rng.random(R) < 0.4).astype(np.uint8)
    assert np.array_equal(_tri(mt, P, taken, batched=True), _tri_batched_ref(P, taken)[0])
    # re-queries on both sides of the queries_per_prob boundaries
    for q0 in (0, Q - 1, Q, 2 * Q - 1, 2 * Q, 3 * Q, 5 * Q - 1):
        got = _tri(mt, P, taken, q0, batched=True)
        assert np.array_equal(got[:-1], want), q0
        assert np.array_equal(got[-1], _tri_batched_ref(P, taken)[0][q0]), q0


def test_triangulation_gates_on_their_knife_edges(mt):
    """candidates 1e-9 relative inside and outside the epipolar-plane threshold (0.2 deg x scale) and the epipole bound
    (cos 0.998), each the only candidate of its query: the device keeps exactly the inside ones"""
    rel = (-1e-9, 1e-9)
    qb, tb, q8, t8, qs, expect = [], [], [], [], [], []
    for s in SCALE_FACTORS[[0, 3, 7]]:
        for r in rel:            # epipolar: E = I, b2 = e_z, residual = asin(b1_z)
            x = np.sin(ref.EPIPOLAR_THR * float(s) * (1 + r))
            qb.append([np.sqrt(1 - x * x), 0, x]); tb.append([0, 0, 1.0]); q8.append(1); t8.append(1); qs.append(s); expect.append(r < 0)
    for r in rel:                # epipole (0, 0, 1): cos_dist = b2_z; b1 = e_y is on b2's epipolar plane (residual 0)
        c = ref.EPIPOLE_COS * (1 + r)
        b2 = [np.sqrt(1 - c * c), 0, c]
        for st in ((0, 0), (1, 0), (0, 1)):
            qb.append([0, 1.0, 0]); tb.append(b2); q8.append(st[0]); t8.append(st[1]); qs.append(1.0); expect.append(r < 0 or st != (0, 0))
    n = len(qb)
    d = np.random.default_rng(35).integers(0, 256, (1, 32), dtype=np.uint8)
    P = dict(qdesc=np.repeat(d, n, axis=0), qbearing=np.array(qb), qscale=np.array(qs, np.float32), qstereo=np.array(q8, np.uint8),
             qseg=np.stack([np.arange(n), np.arange(n) + 1], 1).astype(np.int32), tdesc=np.repeat(d, n, axis=0), tbearing=np.array(tb),
             tstereo=np.array(t8, np.uint8), E=np.eye(3).reshape(9), epipole=np.array([0, 0, 1.0]))
    want, _ = _tri_ref(P)
    assert np.array_equal(want[:, 0] != EMPTY, expect)
    got = _tri(mt, P)
    assert np.array_equal(got, want), (got[:, 0], want[:, 0])
