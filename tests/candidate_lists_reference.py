"""Plain numpy reference of the matchers' device candidate lists: for each query, the K = 8 smallest keys
(distance << 16 | tie) over its admissible candidates, ascending, padded with 0xFFFFFFFF.

- brute force (k_hamming_topk + k_topk_merge) and its re-query (k_hamming_one): every train descriptor, tie = train index;
- bow_tree (k_node_topk): the ranks of the query's segment, tie = rank;
- match_for_triangulation / create_new_landmarks (k_triangulation_topk): the ranks of the query's segment that pass the
  distance, epipole and epipolar-plane tests, tie = 0xFFFF - rank (the last of equal distances wins).

Hamming distances are popcounts of the XOR (a 16-bit word table built by np.unpackbits); the top K is an exact np.lexsort
on (distance, tie) of the K smallest pairs.  Large shapes are processed in query chunks, so memory stays bounded."""
import numpy as np

K = 8
EMPTY = 0xFFFFFFFF
HAMMING_DIST_THR_LOW = 50
EPIPOLE_COS = 0.998
EPIPOLAR_THR = 0.2 * np.pi / 180.0

# popcount of every 16-bit word
_POPCOUNT = np.unpackbits(np.arange(1 << 16, dtype="<u2").view(np.uint8)[:, None], axis=1).reshape(-1, 16).sum(axis=1).astype(np.uint8)
_CHUNK_BYTES = 1 << 26


def hamming(q, t):
    """(len(q), len(t)) int32 Hamming distances of 32-byte descriptors."""
    q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(t, np.uint8).reshape(-1, 32)
    out = np.empty((len(q), len(t)), np.int32)
    q16, t16 = q.view("<u2"), t.view("<u2")
    step = max(1, _CHUNK_BYTES // (32 * max(len(t), 1)))
    for a in range(0, len(q), step):
        out[a:a + step] = _POPCOUNT[q16[a:a + step, None, :] ^ t16[None, :, :]].sum(axis=2, dtype=np.int32)
    return out


def topk_keys(dist, tie, valid=None, k=K):
    """Rows of candidates -> (rows, k) uint32 keys of the k smallest (distance, tie) pairs among the valid ones.
    dist: (rows, m) int; tie: (m,) or (rows, m) int in 0 .. 0xFFFF, unique within a row; valid: (rows, m) bool or None."""
    dist = np.asarray(dist, np.int64)
    rows, m = dist.shape
    tie = np.broadcast_to(np.asarray(tie, np.int64), dist.shape)
    out = np.full((rows, k), EMPTY, np.uint32)
    if m == 0:
        return out
    if valid is None:
        valid = np.ones(dist.shape, bool)
    big = np.int64(1) << 40                      # past every valid (distance, tie) pair
    d = np.where(valid, dist, big)
    if m > k:                                    # the k smallest (distance, tie) pairs of each row, in no order yet
        part = np.argpartition((d << 16) | tie, k - 1, axis=1)[:, :k]
        d, tie = np.take_along_axis(d, part, axis=1), np.take_along_axis(tie, part, axis=1)
    order = np.lexsort((tie, d), axis=1)
    dk = np.take_along_axis(d, order, axis=1); tk = np.take_along_axis(tie, order, axis=1)
    ok = dk < big
    out[:, :order.shape[1]] = np.where(ok, (dk << 16) | tk, EMPTY).astype(np.uint32)
    return out


def bruteforce_topk(query, train, k=K):
    """ovs_match_bruteforce_topk_*: keys (distance << 16 | train index) over all of train."""
    query = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
    train = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
    out = np.full((len(query), k), EMPTY, np.uint32)
    idx = np.arange(len(train))
    step = max(1, _CHUNK_BYTES // (32 * max(len(train), 1)))
    for a in range(0, len(query), step):
        out[a:a + step] = topk_keys(hamming(query[a:a + step], train), idx, k=k)
    return out


def mask_bits(mask_words, n):
    """exclude[j] = bit j & 31 of mask_words[j >> 5], for j < n."""
    w = np.asarray(mask_words, np.uint32)
    j = np.arange(n)
    return ((w[j >> 5] >> (j & 31).astype(np.uint32)) & 1).astype(bool)


def hamming_one(query, train, mask_words):
    """k_hamming_one: one query over train, train descriptor j skipped where its mask bit is set."""
    train = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
    excl = mask_bits(mask_words, len(train))
    return topk_keys(hamming(query, train), np.arange(len(train)), ~excl[None, :])[0]


def node_topk(qdesc, qseg, tdesc, taken=None):
    """k_node_topk: query i over the ranks qseg[i, 0] .. qseg[i, 1] - 1 of tdesc not taken, keys (distance << 16 | rank)."""
    qdesc = np.ascontiguousarray(qdesc, np.uint8).reshape(-1, 32)
    qseg = np.asarray(qseg, np.int64).reshape(-1, 2)
    out = np.full((len(qdesc), K), EMPTY, np.uint32)
    # queries of one segment together
    for (b, e) in np.unique(qseg, axis=0):
        rows = np.flatnonzero((qseg[:, 0] == b) & (qseg[:, 1] == e))
        if e <= b:
            continue
        ranks = np.arange(b, e)
        valid = None if taken is None else np.broadcast_to(~np.asarray(taken[b:e], bool), (len(rows), e - b))
        out[rows] = topk_keys(hamming(qdesc[rows], tdesc[b:e]), ranks, valid)
    return out


def triangulation_gates(qbearing, qscale, qstereo, tbearing, tstereo, E, epipole):
    """The geometric tests of k_triangulation_topk for every (query, candidate) pair of one problem, evaluated in the
    kernel's float64 operation order.  -> passed (q, c) bool, and the relative distance of each pair to the nearest gate it
    evaluates ((q, c) float64, inf where neither applies), so that a caller can keep its cases away from the last-ulp
    difference between the device's acos and numpy's."""
    qb = np.asarray(qbearing, np.float64).reshape(-1, 3); tb = np.asarray(tbearing, np.float64).reshape(-1, 3)
    E = np.asarray(E, np.float64).reshape(9); ep = np.asarray(epipole, np.float64).reshape(3)
    ex = E[0] * tb[:, 0] + E[1] * tb[:, 1] + E[2] * tb[:, 2]
    ey = E[3] * tb[:, 0] + E[4] * tb[:, 1] + E[5] * tb[:, 2]
    ez = E[6] * tb[:, 0] + E[7] * tb[:, 1] + E[8] * tb[:, 2]
    norm = np.sqrt(ex * ex + ey * ey + ez * ez)
    cos_res = (ex[None, :] * qb[:, 0:1] + ey[None, :] * qb[:, 1:2] + ez[None, :] * qb[:, 2:3]) / norm[None, :]
    with np.errstate(invalid="ignore"):
        residual = np.pi / 2.0 - np.abs(np.arccos(cos_res))
    thr = EPIPOLAR_THR * np.asarray(qscale, np.float32).astype(np.float64)[:, None]
    epipolar = residual < thr
    cos_dist = ep[0] * tb[:, 0] + ep[1] * tb[:, 1] + ep[2] * tb[:, 2]
    mono = ~np.asarray(qstereo, bool)[:, None] & ~np.asarray(tstereo, bool)[None, :]
    near_epipole = mono & (EPIPOLE_COS < cos_dist)[None, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        margin = np.abs(residual - thr) / thr
        margin_epi = np.where(mono, np.abs(cos_dist - EPIPOLE_COS)[None, :] / EPIPOLE_COS, np.inf)
    return ~near_epipole & epipolar, np.fmin(np.where(np.isnan(margin), np.inf, margin), margin_epi)


def triangulation_topk(qdesc, qbearing, qscale, qstereo, qseg, tdesc, tbearing, tstereo, E, epipole, taken=None,
                       with_margin=False):
    """k_triangulation_topk<false> (one problem): query i over the ranks of its segment not taken, with distance <=
    HAMMING_DIST_THR_LOW, passing the epipole test (both keypoints monocular only) and the epipolar-plane test; keys
    (distance << 16 | 0xFFFF - rank).  with_margin: also the smallest relative gate distance over the pairs the kernel
    evaluates geometrically (distance gate passed, not taken)."""
    qdesc = np.ascontiguousarray(qdesc, np.uint8).reshape(-1, 32)
    qseg = np.asarray(qseg, np.int64).reshape(-1, 2)
    qb = np.asarray(qbearing, np.float64).reshape(-1, 3); tb = np.asarray(tbearing, np.float64).reshape(-1, 3)
    qs = np.asarray(qscale, np.float32); q8 = np.asarray(qstereo, np.uint8); t8 = np.asarray(tstereo, np.uint8)
    out = np.full((len(qdesc), K), EMPTY, np.uint32)
    margin = np.inf
    for (b, e) in np.unique(qseg, axis=0):
        rows = np.flatnonzero((qseg[:, 0] == b) & (qseg[:, 1] == e))
        if e <= b:
            continue
        d = hamming(qdesc[rows], tdesc[b:e])
        passed, m = triangulation_gates(qb[rows], qs[rows], q8[rows], tb[b:e], t8[b:e], E, epipole)
        free = np.ones(e - b, bool) if taken is None else ~np.asarray(taken[b:e], bool)
        evaluated = (d <= HAMMING_DIST_THR_LOW) & free[None, :]
        if evaluated.any():
            margin = min(margin, float(m[evaluated].min()))
        out[rows] = topk_keys(d, 0xFFFF - np.arange(b, e), evaluated & passed)
    return (out, margin) if with_margin else out


def triangulation_topk_batched(qdesc, qbearing, qscale, qstereo, qseg, tdesc, tbearing, tstereo, prob_E, prob_epipole, prob_tbase,
                               queries_per_prob, taken=None, with_margin=False):
    """k_triangulation_topk<true>: query q of problem p = q // queries_per_prob is keypoint entry q - p * queries_per_prob,
    with E_12 prob_E[p], epipole prob_epipole[p], and candidates (and taken flags) from prob_tbase[p] on; ranks (and the
    tie) stay per problem."""
    qseg = np.asarray(qseg, np.int64).reshape(-1, 2)
    nprob = len(prob_tbase)
    ends = list(prob_tbase[1:]) + [len(np.asarray(tstereo))]
    out, margin = [], np.inf
    for p in range(nprob):
        b0, b1 = int(prob_tbase[p]), int(ends[p])
        tk = None if taken is None else np.asarray(taken)[b0:b1]
        keys, m = triangulation_topk(qdesc, qbearing, qscale, qstereo, qseg[p * queries_per_prob:(p + 1) * queries_per_prob],
                                     np.asarray(tdesc).reshape(-1, 32)[b0:b1], np.asarray(tbearing).reshape(-1, 3)[b0:b1],
                                     np.asarray(tstereo)[b0:b1], np.reshape(prob_E, (-1, 9))[p], np.reshape(prob_epipole, (-1, 3))[p], tk,
                                     with_margin=True)
        out.append(keys); margin = min(margin, m)
    out = np.concatenate(out)
    return (out, margin) if with_margin else out


def node_order(bow_node, keep):
    """The keypoints that take part (keep, a vocabulary node) node by node, in index order inside a node: the
    reference's walk over the BoW feature vector."""
    node = np.asarray(bow_node)
    idx = np.flatnonzero(np.asarray(keep, bool) & (node >= 0))
    return idx[np.argsort(node[idx], kind="stable")]


def node_segments(query_nodes, ranked_nodes):
    """(q, 2): the range of ranks whose node is each query's"""
    ranked_nodes = np.asarray(ranked_nodes)
    return np.stack([np.searchsorted(ranked_nodes, query_nodes, "left"), np.searchsorted(ranked_nodes, query_nodes, "right")], 1)


def first_taker(lists, requery, num_candidates, skip=None):
    """match_for_triangulation's sequential loop over candidate lists: query k (in visiting order, skipped where skip[k])
    takes the first candidate (rank 0xFFFF - tie) of lists[k] not taken yet; a list whose K entries are all taken is
    recomputed by requery(k, taken) with the taken candidates excluded, and that list decides.
    -> rank taken by each query (-1: none), whether it came from a re-query, number of re-queries"""
    taken = np.zeros(num_candidates, bool)
    pick = np.full(len(lists), -1, np.int64)
    requeried = np.zeros(len(lists), bool)
    decode = lambda x: 0xFFFF - (int(x) & 0xFFFF)
    for k in range(len(lists)):
        if skip is not None and skip[k]:
            continue
        keys = [int(x) for x in lists[k] if x != EMPTY]
        free = [decode(x) for x in keys if not taken[decode(x)]]
        if not free and len(keys) == K:
            requeried[k] = True
            free = [decode(x) for x in requery(k, taken) if x != EMPTY]
        if free:
            taken[free[0]] = True
            pick[k] = free[0]
    return pick, requeried, int(requeried.sum())


def match_for_triangulation(p, sf):
    """robust::match_for_triangulation without the orientation check on a synth.triangulation_problem p, from the lists
    above and first_taker.  -> matched_idx_2_of_1, number of re-queries"""
    n1 = len(p["desc_1"])
    rank2 = node_order(p["bow_node_2"], p["has_lm_2"] == 0)
    q1 = node_order(p["bow_node_1"], p["has_lm_1"] == 0)
    seg = node_segments(p["bow_node_1"][q1], p["bow_node_2"][rank2]).reshape(-1, 2)
    args = (p["desc_1"][q1], p["bearing_1"][q1], sf[p["octave_1"][q1]], p["is_stereo_1"][q1], seg, p["desc_2"][rank2], p["bearing_2"][rank2],
            p["is_stereo_2"][rank2], p["E_12"], p["epipole_in_2"])
    lists = triangulation_topk(*args)
    pick, _, requeries = first_taker(lists, lambda k, taken: triangulation_topk(*[a[k:k + 1] for a in args[:5]], *args[5:], taken=taken)[0],
                                     len(rank2))
    match = np.full(n1, -1, np.int32)
    match[q1[pick >= 0]] = rank2[pick[pick >= 0]]
    return match, requeries
