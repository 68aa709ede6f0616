"""Array-pass model of the device tree distribution (k_tree_distribute in csrc/orb_extractor.cu).

The kernel restates orb_extractor::distribute_keypoints_via_tree without the std::list: every node carries
the serial number of its creation, the list order is recovered at the end by sorting on it (children are
pushed to the list front in creation order, so the list is "descending serial", with the surviving initial
nodes behind in ascending order).  This file is the same sequence of passes in numpy; the CPU suite checks
it against the oracle's list-based tree so that the formulation is pinned independently of the GPU.
"""
import numpy as np


def _centre(b):
    cx = b[:, 0] + ((b[:, 2] - b[:, 0] + 1) >> 1)
    cy = b[:, 1] + ((b[:, 3] - b[:, 1] + 1) >> 1)
    return cx, cy


def _child_boxes(pb, k):
    cx, cy = _centre(pb)
    bx = np.where(k & 1, cx, pb[:, 0]); ex = np.where(k & 1, pb[:, 2], cx)
    by = np.where(k & 2, cy, pb[:, 1]); ey = np.where(k & 2, pb[:, 3], cy)
    return np.stack([bx, by, ex, ey], 1)


def distribute(x, y, score, min_x, max_x, min_y, max_y, num_keypts, stats=None):
    """x, y relative to the level border, in candidate (row-major per cell) order.  Returns candidate indices.

    `stats`, if given, receives the sizes that decide where the kernel sorts: "pool_m", the largest node pool of the
    largest-first phase (0 if the phase is not reached), and "nfin", the length of the selection."""
    n = len(x)
    if stats is not None:
        stats.update(pool_m=0, nfin=0)
    if n == 0:
        return np.zeros(0, np.int64)
    x = np.asarray(x, np.int64); y = np.asarray(y, np.int64); score = np.asarray(score, np.int64)
    N = int(num_keypts)
    ratio = float(max_x - min_x) / (max_y - min_y)
    if ratio > 1:
        gx, gy = int(np.floor(ratio + 0.5)), 1   # std::round of a positive value
        dx, dy = float(max_x - min_x) / gx, float(max_y - min_y)
    else:
        gx, gy = 1, int(np.floor(1 / ratio + 0.5))
        dx, dy = float(max_x - min_x), float(max_y - min_y) / gy
    nini = gx * gy
    k0 = np.minimum((x.astype(np.float32).astype(np.float64) / dx).astype(np.int64)
                    + (y.astype(np.float32).astype(np.float64) / dy).astype(np.int64) * gx, nini - 1)
    cc = np.bincount(k0, minlength=nini)
    fin_key = []; fin_cand = []                    # order key (ascending = list order), candidate
    idx = np.arange(n)

    def best_of(groups, live, ngroups):
        key = ((score << 24) | (0xFFFFFF - idx))[live]
        best = np.zeros(ngroups, np.int64)
        np.maximum.at(best, groups, key)
        return 0xFFFFFF - (best & 0xFFFFFF)

    ii = np.arange(nini)
    ibox = np.stack([(dx * (ii % gx)).astype(np.int64), (dy * (ii // gx)).astype(np.int64),
                     (dx * (ii % gx + 1)).astype(np.int64), (dy * (ii // gx + 1)).astype(np.int64)], 1)
    act = np.nonzero(cc > 1)[0]                    # ascending: sweep 1 walks the initial nodes front to back
    nidx = np.full(nini, -1); nidx[act] = np.arange(len(act))
    leaf = cc[k0] == 1
    fin_key += list(0x80000000 + k0[leaf]); fin_cand += list(idx[leaf])
    node = np.where(leaf, -1, nidx[k0])
    box = ibox[act]; cnt = cc[act]; ser = act.copy()
    Lsize = int((cc > 0).sum()); sb = nini; m = len(act)

    def count_children():
        live = node >= 0
        cx, cy = _centre(box)
        q = np.zeros(n, np.int64)
        q[live] = (cx[node[live]] <= x[live]).astype(np.int64) + 2 * (cy[node[live]] <= y[live]).astype(np.int64)
        c = np.bincount(4 * node[live] + q[live], minlength=4 * m)
        return q, c

    def build_next(c4):
        nonlocal box, cnt, ser, node
        big = np.nonzero(c4 > 1)[0][::-1]          # descending child index = descending serial
        nid = np.full(4 * m, -1); nid[big] = np.arange(len(big))
        live = node >= 0
        ch = np.where(live, 4 * node + quad, 0)
        leafc = live & (c4[ch] == 1)
        fin_key.extend(list(0x7FFFFFFF - (sb + ch[leafc]))); fin_cand.extend(list(idx[leafc]))
        newnode = np.where(live & ~leafc, nid[ch], -1)
        nbox = _child_boxes(box[big >> 2], big & 3)
        box, cnt, ser = nbox, c4[big], sb + big
        node = newnode
        return len(big)

    phase_b = False
    while True:                                    # phase A: whole-list sweeps
        if m == 0:
            break
        prev = Lsize
        quad, c4 = count_children()
        ne = int((c4 > 0).sum())
        m_old = m
        pl = build_next(c4)
        Lsize = Lsize - m_old + ne; sb += 4 * m_old; m = pl
        if N <= Lsize or Lsize == prev:
            break
        if N < Lsize + 3 * m:
            phase_b = True
            break
    while phase_b:                                 # phase B: largest nodes first, stop at the budget
        if m == 0:
            break
        if stats is not None:
            stats["pool_m"] = max(stats["pool_m"], m)
        prev = Lsize
        order = np.lexsort((np.arange(m), -cnt))   # (count desc, serial desc) == (count desc, index asc)
        rank = np.empty(m, np.int64); rank[order] = np.arange(m)
        box, cnt, ser = box[order], cnt[order], ser[order]
        node = np.where(node >= 0, rank[np.maximum(node, 0)], -1)
        quad, c4 = count_children()
        ne_r = (c4.reshape(m, 4) > 0).sum(1)
        P = np.cumsum(ne_r - 1)
        hit = np.nonzero(Lsize + P >= N)[0]
        if len(hit):
            p = int(hit[0])
            live = node >= 0
            fid = np.where(node <= p, 4 * node + quad, 4 * m + node)
            best = best_of(fid[live], live, 5 * m)
            for f in range(4 * (p + 1)):
                if c4[f] > 0:
                    fin_key.append(0x7FFFFFFF - (sb + f)); fin_cand.append(best[f])
            for r in range(p + 1, m):
                fin_key.append(0x7FFFFFFF - ser[r]); fin_cand.append(best[4 * m + r])
            Lsize += int(P[p]); m = 0
            break
        m_old = m
        pl = build_next(c4)
        Lsize += int(P[-1]); sb += 4 * m_old; m = pl
        if Lsize == prev:
            break
    if m:                                          # nodes never split: best response of each
        live = node >= 0
        best = best_of(node[live], live, m)
        for r in range(m):
            fin_key.append((0x7FFFFFFF - ser[r]) if ser[r] >= nini else (0x80000000 + ser[r])); fin_cand.append(best[r])
    if stats is not None:
        stats["nfin"] = len(fin_key)
    fk = np.asarray(fin_key, np.int64); fc = np.asarray(fin_cand, np.int64)
    assert len(np.unique(fk)) == len(fk)
    return fc[np.argsort(fk)]
