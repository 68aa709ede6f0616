"""Plain sequential numpy restatement of the grid-windowed matchers (match::projection, match::area) and of
match::angle_checker, written from their documented semantics, plus the named cases that the oracle
(tests/test_window_match_reference.py) and the GPU (tests/test_window_match_reference_gpu.py) are both held to.

Semantics restated here (float32 wherever the matchers compute in float):
  grid       data::get_cell_indices: cx = floor((x - min_x) * inv_cell_width), likewise cy; a keypoint outside
             [0, cols) x [0, rows) (or not finite) is in no cell.  Keypoints are visited cell by cell, cx major and cy
             minor, in index order inside a cell.
  window     data::frame::get_keypoints_in_cell: cells floor((ref - min - margin) * inv) .. ceil((ref - min + margin) * inv),
             clipped to the grid; strict box |kp - ref| < margin on both axes; level gate kp.octave >= min_level
             (active when min_level > 0) and kp.octave <= max_level (active when max_level >= 0); the x_right test
             |q.x_right - kp.x_right| <= margin only where the keypoint's 0 < x_right.
  matchers   a sequential scan over the window in visiting order, `d < best` (first visited wins ties), with the
             per-matcher thresholds, ratio tests and "a keypoint is taken once" bookkeeping documented on each function.

Besides the matches each matcher returns a Counter of the events its case is meant to reach: boundary hits of the window,
threshold decisions, and -- modelled on the documented replay of match_window.cu (top-4 list per query from one GPU
search, then a sequential replay that re-queries when the list cannot decide) -- how often the replay lands in each
undecided branch.  The cases assert these counts, so a case that stops reaching its edge fails."""
from collections import Counter
from fractions import Fraction

import numpy as np

THR_LOW = 50
THR_HIGH = 100
MAX_DIST = 256
TOPK = 4
F32 = np.float32

_POPCOUNT = np.array([bin(i).count("1") for i in range(256)], np.int64)


def hamming(q, D):
    """Hamming distances between one 32-byte descriptor q and the rows of D."""
    return _POPCOUNT[np.bitwise_xor(D, q)].sum(axis=1)


# ----------------------------------------------------------------------------------------------- frame and grid
class Grid:
    """camera::base image bounds -> the keypoint grid (inverse cell sizes computed in double, stored as float)."""

    def __init__(self, min_x, max_x, min_y, max_y, cols=64, rows=48):
        self.bounds = (float(min_x), float(max_x), float(min_y), float(max_y))
        self.min_x, self.min_y = F32(min_x), F32(min_y)
        self.inv_w = F32(float(cols) / (float(max_x) - float(min_x)))
        self.inv_h = F32(float(rows) / (float(max_y) - float(min_y)))
        self.cols, self.rows = int(cols), int(rows)

    def args(self):
        """Arguments of match.camera_grid / oracle.om_grid."""
        return self.bounds + (self.cols, self.rows)


class Frame:
    """The matcher's view of a frame: keypoints (x, y, octave, angle, x_right or None), descriptors, grid."""

    def __init__(self, x, y, octave, angle, x_right, desc, grid):
        self.x = np.ascontiguousarray(x, F32); self.y = np.ascontiguousarray(y, F32)
        self.octave = np.ascontiguousarray(octave, np.int32); self.angle = np.ascontiguousarray(angle, F32)
        self.x_right = None if x_right is None else np.ascontiguousarray(x_right, F32)
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        self.grid = grid
        self.n = len(self.x)
        g = grid
        with np.errstate(invalid="ignore", over="ignore"):
            fx = (self.x - g.min_x) * g.inv_w
            fy = (self.y - g.min_y) * g.inv_h
        ok = np.isfinite(fx) & np.isfinite(fy)
        cx = np.full(self.n, -1, np.int64); cy = np.full(self.n, -1, np.int64)
        cx[ok] = np.floor(fx[ok].astype(np.float64)); cy[ok] = np.floor(fy[ok].astype(np.float64))
        ok &= (0 <= cx) & (cx < g.cols) & (0 <= cy) & (cy < g.rows)
        idx = np.flatnonzero(ok)
        order = np.lexsort((idx, cy[idx], cx[idx]))       # cx major, cy minor, index order inside a cell
        self.rank_to_idx = idx[order]
        cell = cx[self.rank_to_idx] * g.rows + cy[self.rank_to_idx]
        self.cell_start = np.searchsorted(cell, np.arange(g.cols * g.rows + 1))
        r = self.rank_to_idx
        self.sx, self.sy, self.soct = self.x[r], self.y[r], self.octave[r]
        self.sxr = None if self.x_right is None else self.x_right[r]
        self.sdesc = self.desc[r]
        self.in_grid = ok


def window(f, ref_x, ref_y, margin, min_level, max_level, q_xr=None, stats=None):
    """get_keypoints_in_cell (+ the x_right test when q_xr is given and the frame has x_right): the candidates' ranks in
    visiting order.  stats counts the boundary events of the query."""
    g = f.grid
    ref_x, ref_y, margin = F32(ref_x), F32(ref_y), F32(margin)
    with np.errstate(invalid="ignore", over="ignore"):
        lo_x = ((ref_x - g.min_x) - margin) * g.inv_w
        hi_x = ((ref_x - g.min_x) + margin) * g.inv_w
        lo_y = ((ref_y - g.min_y) - margin) * g.inv_h
        hi_y = ((ref_y - g.min_y) + margin) * g.inv_h
    if stats is not None:
        stats["cell_edge_exact"] += sum(bool(np.isfinite(v) and v == np.floor(v)) for v in (lo_x, hi_x, lo_y, hi_y))
    min_cx = max(0, int(np.floor(np.float64(lo_x))))
    max_cx = min(g.cols - 1, int(np.ceil(np.float64(hi_x))))
    min_cy = max(0, int(np.floor(np.float64(lo_y))))
    max_cy = min(g.rows - 1, int(np.ceil(np.float64(hi_y))))
    if g.cols <= min_cx or max_cx < 0 or g.rows <= min_cy or max_cy < 0:
        if stats is not None:
            stats["window_off_grid"] += 1
        return np.zeros(0, np.int64)
    if stats is not None and (min_cx == 0 or min_cy == 0 or max_cx == g.cols - 1 or max_cy == g.rows - 1):
        stats["window_clipped"] += 1
    cs = f.cell_start
    ranges = [(cs[cx * g.rows + min_cy], cs[cx * g.rows + max_cy + 1]) for cx in range(min_cx, max_cx + 1)]
    ranks = np.concatenate([np.arange(a, b) for a, b in ranges]) if ranges else np.zeros(0, np.int64)
    if len(ranks) == 0:
        return ranks
    o = f.soct[ranks]
    keep = np.ones(len(ranks), bool)
    if 0 < min_level or 0 <= max_level:
        keep &= o >= min_level
        if 0 <= max_level:
            keep &= o <= max_level
    dx = np.abs(f.sx[ranks] - ref_x); dy = np.abs(f.sy[ranks] - ref_y)
    if stats is not None:
        stats["box_edge_exact"] += int(np.sum(keep & (((dx == margin) & (dy <= margin)) | ((dy == margin) & (dx <= margin)))))
        # one float step of the keypoint coordinate away from the edge, inside the box
        in_x = (dx < margin) & (margin - dx <= np.spacing(np.abs(f.sx[ranks])))
        in_y = (dy < margin) & (margin - dy <= np.spacing(np.abs(f.sy[ranks])))
        stats["box_edge_inside"] += int(np.sum(keep & ((in_x & (dy < margin)) | (in_y & (dx < margin)))))
        if 0 < min_level or 0 <= max_level:
            box = (dx < margin) & (dy < margin)
            stats["level_edge_in"] += int(np.sum(box & ((o == min_level) | (o == max_level))))
            stats["level_edge_out"] += int(np.sum(box & ((o == min_level - 1) | ((0 <= max_level) & (o == max_level + 1)))))
    keep &= (dx < margin) & (dy < margin)
    if q_xr is not None and f.sxr is not None:
        kxr = f.sxr[ranks]
        err = np.abs(F32(q_xr) - kxr)
        tested = keep & (F32(0) < kxr)
        if stats is not None:
            step_up = F32(np.nextafter(margin, F32(np.inf)))
            stats["xr_edge_equal"] += int(np.sum(tested & (err == margin)))
            stats["xr_edge_above"] += int(np.sum(tested & (err == step_up)))
            stats["xr_untested_nonpositive"] += int(np.sum(keep & (kxr <= 0)))
        keep &= ~(tested & (margin < err))
    return ranks[keep]


def _topk(d, ranks):
    """The GPU search's per-query list: the 4 smallest (distance, rank) keys."""
    order = np.lexsort((ranks, d))[:TOPK]
    return d[order], ranks[order]


def _replay_branch(stats, name, lst_d, lst_idx, valid, thr, ratio_hi=None):
    """Models the replay in match_window.cu (resolve()): which branch the GPU's top-4 list of this query takes once the
    keypoints taken by earlier queries are removed.  ratio_hi(best, lower_bound) -> True when the ratio test needs the true
    second best."""
    exhausted = len(lst_d) < TOPK
    vd = [d for d, i in zip(lst_d, lst_idx) if valid(i, d)]
    lb = MAX_DIST if exhausted else int(lst_d[TOPK - 1])
    if len(vd) >= 2 or exhausted:
        return
    if len(vd) == 1 and ratio_hi is not None and vd[0] <= thr and ratio_hi(vd[0], lb):
        stats[name + "_requery_r1"] += 1
    elif len(vd) == 0 and lb <= thr:
        stats[name + "_requery_r0"] += 1
        if lb == thr:
            stats[name + "_requery_r0_at_thr"] += 1     # the lower bound sits exactly on the threshold


# ----------------------------------------------------------------------------------------------- angle_checker
def angle_bins(deltas):
    d = np.asarray(deltas, F32).copy()
    neg = d < 0.0
    d[neg] = (d[neg].astype(np.float64) + 360.0).astype(F32)
    big = 360.0 <= d
    d[big] = (d[big].astype(np.float64) - 360.0).astype(F32)
    r = np.rint(d * F32(F32(1.0) / F32(30))).astype(np.int64)      # lrintf: round half to even
    return (r & 0xFFFFFFFF) % 30                                       # unsigned modulo, as the C code


def angle_checker_invalid(deltas):
    """match::angle_checker<int>(30, 3): keep the three fullest bins (ties: lower bin first); a runner-up bin holding fewer
    than 0.1f * the fullest bin's count is dropped with every bin after it."""
    b = angle_bins(deltas)
    count = np.bincount(b, minlength=30)
    order = np.argsort(-count, kind="stable")
    keep = np.zeros(30, bool)
    top = count[order[0]] if len(b) else 0
    for r in range(3):
        if r > 0 and F32(count[order[r]]) < F32(0.1) * F32(top):
            break
        keep[order[r]] = True
    return ~keep[b]


# ----------------------------------------------------------------------------------------------- matchers
def match_frame_and_landmarks(f, scale_factors, reproj_xy, x_right_in_tracking, pred_level, lm_desc, lm_usable=None,
                              kp_has_observed_lm=None, margin=5.0, lowe_ratio=0.6):
    """projection::match_frame_and_landmarks: each usable landmark in order searches margin * scale_factors[level] over the
    levels [level - 1, level] among keypoints without a landmark; best <= THR_HIGH; the ratio test best > ratio * second
    rejects only when best and second-best keypoints have the same octave; the keypoint then has a landmark (first taker)."""
    sf = np.asarray(scale_factors, F32)
    ratio = F32(lowe_ratio)
    st = Counter()
    has = np.zeros(f.n, bool) if kp_has_observed_lm is None else np.asarray(kp_has_observed_lm).astype(bool).copy()
    has_rank = has[f.rank_to_idx]
    out = np.full(f.n, -1, np.int32)
    lists = []
    for l in range(len(pred_level)):
        if lm_usable is not None and not lm_usable[l]:
            continue
        lvl = int(pred_level[l])
        m = F32(margin) * sf[lvl]
        qxr = None
        if f.x_right is not None:
            qxr = F32(-1.0) if x_right_in_tracking is None else F32(x_right_in_tracking[l])
        ranks = window(f, reproj_xy[l][0], reproj_xy[l][1], m, lvl - 1, lvl, qxr, st)
        st["pred_level_%d" % lvl] += 1
        ranks0 = ranks[~has_rank[ranks]] if len(ranks) else ranks
        lists.append((l, ranks, _topk(hamming(lm_desc[l], f.sdesc[ranks0]), ranks0) if len(ranks0) else ([], [])))
    n = 0
    for l, ranks, (ld, lr) in lists:
        _replay_branch(st, "lm", ld, lr, lambda r, d: not has_rank[r], THR_HIGH,
                       lambda b, lb: F32(b) > ratio * F32(lb))
        ranks = ranks[~has_rank[ranks]] if len(ranks) else ranks
        if len(ranks) == 0:
            st["no_candidate"] += 1
            continue
        d = hamming(lm_desc[l], f.sdesc[ranks])
        ok = d < MAX_DIST
        ranks, d = ranks[ok], d[ok]
        if len(ranks) == 0:
            continue
        order = np.argsort(d, kind="stable")
        best, b_r = int(d[order[0]]), ranks[order[0]]
        if best > THR_HIGH:
            st["thr_high_reject"] += 1
            continue
        if best == THR_HIGH:
            st["thr_high_equal"] += 1
        if len(order) > 1:
            second, s_r = int(d[order[1]]), ranks[order[1]]
            same = f.soct[b_r] == f.soct[s_r]
            rejects = F32(best) > ratio * F32(second)
            if best == Fraction(str(lowe_ratio)) * second:
                st["ratio_exact_same" if same else "ratio_exact_diff"] += 1
            if rejects and not same:
                st["ratio_spared_by_level"] += 1
            if same and rejects:
                st["ratio_reject"] += 1
                continue
        out[f.rank_to_idx[b_r]] = l
        has_rank[b_r] = True
        n += 1
    st["matches"] = n
    return n, out, st


def match_best(f, ref_xy, ref_x_right, margin, min_level, max_level, q_angle, q_desc, usable=None, kp_unavailable=None,
               hamm_dist_thr=THR_HIGH, check_orientation=True):
    """The loop behind current_and_last, frame_and_keyframe and Sim3: each usable query in order takes the nearest still
    available keypoint of its window when best <= hamm_dist_thr; then the angle histogram drops the matches outside the
    dominant rotations.  The x_right test applies when the frame has x_right and ref_x_right is given."""
    st = Counter()
    taken = np.zeros(f.n, bool) if kp_unavailable is None else np.asarray(kp_unavailable).astype(bool).copy()
    taken_rank = taken[f.rank_to_idx]
    out = np.full(f.n, -1, np.int32)
    thr = int(hamm_dist_thr)
    lists = []
    for q in range(len(margin)):
        if usable is not None and not usable[q]:
            continue
        qxr = None if (ref_x_right is None or f.x_right is None) else ref_x_right[q]
        ranks = window(f, ref_xy[q][0], ref_xy[q][1], margin[q], int(min_level[q]), int(max_level[q]), qxr, st)
        ranks0 = ranks[~taken_rank[ranks]] if len(ranks) else ranks
        lists.append((q, ranks, _topk(hamming(q_desc[q], f.sdesc[ranks0]), ranks0) if len(ranks0) else ([], [])))
    deltas, dkp = [], []
    n = 0
    for q, ranks, (ld, lr) in lists:
        _replay_branch(st, "best", ld, lr, lambda r, d: not taken_rank[r], thr)
        ranks = ranks[~taken_rank[ranks]] if len(ranks) else ranks
        if len(ranks) == 0:
            st["no_candidate"] += 1
            continue
        d = hamming(q_desc[q], f.sdesc[ranks])
        ok = d < MAX_DIST
        ranks, d = ranks[ok], d[ok]
        if len(ranks) == 0:
            continue
        j = int(np.argmin(d))
        if d[j] > thr:
            st["thr_reject"] += 1
            continue
        if d[j] == thr:
            st["thr_equal"] += 1
        if np.sum(d == d[j]) > 1:
            st["tie_first_wins"] += 1
        i = f.rank_to_idx[ranks[j]]
        out[i] = q
        taken_rank[ranks[j]] = True
        n += 1
        if check_orientation:
            deltas.append(F32(q_angle[q]) - f.angle[i]); dkp.append(i)
    if check_orientation and deltas:
        inv = angle_checker_invalid(np.array(deltas, F32))
        for k in np.flatnonzero(inv):
            out[dkp[k]] = -1
            n -= 1
        st["orientation_dropped"] += int(inv.sum())
    st["matches"] = n
    return n, out, st


def match_current_and_last_frames(f, scale_factors, num_scale_levels, last_usable, reproj_xy, reproj_x_right, last_level, last_angle,
                                  lm_desc, kp_has_observed_lm=None, margin=20.0, assume_forward=False, assume_backward=False,
                                  check_orientation=True):
    """projection::match_current_and_last_frames: margin * scale_factors[level]; levels [level, top] forward, [0, level]
    backward, else [level - 1, level + 1]; THR_HIGH; the x_right test whenever the current frame has x_right (a missing
    reprojected x_right is -1)."""
    sf = np.asarray(scale_factors, F32)
    lv = np.asarray(last_level, np.int64)
    mg = np.where(last_usable.astype(bool), F32(margin) * sf[np.clip(lv, 0, len(sf) - 1)], F32(0)).astype(F32)
    if assume_forward:
        lo, hi = lv, np.full(len(lv), num_scale_levels - 1)
    elif assume_backward:
        lo, hi = np.zeros(len(lv), np.int64), lv
    else:
        lo, hi = lv - 1, lv + 1
    xr = reproj_x_right
    if xr is None and f.x_right is not None:
        xr = np.full(len(lv), -1, F32)
    return match_best(f, reproj_xy, xr, mg, lo, hi, last_angle, lm_desc, last_usable, kp_has_observed_lm, THR_HIGH, check_orientation)


def match_frame_and_keyframe(f, scale_factors, reproj_xy, pred_level, keyfrm_angle, lm_desc, usable, kp_has_lm, margin, hamm_dist_thr,
                             check_orientation=True):
    """projection::match_frame_and_keyframe: margin * scale_factors[level], levels [level - 1, level + 1]."""
    lv = np.asarray(pred_level, np.int64)
    mg = (F32(margin) * np.asarray(scale_factors, F32)[lv]).astype(F32)
    return match_best(f, reproj_xy, None, mg, lv - 1, lv + 1, keyfrm_angle, lm_desc, usable, kp_has_lm, hamm_dist_thr, check_orientation)


def match_by_Sim3_transform(f, scale_factors, reproj_xy, pred_level, lm_desc, usable, kp_already_matched, margin):
    """projection::match_by_Sim3_transform: margin * scale_factors[level], levels [level - 1, level], THR_LOW, no orientation check."""
    lv = np.asarray(pred_level, np.int64)
    mg = (F32(margin) * np.asarray(scale_factors, F32)[lv]).astype(F32)
    return match_best(f, reproj_xy, None, mg, lv - 1, lv, np.zeros(len(lv), F32), lm_desc, usable, kp_already_matched, THR_LOW, False)


def match_in_consistent_area(f2, octave_1, angle_1, desc_1, prev_matched_xy, margin=100, lowe_ratio=0.9, check_orientation=True):
    """area::match_in_consistent_area: only the level-0 keypoints of frame 1 search, in index order, the window `margin` at
    level 0 of frame 2.  A frame-2 keypoint already matched at distance c is a candidate only at d < c, and is then taken
    from its earlier query.  Accepted at best <= THR_LOW and second * ratio >= best (no level condition).  The angle
    histogram counts every accepted match, also those later taken away.  No x_right test."""
    ratio = F32(lowe_ratio)
    st = Counter()
    n1 = len(octave_1)
    prev = np.array(prev_matched_xy, F32).copy()
    out = np.full(n1, -1, np.int32)
    cap = np.full(f2.n, MAX_DIST, np.int64)            # matched distance, per frame-2 keypoint index
    owner = np.full(f2.n, -1, np.int64)
    lists = []
    for i in range(n1):
        if 0 < octave_1[i]:
            continue
        lvl = int(octave_1[i])
        ranks = window(f2, prev[i, 0], prev[i, 1], F32(margin), lvl, lvl, None, st)
        lists.append((i, ranks, _topk(hamming(desc_1[i], f2.sdesc[ranks]), ranks) if len(ranks) else ([], [])))
    deltas, didx = [], []
    n = 0
    for i, ranks, (ld, lr) in lists:
        cap_rank = cap[f2.rank_to_idx]
        _replay_branch(st, "area", ld, lr, lambda r, d: d < cap_rank[r], THR_LOW, lambda b, lb: F32(lb) * ratio < F32(b))
        if len(ranks) == 0:
            continue
        d = hamming(desc_1[i], f2.sdesc[ranks])
        ok = d < cap_rank[ranks]
        if not ok.all():
            st["area_capped_out"] += 1
        ranks, d = ranks[ok], d[ok]
        if len(ranks) == 0:
            continue
        order = np.argsort(d, kind="stable")
        best = int(d[order[0]])
        second = int(d[order[1]]) if len(order) > 1 else MAX_DIST
        if best > THR_LOW:
            st["thr_low_reject"] += 1
            continue
        if best == THR_LOW:
            st["thr_low_equal"] += 1
        if F32(second) * ratio < F32(best):
            st["ratio_reject"] += 1
            continue
        if best == Fraction(str(lowe_ratio)) * second:
            st["ratio_exact"] += 1
        j = f2.rank_to_idx[ranks[order[0]]]
        if owner[j] >= 0:
            out[owner[j]] = -1
            n -= 1
            st["area_reassigned"] += 1
        out[i] = j
        owner[j] = i
        cap[j] = best
        n += 1
        if check_orientation:
            deltas.append(F32(angle_1[i]) - f2.angle[j]); didx.append(i)
    if check_orientation and deltas:
        inv = angle_checker_invalid(np.array(deltas, F32))
        for k in np.flatnonzero(inv):
            if out[didx[k]] >= 0:
                out[didx[k]] = -1
                n -= 1
                st["orientation_dropped"] += 1
    st["matches"] = n
    ok = out >= 0
    prev[ok, 0] = f2.x[out[ok]]; prev[ok, 1] = f2.y[out[ok]]
    return n, out, prev, st


def window_topk(f, ref_xy, margin, min_level, max_level, q_desc, x_right_q=None):
    """The 4 best candidates of every query in visiting order (-1 / 256 where absent) and the boundary-event counts."""
    st = Counter()
    nq = len(margin)
    idx = np.full((nq, TOPK), -1, np.int32); dist = np.full((nq, TOPK), MAX_DIST, np.int32)
    for q in range(nq):
        qxr = None if x_right_q is None else x_right_q[q]
        ranks = window(f, ref_xy[q][0], ref_xy[q][1], margin[q], int(min_level[q]), int(max_level[q]), qxr, st)
        if len(ranks):
            d, r = _topk(hamming(q_desc[q], f.sdesc[ranks]), ranks)
            idx[q, :len(r)] = f.rank_to_idx[r]; dist[q, :len(d)] = d
    return idx, dist, st


# ----------------------------------------------------------------------------------------------- case construction
def flip_bits(desc, k, rng):
    """desc with exactly k distinct bits flipped (distance k)."""
    out = np.array(desc, np.uint8).copy()
    bits = rng.choice(256, k, replace=False)
    for b in bits:
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def scale_factors(scale_factor=1.2, num_levels=8):
    """The scale factors of an 8-level 1.2 pyramid, as the benchmark passes them."""
    return np.array([scale_factor ** i for i in range(num_levels)], F32)


class Case:
    """A frame plus the matcher calls to run on it.  calls: list of (kind, kwargs); kinds are 'landmarks', 'current_and_last',
    'frame_and_keyframe', 'sim3', 'best', 'area', 'topk', 'angles'.  expect: list of (call number, stat name, minimum)."""

    def __init__(self, name, frame, calls, expect):
        self.name, self.frame, self.calls, self.expect = name, frame, calls, expect


def run_reference(case, kind, kw):
    f = case.frame
    if kind == "landmarks":
        return match_frame_and_landmarks(f, **kw)
    if kind == "current_and_last":
        return match_current_and_last_frames(f, **kw)
    if kind == "frame_and_keyframe":
        return match_frame_and_keyframe(f, **kw)
    if kind == "sim3":
        return match_by_Sim3_transform(f, **kw)
    if kind == "best":
        return match_best(f, **kw)
    if kind == "area":
        return match_in_consistent_area(f, **kw)
    if kind == "topk":
        return window_topk(f, **kw)
    if kind == "angles":
        inv = angle_checker_invalid(kw["deltas"])
        return (inv, Counter(kept=int((~inv).sum())))
    raise ValueError(kind)


def run_oracle(O, case, kind, kw):
    """The same call on the C oracle (oracle/match_oracle.c); returns the reference's tuple without the stats."""
    f = case.frame
    fo = O.MatchFrame(f.x, f.y, f.octave, f.angle, f.x_right, f.desc, O.om_grid(*f.grid.args()))
    if kind == "landmarks":
        k = dict(kw)
        xr = k.pop("x_right_in_tracking")
        if xr is None and f.x_right is not None:
            xr = np.full(len(k["pred_level"]), -1, F32)
        return O.projection_match_frame_and_landmarks(fo, k["scale_factors"], k["reproj_xy"], xr, k["pred_level"], k["lm_desc"],
                                                      k.get("lm_usable"), k.get("kp_has_observed_lm"), k.get("margin", 5.0), k.get("lowe_ratio", 0.6))
    if kind == "current_and_last":
        k = dict(kw)
        xr = k["reproj_x_right"]
        if xr is None and f.x_right is not None:
            xr = np.full(len(k["last_level"]), -1, F32)
        return O.projection_match_current_and_last(fo, k["scale_factors"], k["num_scale_levels"], k["last_usable"], k["reproj_xy"], xr,
                                                   k["last_level"], k["last_angle"], k["lm_desc"], k.get("kp_has_observed_lm"),
                                                   k.get("margin", 20.0), k.get("assume_forward", False), k.get("assume_backward", False),
                                                   k.get("check_orientation", True))
    if kind == "frame_and_keyframe":
        lv = np.asarray(kw["pred_level"], np.int32)
        mg = F32(kw["margin"]) * np.asarray(kw["scale_factors"], F32)[lv]
        return O.projection_match_best(fo, kw["reproj_xy"], None, mg, lv - 1, lv + 1, kw["keyfrm_angle"], kw["lm_desc"], kw["usable"],
                                       kw["kp_has_lm"], kw["hamm_dist_thr"], kw.get("check_orientation", True))
    if kind == "sim3":
        lv = np.asarray(kw["pred_level"], np.int32)
        mg = F32(kw["margin"]) * np.asarray(kw["scale_factors"], F32)[lv]
        return O.projection_match_best(fo, kw["reproj_xy"], None, mg, lv - 1, lv, np.zeros(len(lv), F32), kw["lm_desc"], kw["usable"],
                                       kw["kp_already_matched"], THR_LOW, False)
    if kind == "best":
        return O.projection_match_best(fo, kw["ref_xy"], kw["ref_x_right"], kw["margin"], kw["min_level"], kw["max_level"], kw["q_angle"],
                                       kw["q_desc"], kw.get("usable"), kw.get("kp_unavailable"), kw.get("hamm_dist_thr", THR_HIGH),
                                       kw.get("check_orientation", True))
    if kind == "area":
        f1 = O.MatchFrame(np.zeros(len(kw["octave_1"]), F32), np.zeros(len(kw["octave_1"]), F32), kw["octave_1"], kw["angle_1"], None,
                          kw["desc_1"], O.om_grid(*f.grid.args()))
        return O.area_match_in_consistent_area(f1, fo, kw["prev_matched_xy"], kw.get("margin", 100), kw.get("lowe_ratio", 0.9),
                                               kw.get("check_orientation", True))
    if kind == "topk":
        nq = len(kw["margin"])
        idx = np.full((nq, TOPK), -1, np.int32); dist = np.full((nq, TOPK), MAX_DIST, np.int32)
        for q in range(nq):
            cand = O.get_keypoints_in_cell(fo, kw["ref_xy"][q][0], kw["ref_xy"][q][1], kw["margin"][q], kw["min_level"][q], kw["max_level"][q])
            d = np.array([O.hamming(kw["q_desc"][q], f.desc[c]) for c in cand], np.int64)
            order = np.argsort(d, kind="stable")[:TOPK]
            idx[q, :len(order)] = cand[order]; dist[q, :len(order)] = d[order]
        return idx, dist
    if kind == "angles":
        return (O.angle_checker_invalid(kw["deltas"]),)
    raise ValueError(kind)


# ----------------------------------------------------------------------------------------------- the named cases
W0, H0 = 752, 480
SF = scale_factors()


def _lattice(k, step=40, pad=30, W=W0, H=H0):
    per_row = (W - 2 * pad) // step + 1
    return F32(pad + step * (k % per_row)), F32(pad + step * (k // per_row))


def _landmarks_like_bench(kps, desc, n_total, W, H, rng):
    """bench.py make_landmark_sets: one landmark per keypoint (within sigma 2 px, level = octave, a few bits flipped), the
    rest uniform with unrelated descriptors, in a permuted map order."""
    n = len(kps)
    xy = np.stack([kps["x"], kps["y"]], 1).astype(F32) + rng.normal(0, 2.0, (n, 2)).astype(F32)
    d = desc.copy()
    flip = rng.integers(0, 256, d.shape, dtype=np.uint8) & rng.integers(0, 256, d.shape, dtype=np.uint8) & rng.integers(0, 256, d.shape, dtype=np.uint8)
    d ^= flip & rng.integers(0, 256, d.shape, dtype=np.uint8)
    level = kps["octave"].astype(np.int32); angle = kps["angle"].astype(F32)
    extra = max(0, n_total - n)
    if extra:
        xy = np.concatenate([xy, np.stack([rng.uniform(0, W, extra), rng.uniform(0, H, extra)], 1).astype(F32)])
        d = np.concatenate([d, rng.integers(0, 256, (extra, 32), dtype=np.uint8)])
        level = np.concatenate([level, rng.integers(0, 8, extra).astype(np.int32)])
        angle = np.concatenate([angle, rng.uniform(0, 360, extra).astype(F32)])
        perm = rng.permutation(len(xy))
        xy, d, level, angle = xy[perm], d[perm], level[perm], angle[perm]
    return np.ascontiguousarray(xy), np.ascontiguousarray(d), np.ascontiguousarray(level), np.ascontiguousarray(angle)


def bench4(kps, desc, seed=17):
    """Config 4's projection match: 20 000 landmarks into a 4000-keypoint 1920 x 960 frame, margin 5, levels 0-7."""
    W, H = 1920, 960
    f = Frame(kps["x"], kps["y"], kps["octave"], kps["angle"], None, desc, Grid(0, W, 0, H))
    xy, d, level, _ = _landmarks_like_bench(kps, desc, 20000, W, H, np.random.default_rng(seed))
    kw = dict(scale_factors=SF, reproj_xy=xy, x_right_in_tracking=None, pred_level=level, lm_desc=d, margin=5.0, lowe_ratio=0.6)
    expect = [(0, "no_candidate", 10000), (0, "matches", len(kps) // 2), (0, "ratio_reject", 1)] + \
             [(0, "pred_level_%d" % l, 100) for l in range(8)]
    return Case("bench4", f, [("landmarks", kw)], expect)


def bench2(kps_last, desc_last, kps_cur, desc_cur, seed=17):
    """Config 2's tracking match: the last frame's keypoints (1000, 752 x 480) reprojected into the current frame,
    current_and_last at margin 20 with the orientation check."""
    f = Frame(kps_cur["x"], kps_cur["y"], kps_cur["octave"], kps_cur["angle"], None, desc_cur, Grid(0, W0, 0, H0))
    xy, d, level, angle = _landmarks_like_bench(kps_last, desc_last, 0, W0, H0, np.random.default_rng(seed))
    kw = dict(scale_factors=SF, num_scale_levels=8, last_usable=np.ones(len(xy), np.uint8), reproj_xy=xy, reproj_x_right=None,
              last_level=level, last_angle=angle, lm_desc=d, margin=20.0)
    return Case("bench2", f, [("current_and_last", kw)], [(0, "matches", len(kps_cur) // 2), (0, "orientation_dropped", 1)])


def offset_grid(seed=31):
    """Grid bounds of undistorted perspective images: negative min_x / min_y, non-integer cell sizes.  Keypoints outside
    the grid (beyond either bound, at max_y, at -1e6 as non-converged undistortion returns, NaN) are in no cell; at max_x
    float rounding puts the keypoint in the last column (63.999996).  Queries whose cell-range arguments are exact integers."""
    rng = np.random.default_rng(seed)
    g = Grid(-13.37, 765.1, -7.9, 489.2)
    n = 700
    x = rng.uniform(-13.37, 765.1, n).astype(F32); y = rng.uniform(-7.9, 489.2, n).astype(F32)
    specials = [(-13.5, 100.0), (766.0, 200.0), (765.1, 300.0), (300.0, 489.2), (-1e6, -1e6), (np.nan, 200.0), (200.0, np.nan),
                (-13.37, 50.0), (400.0, -7.9), (765.1, 489.2)]
    sx = np.array([s[0] for s in specials], F32); sy = np.array([s[1] for s in specials], F32)
    x = np.concatenate([x, sx]); y = np.concatenate([y, sy])
    N = len(x)
    octv = rng.integers(0, 8, N).astype(np.int32); ang = rng.uniform(0, 360, N).astype(F32)
    desc = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    f = Frame(x, y, octv, ang, None, desc, g)
    assert list(f.in_grid[n:]) == [False, False, True, False, False, False, False, True, True, False]
    # queries: near random keypoints, at the specials, and with exact-integer cell-range arguments
    sel = rng.integers(0, n, 300)
    ref = [(x[i] + rng.normal(0, 3), y[i] + rng.normal(0, 3)) for i in sel] + [(a + 1.0, b - 1.0) for a, b in specials if np.isfinite(a + b)]
    margin = list(rng.choice([3.0, 9.5, 25.0], len(ref)))
    qd = [flip_bits(desc[i], int(rng.integers(0, 30)), rng) for i in sel] + [flip_bits(desc[n + k], 3, rng) for k, (a, b) in enumerate(specials)
                                                                            if np.isfinite(a + b)]
    for k in range(40):
        m = F32(rng.choice([4.0, 12.0, 30.0]))
        cx = int(rng.integers(2, 60)); cy = int(rng.integers(2, 45))
        rx = F32(g.min_x + m + F32(cx) / g.inv_w)
        for _ in range(64):   # walk to a float whose cell-range argument is exactly cx
            v = ((rx - g.min_x) - m) * g.inv_w
            if v == cx:
                break
            rx = F32(np.nextafter(rx, F32(np.inf) if v < cx else F32(-np.inf)))
        ry = F32(g.min_y - m + F32(cy) / g.inv_h)
        for _ in range(64):
            v = ((ry - g.min_y) + m) * g.inv_h
            if v == cy:
                break
            ry = F32(np.nextafter(ry, F32(np.inf) if v < cy else F32(-np.inf)))
        ref.append((rx, ry)); margin.append(m); qd.append(rng.integers(0, 256, 32, dtype=np.uint8))
    ref = np.array(ref, F32); margin = np.array(margin, F32); qd = np.array(qd, np.uint8)
    nq = len(ref)
    lo = np.full(nq, -1, np.int32); hi = np.full(nq, -1, np.int32)
    calls = [("topk", dict(ref_xy=ref, margin=margin, min_level=lo, max_level=hi, q_desc=qd)),
             ("best", dict(ref_xy=ref, ref_x_right=None, margin=margin, min_level=lo, max_level=hi, q_angle=np.zeros(nq, F32), q_desc=qd,
                           hamm_dist_thr=THR_HIGH, check_orientation=False))]
    return Case("offset_grid", f, calls, [(0, "cell_edge_exact", 60), (1, "matches", 100)])


def window_edges(seed=32):
    """Windows clipped at each border and corner, wholly off the grid, margins of one cell and of more than ten, and
    keypoints at exactly |d| = margin (outside) and one float step inside it."""
    rng = np.random.default_rng(seed)
    n = 600
    x = rng.uniform(0, W0, n).astype(F32); y = rng.uniform(0, H0, n).astype(F32)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    ref, margin, qd = [], [], []
    # clipped and off-grid windows
    for rx, ry in [(2, 240), (750, 240), (376, 2), (376, 478), (1, 1), (751, 1), (1, 479), (751, 479), (-10, 240), (760, 470),
                   (-100, 240), (900, 240), (376, -100), (376, 700), (-100, -100), (-31, 240)]:
        for m in (5.0, 20.0):
            ref.append((rx, ry)); margin.append(m); qd.append(rng.integers(0, 256, 32, dtype=np.uint8))
    # one cell (cell width 11.75) and more than ten cells
    for k in range(30):
        i = int(rng.integers(0, n))
        ref.append((x[i] + 0.5, y[i] - 0.5)); margin.append(5.0 if k % 2 else 130.0); qd.append(flip_bits(desc[i], 40, rng))
    # exact box edges: dyadic coordinates, so that |kp - ref| is exactly the margin or one float step inside it
    ex, ey, ed = [], [], []
    for k in range(24):
        cxq, cyq = _lattice(k, step=60, pad=40)
        rx, ry, m = F32(cxq + 0.5), F32(cyq + 0.25), F32(7.25)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        inside = [F32(np.nextafter(rx + m, F32(0))), F32(np.nextafter(rx - m, F32(np.inf)))]
        side = k % 4
        if side == 0:
            pts = [(rx + m, ry), (inside[0], ry + 1)]
        elif side == 1:
            pts = [(rx - m, ry), (inside[1], ry - 1)]
        elif side == 2:
            pts = [(rx, ry + m), (rx + 1, F32(np.nextafter(ry + m, F32(0))))]
        else:
            pts = [(rx + m, ry - m), (rx - 2, F32(np.nextafter(ry - m, F32(np.inf))))]
        for j, (px, py) in enumerate(pts):
            ex.append(px); ey.append(py); ed.append(flip_bits(base, 2 + 3 * j, rng))   # the excluded one would be the best
        ref.append((rx, ry)); margin.append(m); qd.append(base)
    x = np.concatenate([x, np.array(ex, F32)]); y = np.concatenate([y, np.array(ey, F32)]); desc = np.concatenate([desc, np.array(ed, np.uint8)])
    N = len(x)
    f = Frame(x, y, rng.integers(0, 8, N), rng.uniform(0, 360, N), None, desc, Grid(0, W0, 0, H0))
    ref = np.array(ref, F32); margin = np.array(margin, F32); qd = np.array(qd, np.uint8)
    nq = len(ref)
    lo = np.full(nq, -1, np.int32); hi = np.full(nq, -1, np.int32)
    calls = [("topk", dict(ref_xy=ref, margin=margin, min_level=lo, max_level=hi, q_desc=qd)),
             ("best", dict(ref_xy=ref, ref_x_right=None, margin=margin, min_level=lo, max_level=hi, q_angle=np.zeros(nq, F32), q_desc=qd,
                           hamm_dist_thr=THR_HIGH, check_orientation=False))]
    return Case("window_edges", f, calls, [(0, "box_edge_exact", 24), (0, "box_edge_inside", 24), (0, "window_off_grid", 10),
                                           (0, "window_clipped", 20), (1, "matches", 24)])


def levels(seed=33):
    """Keypoints on every octave around each query; predicted level 0 (min_level -1) to 7; forward [lvl, 7], backward
    [0, lvl] and [lvl - 1, lvl + 1].  The nearest descriptors sit on the octaves just outside each level range."""
    rng = np.random.default_rng(seed)
    x, y, octv, desc = [], [], [], []
    qxy, qlvl, qd = [], [], []
    for k in range(64):
        cx, cy = _lattice(k, step=60, pad=40)
        lvl = k % 8
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        for o in range(8):
            gap = min(abs(o - (lvl - 2)), abs(o - (lvl + 2)), abs(o - (lvl + 1)))   # octaves next to the ranges are the nearest
            x.append(cx + rng.uniform(-3, 3)); y.append(cy + rng.uniform(-3, 3)); octv.append(o)
            desc.append(flip_bits(base, 4 + 3 * gap + o % 2, rng))
        qxy.append((cx, cy)); qlvl.append(lvl); qd.append(base)
    x = np.array(x, F32); y = np.array(y, F32); N = len(x)
    f = Frame(x, y, np.array(octv, np.int32), rng.uniform(0, 360, N), None, np.array(desc, np.uint8), Grid(0, W0, 0, H0))
    qxy = np.array(qxy, F32); qlvl = np.array(qlvl, np.int32); qd = np.array(qd, np.uint8); nq = len(qlvl)
    mg = (F32(5.0) * SF[qlvl]).astype(F32)
    cal = dict(scale_factors=SF, num_scale_levels=8, last_usable=np.ones(nq, np.uint8), reproj_xy=qxy, reproj_x_right=None,
               last_level=qlvl, last_angle=np.zeros(nq, F32), lm_desc=qd, margin=5.0, check_orientation=False)
    calls = [("landmarks", dict(scale_factors=SF, reproj_xy=qxy, x_right_in_tracking=None, pred_level=qlvl, lm_desc=qd, margin=5.0, lowe_ratio=0.9)),
             ("current_and_last", dict(cal)),
             ("current_and_last", dict(cal, assume_forward=True)),
             ("current_and_last", dict(cal, assume_backward=True)),
             ("topk", dict(ref_xy=qxy, margin=mg, min_level=qlvl - 1, max_level=qlvl, q_desc=qd)),
             ("topk", dict(ref_xy=qxy, margin=mg, min_level=qlvl, max_level=np.full(nq, 7, np.int32), q_desc=qd)),
             ("topk", dict(ref_xy=qxy, margin=mg, min_level=np.zeros(nq, np.int32), max_level=qlvl, q_desc=qd))]
    expect = [(c, s, 40) for c in range(len(calls)) for s in ("level_edge_in", "level_edge_out")] + \
             [(0, "pred_level_0", 8), (0, "pred_level_7", 8)]
    return Case("levels", f, calls, expect)


def thresholds(seed=34):
    """One query per scenario, each in a window of its own: single candidates at distances 49/50/51 and 99/100/101, and
    best / second pairs at exactly ratio x second (0.6: 30/50, 60/100; 0.8: 40/50; 0.9: 45/50) and just beyond it, once
    with equal octaves and once with different ones."""
    rng = np.random.default_rng(seed)
    x, y, octv, desc = [], [], [], []
    qxy, qd = [], []
    scen = [(d,) for d in (49, 50, 51, 99, 100, 101)]
    for b, s in [(30, 50), (60, 100), (40, 50), (45, 50), (31, 50), (61, 100), (41, 50), (46, 50), (20, 50)]:
        scen += [(b, s, True), (b, s, False)]
    for k, sc in enumerate(scen):
        cx, cy = _lattice(k, step=50, pad=40)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        qxy.append((cx, cy)); qd.append(base)
        if len(sc) == 1:
            x.append(cx + 1.0); y.append(cy - 1.0); octv.append(0); desc.append(flip_bits(base, sc[0], rng))
        else:
            b, s, same = sc
            for dd, o, off in [(s, 0 if same else 1, -1.5), (b, 0, 1.5)]:     # the second best is visited first
                x.append(cx + off); y.append(cy + 0.5); octv.append(o); desc.append(flip_bits(base, dd, rng))
    x = np.array(x, F32); y = np.array(y, F32); N = len(x)
    f = Frame(x, y, np.array(octv, np.int32), np.zeros(N, F32), None, np.array(desc, np.uint8), Grid(0, W0, 0, H0))
    qxy = np.array(qxy, F32); qd = np.array(qd, np.uint8); nq = len(qxy)
    lv = np.ones(nq, np.int32)          # levels [0, 1], margin 5 * 1.2
    calls, expect = [], []
    for r in (0.6, 0.8, 0.9):
        calls.append(("landmarks", dict(scale_factors=SF, reproj_xy=qxy, x_right_in_tracking=None, pred_level=lv, lm_desc=qd, margin=5.0, lowe_ratio=r)))
        expect += [(len(calls) - 1, "ratio_exact_same", 1), (len(calls) - 1, "ratio_exact_diff", 1), (len(calls) - 1, "ratio_reject", 1),
                   (len(calls) - 1, "ratio_spared_by_level", 1), (len(calls) - 1, "thr_high_equal", 1), (len(calls) - 1, "thr_high_reject", 1)]
        calls.append(("area", dict(octave_1=np.zeros(nq, np.int32), angle_1=np.zeros(nq, F32), desc_1=qd, prev_matched_xy=qxy, margin=5,
                                   lowe_ratio=r, check_orientation=False)))
        expect += [(len(calls) - 1, "ratio_exact", 1), (len(calls) - 1, "ratio_reject", 1), (len(calls) - 1, "thr_low_equal", 1),
                   (len(calls) - 1, "thr_low_reject", 1)]
    for thr in (THR_LOW, THR_HIGH):
        calls.append(("best", dict(ref_xy=qxy, ref_x_right=None, margin=np.full(nq, 5.0, F32), min_level=np.full(nq, -1, np.int32),
                                   max_level=np.full(nq, -1, np.int32), q_angle=np.zeros(nq, F32), q_desc=qd, hamm_dist_thr=thr, check_orientation=False)))
        expect += [(len(calls) - 1, "thr_equal", 1), (len(calls) - 1, "thr_reject", 1)]
    calls.append(("sim3", dict(scale_factors=SF, reproj_xy=qxy, pred_level=lv, lm_desc=qd, usable=None, kp_already_matched=None, margin=5.0)))
    expect += [(len(calls) - 1, "thr_equal", 1), (len(calls) - 1, "thr_reject", 1)]
    return Case("thresholds", f, calls, expect)


def ties(seed=35):
    """Many candidates at one distance, laid out so that visiting order (cell by cell) differs from index order: the
    first visited wins, and the second best -- whose octave decides whether the ratio test applies -- is the first visited
    of the tied runners-up."""
    rng = np.random.default_rng(seed)
    x, y, octv, desc = [], [], [], []
    qxy, qd = [], []
    for k in range(40):
        cx, cy = _lattice(k, step=60, pad=40)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        qxy.append((cx, cy)); qd.append(base)
        if k % 2 == 0:      # six keypoints at one distance, indices in reverse visiting order
            for j in range(6):
                x.append(cx + 14.0 - 5.5 * j); y.append(cy + (j % 3) - 1.0); octv.append(j % 2); desc.append(flip_bits(base, 20, rng))
        else:               # a unique best, then tied runners-up on different octaves (which one is visited first alternates)
            first_o = (k // 2) % 2
            x.append(cx + 12.0); y.append(cy); octv.append(1); desc.append(flip_bits(base, 10, rng))
            x.append(cx + 5.0); y.append(cy + 1.0); octv.append(1 - first_o); desc.append(flip_bits(base, 16, rng))
            x.append(cx - 12.0); y.append(cy - 1.0); octv.append(first_o); desc.append(flip_bits(base, 16, rng))
    x = np.array(x, F32); y = np.array(y, F32); N = len(x)
    f = Frame(x, y, np.array(octv, np.int32), np.zeros(N, F32), None, np.array(desc, np.uint8), Grid(0, W0, 0, H0))
    qxy = np.array(qxy, F32); qd = np.array(qd, np.uint8); nq = len(qxy)
    lv = np.ones(nq, np.int32)
    mg = np.full(nq, 16.0, F32)
    calls = [("landmarks", dict(scale_factors=SF, reproj_xy=qxy, x_right_in_tracking=None, pred_level=lv, lm_desc=qd, margin=14.0, lowe_ratio=0.8)),
             ("best", dict(ref_xy=qxy, ref_x_right=None, margin=mg, min_level=np.full(nq, -1, np.int32), max_level=np.full(nq, -1, np.int32),
                           q_angle=np.zeros(nq, F32), q_desc=qd, hamm_dist_thr=THR_HIGH, check_orientation=False)),
             ("topk", dict(ref_xy=qxy, margin=mg, min_level=np.full(nq, -1, np.int32), max_level=np.full(nq, -1, np.int32), q_desc=qd)),
             ("area", dict(octave_1=np.zeros(nq, np.int32), angle_1=np.zeros(nq, F32), desc_1=qd, prev_matched_xy=qxy, margin=16, lowe_ratio=0.7,
                           check_orientation=False))]
    return Case("ties", f, calls, [(0, "ratio_spared_by_level", 5), (0, "ratio_reject", 5), (1, "tie_first_wins", 15), (3, "matches", 5)])


def contention(seed=36, lowe_ratio=0.8):
    """Few keypoints, many queries with near-identical descriptors: the GPU's top-4 lists run out on keypoints taken by
    earlier queries, so every replay must reach its undecided branches and re-query."""
    rng = np.random.default_rng(seed)
    x, y, octv, desc = [], [], [], []
    qxy, qd = [], []
    for k in range(12):
        cx, cy = _lattice(k, step=80, pad=60)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        for j in range(9):
            x.append(cx + rng.uniform(-3, 3)); y.append(cy + rng.uniform(-3, 3)); octv.append(j % 2)
            desc.append(flip_bits(base, int(rng.integers(1, 12)), rng))
        for j in range(24):
            qxy.append((cx + rng.uniform(-1, 1), cy + rng.uniform(-1, 1))); qd.append(flip_bits(base, int(rng.integers(1, 12)), rng))
    # the list's 4th distance exactly at the threshold: four earlier queries take the four listed keypoints (distance 0
    # each), the last query's list then holds only taken keypoints, and the keypoint after them -- at the threshold too --
    # is found only by the re-query
    for k, dists in [(12, (90, 95, 98, THR_HIGH, THR_HIGH)), (13, (40, 45, 48, THR_LOW, THR_LOW))]:
        cx, cy = _lattice(k, step=80, pad=60)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        kd = [flip_bits(base, dd, rng) for dd in dists]
        for j, d_ in enumerate(kd):
            x.append(cx - 4.0 + 2.0 * j); y.append(cy); octv.append(0); desc.append(d_)
        for j in range(4):
            qxy.append((cx, cy)); qd.append(kd[j])
        qxy.append((cx, cy)); qd.append(base)
    x = np.array(x, F32); y = np.array(y, F32); N = len(x)
    f = Frame(x, y, np.array(octv, np.int32), rng.uniform(0, 360, N), None, np.array(desc, np.uint8), Grid(0, W0, 0, H0))
    qxy = np.array(qxy, F32); qd = np.array(qd, np.uint8); nq = len(qxy)
    lv = np.ones(nq, np.int32)
    calls = [("landmarks", dict(scale_factors=SF, reproj_xy=qxy, x_right_in_tracking=None, pred_level=lv, lm_desc=qd, margin=8.0, lowe_ratio=lowe_ratio)),
             ("best", dict(ref_xy=qxy, ref_x_right=None, margin=np.full(nq, 8.0, F32), min_level=np.zeros(nq, np.int32), max_level=lv,
                           q_angle=np.zeros(nq, F32), q_desc=qd, hamm_dist_thr=THR_HIGH, check_orientation=False)),
             ("area", dict(octave_1=np.zeros(nq, np.int32), angle_1=np.zeros(nq, F32), desc_1=qd, prev_matched_xy=qxy, margin=8, lowe_ratio=0.9,
                           check_orientation=False))]
    expect = [(0, "lm_requery_r1", 1), (0, "lm_requery_r0", 1), (0, "lm_requery_r0_at_thr", 1), (1, "best_requery_r0", 1),
              (1, "best_requery_r0_at_thr", 1), (2, "area_requery_r1", 1), (2, "area_requery_r0", 1), (2, "area_requery_r0_at_thr", 1),
              (2, "area_reassigned", 1)]
    return Case("contention", f, calls, expect)


def _angle_sets():
    """Delta-angle multisets, one histogram each: rounding of exact float halves (15, 135, 255 -> even bins 0, 4, 8; 45 ->
    bin 2), -0.0, -1e-6 (360.0f after the wrap, then bin 0), equal counts in different bins (lower bin first), and
    runner-up bins at exactly a tenth of the top count and one below it."""
    sets = [[0.0] * 10 + [60.0] * 8 + [120.0] * 6 + [15.0, 135.0, 45.0],
            [240.0] * 10 + [0.0] * 8 + [60.0] * 6 + [255.0, -0.0, -1e-6, 15.0],
            [90.0] * 5 + [210.0] * 5 + [330.0] * 5 + [600.0 - 360.0 - 90.0] * 5 + [-1e-6] * 2,
            [3.0] * 5 + [-3.0] * 5 + [30.0] * 5 + [180.0] * 5]
    for top in (30, 50, 70):
        sets.append([0.0] * top + [150.0] * (top // 10) + [300.0] * (top // 10 - 1))
        sets.append([0.0] * top + [150.0] * (top // 10) + [300.0] * (top // 10) + [90.0] * (top // 10))
    return [np.array(s, F32) for s in sets]


def angles(seed=37):
    """The angle histogram through match_best: one query per keypoint (distance 0), keypoint angle 0 and query angle =
    the delta, so each call's histogram is exactly one of the delta sets."""
    rng = np.random.default_rng(seed)
    sets = _angle_sets()
    n = max(len(s) for s in sets)
    pts = [_lattice(k, step=24, pad=12) for k in range(n)]
    x = np.array([p[0] for p in pts], F32); y = np.array([p[1] for p in pts], F32)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    f = Frame(x, y, np.zeros(n, np.int32), np.zeros(n, F32), None, desc, Grid(0, W0, 0, H0))
    calls, expect = [], []
    for s in sets:
        m = len(s)
        calls.append(("angles", dict(deltas=s)))
        calls.append(("best", dict(ref_xy=np.stack([x[:m] + 0.5, y[:m]], 1), ref_x_right=None, margin=np.full(m, 4.0, F32),
                                   min_level=np.full(m, -1, np.int32), max_level=np.full(m, -1, np.int32), q_angle=s, q_desc=desc[:m],
                                   hamm_dist_thr=THR_HIGH, check_orientation=True)))
        # the first two sets keep every match (their probes land in the three kept bins); the others drop some
        expect.append((len(calls) - 1, "matches", m) if len(calls) <= 4 else (len(calls) - 1, "orientation_dropped", 1))
    return Case("angles", f, calls, expect)


def x_right(seed=38):
    """A stereo frame: around each query a keypoint with x_right -1, one with 0 (neither is tested), one with x_right 1.0,
    the query's x_right error to it exactly the margin or one float step either side, and the nearest descriptor on a
    keypoint with x_right 64 far from the query's.  The area matcher has no x_right test, so that one is its match."""
    rng = np.random.default_rng(seed)
    m = F32(5.0)
    errs = [m, F32(np.nextafter(m, F32(np.inf))), F32(np.nextafter(m, F32(0)))]
    x, y, xr, desc = [], [], [], []
    qxy, qxr, qd = [], [], []
    for k in range(30):
        cx, cy = _lattice(k, step=60, pad=40)
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        for j, (kxr, dd) in enumerate([(F32(1.0), 5), (F32(-1.0), 10), (F32(0.0), 12), (F32(64.0), 3)]):
            x.append(cx + j - 1.0); y.append(cy + 0.5); xr.append(kxr); desc.append(flip_bits(base, dd, rng))
        e = errs[k % 3]
        qxy.append((cx, cy)); qxr.append(F32(1.0) + e if k % 2 else F32(1.0) - e); qd.append(base)
    x = np.array(x, F32); N = len(x)
    f = Frame(x, np.array(y, F32), np.zeros(N, np.int32), np.zeros(N, F32), np.array(xr, F32), np.array(desc, np.uint8), Grid(0, W0, 0, H0))
    qxy = np.array(qxy, F32); qxr = np.array(qxr, F32); qd = np.array(qd, np.uint8); nq = len(qxy)
    z = np.zeros(nq, np.int32)
    calls = [("landmarks", dict(scale_factors=SF, reproj_xy=qxy, x_right_in_tracking=qxr, pred_level=z, lm_desc=qd, margin=5.0, lowe_ratio=0.9)),
             ("current_and_last", dict(scale_factors=SF, num_scale_levels=8, last_usable=np.ones(nq, np.uint8), reproj_xy=qxy, reproj_x_right=qxr,
                                       last_level=z, last_angle=np.zeros(nq, F32), lm_desc=qd, margin=5.0, check_orientation=False)),
             ("best", dict(ref_xy=qxy, ref_x_right=qxr, margin=np.full(nq, m, F32), min_level=z - 1, max_level=z + 1, q_angle=np.zeros(nq, F32),
                           q_desc=qd, hamm_dist_thr=THR_HIGH, check_orientation=False)),
             ("area", dict(octave_1=z, angle_1=np.zeros(nq, F32), desc_1=qd, prev_matched_xy=qxy, margin=5, lowe_ratio=0.9, check_orientation=False))]
    expect = [(c, s, 5) for c in range(3) for s in ("xr_edge_equal", "xr_edge_above", "xr_untested_nonpositive")] + [(3, "matches", 25)]
    return Case("x_right", f, calls, expect)


SYNTHETIC_CASES = {c.__name__: c for c in (offset_grid, window_edges, levels, thresholds, ties, contention, angles, x_right)}
