"""Plain sequential numpy restatement of the compute of match::fuse::replace_duplication (DESIGN.md section 5, f16): the geometry
of every queried landmark in its target keyframe, then the target's windowed search.  It shares no code with oracle/ or csrc/; the
window is window_match_reference's restatement of get_keypoints_in_cell.

Semantics restated here (float32 wherever the reference computes in float):
  geometry   not finite -> rejected; camera reproject_to_image; dist = sqrt((x^2 + y^2) + z^2) of pos_w - cam_center in double
             against (float)(0.7 min_valid_dist) and (float)(1.3 max_valid_dist) compared in double; ((v.x n.x + v.y n.y) + v.z n.z)
             < 0.5 dist rejects; the level is predict_scale_level((float)dist).
  window     margin = f32(margin) * scale_factors[level], octaves level - 1 .. level, no x_right margin test.
  gate       ex = ref.x - kp.x, ey = ref.y - kp.y; a keypoint is stereo when its x_right >= 0 (so -0.0 and 0.0 are stereo, unlike
             the projection matcher's 0 < x_right), er = query x_right - kp x_right; rejected when ((ex^2 + ey^2) + er^2) * w >
             CHI_SQ_3D, or (ex^2 + ey^2) * w > CHI_SQ_2D without a stereo keypoint, w = inv_level_sigma_sq[kp octave].
  choice     the nearest descriptor, d < best in visiting order (the first visited wins a tie), accepted at best <= THR_LOW.

Every query also returns a Counter of the edges it reached; the named cases at the end of this module assert them."""
import functools
from collections import Counter

import numpy as np

import tracking_reference as REF
import window_match_reference as WR

F32 = np.float32
THR_LOW = WR.THR_LOW
MAX_DIST = WR.MAX_DIST
# The chi-square bounds of the fuse gate as float32 (ORB-SLAM2's values; see DESIGN.md section 5, f16: an unpinned recollection)
CHI_SQ_2D = F32(5.99)
CHI_SQ_3D = F32(7.8)


def fuse_observe_reference(g, pos_w, mean_normal, min_valid_dist, max_valid_dist):
    """-> passed (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32, pred_level (n,) i32: not finite -> rejected; reproject_to_image;
    dist = sqrt((x^2 + y^2) + z^2) in double against the float bounds (float)(0.7 min) and (float)(1.3 max) compared in double;
    ((v.x n.x + v.y n.y) + v.z n.z) < 0.5 dist rejects; predict_scale_level((float)dist)."""
    P = np.asarray(pos_w, np.float64).reshape(-1, 3)
    N = np.asarray(mean_normal, np.float64).reshape(-1, 3)
    lo_raw = np.asarray(min_valid_dist, np.float32); hi_raw = np.asarray(max_valid_dist, np.float32)
    ok, uv, xr = REF.reproject(g, P)
    C = np.array(g.cam_center[:], np.float64)
    with np.errstate(all="ignore"):
        ok &= np.isfinite(P).all(1) & np.isfinite(uv).all(1)
        v = P - C
        dist = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
        lo = (0.7 * lo_raw.astype(np.float64)).astype(np.float32).astype(np.float64)
        hi = (1.3 * hi_raw.astype(np.float64)).astype(np.float32).astype(np.float64)
        ok &= ~((dist < lo) | (hi < dist))
        dot = (v[:, 0] * N[:, 0] + v[:, 1] * N[:, 1]) + v[:, 2] * N[:, 2]
        ok &= ~(dot < 0.5 * dist)
        level = REF.predict_scale_level(dist.astype(np.float32), hi_raw, g.log_scale_factor, g.num_scale_levels)
    return (ok, np.where(ok[:, None], uv, np.float32(0)).astype(np.float32), np.where(ok, xr, np.float32(0)).astype(np.float32),
            np.where(ok, level, 0).astype(np.int32))


class Target:
    """One target keyframe: its frame_geometry, scale_factors_ and inv_level_sigma_sq_, keypoints (x, y, octave, descriptors,
    stereo x_right or None) and its grid (window_match_reference.Grid, any bounds, cols and rows)."""

    def __init__(self, geometry, scale_factors, inv_level_sigma_sq, x, y, octave, desc, grid, x_right=None):
        self.geometry = geometry
        self.scale_factors = np.ascontiguousarray(scale_factors, F32)
        self.inv_level_sigma_sq = np.ascontiguousarray(inv_level_sigma_sq, F32)
        assert len(self.scale_factors) == len(self.inv_level_sigma_sq) == geometry.num_scale_levels
        n = len(x)
        self.frame = WR.Frame(x, y, octave, np.zeros(n, F32), x_right, desc, grid)
        self.n = n


def _gate(f, ranks, ref_x, ref_y, q_xr, w_table, st):
    """The chi-square gate on the candidates `ranks` of one query -> boolean mask of those kept, counting its edges."""
    if len(ranks) == 0:
        return np.zeros(0, bool)
    ex = ref_x - f.sx[ranks]; ey = ref_y - f.sy[ranks]
    w = w_table[f.soct[ranks]]
    e2 = ex * ex + ey * ey
    kxr = f.sxr[ranks] if f.sxr is not None else np.full(len(ranks), F32(-1))
    stereo = kxr >= F32(0)
    er = q_xr - kxr
    p3 = (e2 + er * er) * w
    p2 = e2 * w
    keep = np.where(stereo, ~(p3 > CHI_SQ_3D), ~(p2 > CHI_SQ_2D))
    st["chi2_mono_equal"] += int(np.sum(~stereo & (p2 == CHI_SQ_2D)))
    st["chi2_mono_above"] += int(np.sum(~stereo & (p2 == np.nextafter(CHI_SQ_2D, F32(np.inf)))))
    st["chi2_stereo_equal"] += int(np.sum(stereo & (p3 == CHI_SQ_3D)))
    st["chi2_stereo_above"] += int(np.sum(stereo & (p3 == np.nextafter(CHI_SQ_3D, F32(np.inf)))))
    st["chi2_rejected"] += int(np.sum(~keep))
    if f.sxr is not None:
        st["xr_stereo"] += int(np.sum(stereo))
        st["xr_mono"] += int(np.sum(~stereo))
        st["xr_negative_zero"] += int(np.sum((kxr == 0) & np.signbit(kxr)))
        st["xr_positive_zero"] += int(np.sum((kxr == 0) & ~np.signbit(kxr)))
        st["xr_min_positive"] += int(np.sum(kxr == np.nextafter(F32(0), F32(1))))
        st["xr_minus_one"] += int(np.sum(kxr == F32(-1)))
        # candidates whose stereo test decides differently from the monocular one: the x_right >= 0 rule matters there
        st["xr_decides"] += int(np.sum(stereo & ((p3 > CHI_SQ_3D) != (p2 > CHI_SQ_2D))))
    return keep


def search_one(t, ref_xy, q_xr, level, qdesc, margin, st=None):
    """The fuse matching core for one query that passed the geometry -> (keypoint index or -1, Counter)."""
    st = Counter() if st is None else st
    f = t.frame
    ref_x, ref_y = F32(ref_xy[0]), F32(ref_xy[1])
    level = int(level)
    m = F32(F32(margin) * t.scale_factors[level])
    st["pred_level_%d" % level] += 1
    if level == 0:
        st["pred_level_zero"] += 1
    if level == len(t.scale_factors) - 1:
        st["pred_level_top"] += 1
    ranks = WR.window(f, ref_x, ref_y, m, level - 1, level, None, st)
    # the octaves just outside the level range, inside the box (the same window with the range widened by one on each side)
    wide = WR.window(f, ref_x, ref_y, m, level - 2, level + 1, None)
    if len(wide):
        ow = f.soct[wide]
        st["level_out_low"] += int(np.sum(ow == level - 2))
        st["level_out_high"] += int(np.sum(ow == level + 1))
    if len(ranks):
        o = f.soct[ranks]
        st["level_in_low"] += int(np.sum(o == level - 1))
        st["level_in_high"] += int(np.sum(o == level))
    keep = _gate(f, ranks, ref_x, ref_y, F32(q_xr), t.inv_level_sigma_sq, st)
    ranks = ranks[keep]
    if len(ranks) == 0:
        st["no_candidate"] += 1
        return -1, st
    d = WR.hamming(qdesc, f.sdesc[ranks])
    best, j = MAX_DIST, -1
    for k in range(len(ranks)):          # visiting order, d < best: the first visited wins a tie
        if d[k] < best:
            best, j = int(d[k]), k
    if j < 0:
        return -1, st
    ties = np.flatnonzero(d == best)
    if len(ties) > 1:
        st["tie"] += 1
        idx = f.rank_to_idx[ranks[ties]]
        if idx[0] > idx[1:].min():
            st["tie_winner_higher_index"] += 1
        cell = lambda r: (int(np.floor(np.float64((f.sx[r] - f.grid.min_x) * f.grid.inv_w))),
                          int(np.floor(np.float64((f.sy[r] - f.grid.min_y) * f.grid.inv_h))))
        if any(cell(ranks[k]) != cell(ranks[ties[0]]) for k in ties[1:]):
            st["tie_across_cells"] += 1
            if idx[0] > idx[1:].min():
                st["tie_across_cells_winner_higher_index"] += 1
        else:
            st["tie_within_cell"] += 1
    if best > THR_LOW:
        st["hamming_rejected"] += 1
        if best == THR_LOW + 1:
            st["hamming_51_rejected"] += 1
        return -1, st
    if best == THR_LOW:
        st["hamming_50_accepted"] += 1
    r = int(ranks[j])
    if r >= 1 << 15:
        st["rank_ge_32768"] += 1
    if r >= 65280:
        st["rank_ge_65280"] += 1
    st["fused"] += 1
    return int(f.rank_to_idx[r]), st


def search(t, passed, reproj_xy, x_right, pred_level, lm_desc, margin):
    """ovs_fuse_best_keypoints_host's semantics for one target with a stereo query x_right: -> (best_idx (nq,), [Counter])"""
    nq = len(passed)
    best = np.full(nq, -1, np.int32)
    stats = []
    for q in range(nq):
        st = Counter()
        if passed[q]:
            best[q], _ = search_one(t, reproj_xy[q], x_right[q], pred_level[q], lm_desc[q], margin, st)
        stats.append(st)
    return best, stats


def replace_duplication(t, lms, q_lm, margin=3.0):
    """One target and its queries q_lm (landmark row or -1) -> (num_fused, best_idx, passed, reproj_xy, x_right, pred_level, [Counter])."""
    q_lm = np.asarray(q_lm, np.int64)
    nq = len(q_lm)
    rows = np.maximum(q_lm, 0)
    if nq and len(lms["pos_w"]):
        ok, uv, xr, lv = fuse_observe_reference(t.geometry, lms["pos_w"][rows], lms["mean_normal"][rows], lms["min_valid_dist"][rows],
                                                lms["max_valid_dist"][rows])
    else:
        ok, uv, xr, lv = np.zeros(nq, bool), np.zeros((nq, 2), F32), np.zeros(nq, F32), np.zeros(nq, np.int32)
    ok &= q_lm >= 0
    uv = np.where(ok[:, None], uv, F32(0)).astype(F32); xr = np.where(ok, xr, F32(0)).astype(F32); lv = np.where(ok, lv, 0).astype(np.int32)
    desc = np.asarray(lms["lm_desc"], np.uint8).reshape(-1, 32)[rows] if nq else np.zeros((0, 32), np.uint8)
    best, stats = search(t, ok, uv, xr, lv, desc, margin)
    for q in range(nq):
        if q_lm[q] < 0:
            stats[q]["query_skipped"] += 1
        elif not np.isfinite(np.asarray(lms["pos_w"][q_lm[q]], np.float64)).all():
            stats[q]["position_not_finite"] += 1
        elif not ok[q]:
            stats[q]["not_observed"] += 1
    return int((best >= 0).sum()), best, ok, uv, xr, lv, stats


# ----------------------------------------------------------------------------------------------- case construction
def _f32_steps(v, k):
    """the 2k + 1 float32 values v - k ulps .. v + k ulps (v > 0)"""
    b = np.asarray(F32(v)).reshape(1).view(np.int32)[0]
    return (b + np.arange(-k, k + 1, dtype=np.int32)).view(F32)


class _TargetBuilder:
    """A target keyframe under construction: identity pose, a perspective camera (fx = fy = 500 about (cx, cy), stereo with a
    focal_x_baseline) or a 1920 x 960 equirectangular one, its own scale table, grid bounds, cols and rows."""

    def __init__(self, model="perspective", stereo=False, num_levels=8, scale_factor=1.2, bounds=(0.0, 640.0, 0.0, 480.0), cols=64, rows=48,
                 cx=320.0, cy=240.0, fb=386.1448):
        from openvslam_b200.match import frame_geometry
        from openvslam_b200.optimize import camera
        self.model, self.stereo = model, stereo
        if model == "equirectangular":
            bounds = (0.0, 1920.0, 0.0, 960.0)
            cam = camera("equirectangular", cols=1920.0, rows=960.0)
        else:
            cam = camera("perspective", fx=500.0, fy=500.0, cx=cx, cy=cy, focal_x_baseline=fb if stereo else 0.0)
        self.cx, self.cy, self.scale_factor = cx, cy, scale_factor
        self.sf = np.array([scale_factor ** i for i in range(num_levels)], F32)
        self.inv = (1.0 / (self.sf.astype(np.float64) ** 2)).astype(F32)
        self.geometry = frame_geometry(cam, bounds, np.concatenate([np.eye(3).reshape(9), np.zeros(3)]), num_levels, F32(np.log(scale_factor)))
        self.grid = WR.Grid(*bounds, cols=cols, rows=rows)
        self.x, self.y, self.oct, self.desc, self.xr = [], [], [], [], []
        self.queries = []

    def kp(self, x, y, octave, desc, xr=-1.0):
        self.x.append(F32(x)); self.y.append(F32(y)); self.oct.append(int(octave)); self.desc.append(np.asarray(desc, np.uint8))
        self.xr.append(F32(xr))
        return len(self.x) - 1

    def build(self):
        n = len(self.x)
        desc = np.array(self.desc, np.uint8).reshape(n, 32)
        xr = np.array(self.xr, F32) if self.stereo else None
        return Target(self.geometry, self.sf, self.inv, np.array(self.x, F32), np.array(self.y, F32), np.array(self.oct, np.int32), desc,
                      self.grid, xr)


class _Scene:
    """Landmark table and targets of one case."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.pos, self.nrm, self.lo, self.hi, self.desc = [], [], [], [], []
        self.targets = []

    def target(self, **kw):
        t = _TargetBuilder(**kw)
        self.targets.append(t)
        return t

    def landmark(self, p, level, sf, desc=None, nrm=None):
        p = np.asarray(p, np.float64)
        dist = float(np.linalg.norm(p))
        self.pos.append(p)
        self.nrm.append(p / dist if nrm is None else np.asarray(nrm, np.float64))
        self.lo.append(F32(dist))
        self.hi.append(F32(dist * float(sf) ** (level - 0.25)))
        self.desc.append(self.rng.integers(0, 256, 32, dtype=np.uint8) if desc is None else np.asarray(desc, np.uint8))
        return len(self.pos) - 1

    def reprojection(self, t, ref_x, ref_y):
        """where a landmark queried at (ref_x, ref_y) into t lands (reproj_xy, x_right), without adding it"""
        row = self.query(t, ref_x, ref_y, 1)[0]
        t.queries.pop()
        p = [a.pop() for a in (self.pos, self.nrm, self.lo, self.hi, self.desc)]
        _, uv, xr, _ = fuse_observe_reference(t.geometry, p[0][None], p[1][None], [p[2]], [p[3]])
        return uv[0], xr[0]

    def query(self, t, ref_x, ref_y, level, z=4.0, exact=True, row=None):
        """A landmark seen by t at about (ref_x, ref_y) with predicted level `level` (or the existing landmark `row`), queried into
        t -> (row, (u, v) f32, x_right f32, level) from the reference geometry.  exact: a perspective reprojection must land on
        (ref_x, ref_y) exactly."""
        row_given = row is not None
        if row is None:
            if t.model == "equirectangular":
                lon = (float(ref_x) / 1920.0 - 0.5) * 2.0 * np.pi; lat = (float(ref_y) / 960.0 - 0.5) * np.pi
                p = z * np.array([np.sin(lon) * np.cos(lat), np.sin(lat), np.cos(lon) * np.cos(lat)])
            else:
                p = np.array([(float(F32(ref_x)) - t.cx) / 500.0 * z, (float(F32(ref_y)) - t.cy) / 500.0 * z, z])
            row = self.landmark(p, level, t.scale_factor)
        ok, uv, xr, lv = fuse_observe_reference(t.geometry, self.pos[row][None], self.nrm[row][None], [self.lo[row]], [self.hi[row]])
        if row_given:
            pass
        elif t.model != "equirectangular" and exact:
            assert ok[0] and uv[0, 0] == F32(ref_x) and uv[0, 1] == F32(ref_y), (ref_x, ref_y, uv)
        if ok[0] and not row_given:
            assert lv[0] == min(level, len(t.sf) - 1), (level, lv)
        t.queries.append(row)
        return row, uv[0], xr[0], int(lv[0])

    def case(self, name, margin, expect, small=True):
        lms = dict(pos_w=np.array(self.pos, np.float64).reshape(-1, 3), mean_normal=np.array(self.nrm, np.float64).reshape(-1, 3),
                   min_valid_dist=np.array(self.lo, F32), max_valid_dist=np.array(self.hi, F32),
                   lm_desc=np.array(self.desc, np.uint8).reshape(-1, 32))
        q_off = np.concatenate([[0], np.cumsum([len(t.queries) for t in self.targets])]).astype(np.int32)
        q_lm = np.array([r for t in self.targets for r in t.queries], np.int32)
        return Case(name, [t.build() for t in self.targets], [t.model == "equirectangular" for t in self.targets], lms, q_off, q_lm, margin,
                    expect, small)


class Case:
    """targets ([Target]), equirect (per target), the landmark table lms, the CSR queries q_off / q_lm, the margin, and expect:
    {edge counter: minimum over the whole case}.  small: cheap enough for the grid-free window check."""

    def __init__(self, name, targets, equirect, lms, q_off, q_lm, margin, expect, small):
        self.name, self.targets, self.equirect, self.lms = name, targets, equirect, lms
        self.q_off, self.q_lm, self.margin, self.expect, self.small = q_off, q_lm, margin, expect, small


def run_case(case):
    """The reference on every target of a case -> (num_fused, best, passed, reproj_xy, x_right, pred_level) over all queries and the
    summed Counter."""
    Q = int(case.q_off[-1])
    best = np.full(Q, -1, np.int32); ok = np.zeros(Q, bool); uv = np.zeros((Q, 2), F32); xr = np.zeros(Q, F32); lv = np.zeros(Q, np.int32)
    st = Counter()
    for k, t in enumerate(case.targets):
        s = slice(case.q_off[k], case.q_off[k + 1])
        _, best[s], ok[s], uv[s], xr[s], lv[s], stats = replace_duplication(t, case.lms, case.q_lm[s], case.margin)
        for c in stats:
            st.update(c)
        st["target_without_keypoints"] += int(t.n == 0)
        st["target_without_queries"] += int(s.stop == s.start)
        st["target_stereo" if t.frame.x_right is not None else ("target_equirectangular" if case.equirect[k] else "target_mono")] += 1
    return int((best >= 0).sum()), best, ok, uv, xr, lv, st


def _flip(desc, k, rng):
    return WR.flip_bits(desc, k, rng)


def _solve_product(ref_x, ref_y, w, want, theta, q_xr=None, split=0.5):
    """Float32 keypoint coordinates (kx, ky[, kxr]) near the distance sqrt(want / w) from ref at angle theta whose gate product
    ((ex^2 + ey^2)[ + er^2]) * w equals `want` exactly, or None."""
    ref_x, ref_y, w, want = F32(ref_x), F32(ref_y), F32(w), F32(want)
    d = float(np.sqrt(float(want) / float(w)))
    dxy = d if q_xr is None else d * np.sqrt(split)
    kx0 = ref_x - dxy * np.cos(theta); ky0 = ref_y - dxy * np.sin(theta)
    kxs = _f32_steps(kx0, 160)
    if q_xr is None:
        kys = _f32_steps(ky0, 160)
        ex = (ref_x - kxs)[:, None]; ey = (ref_y - kys)[None, :]
        p = (ex * ex + ey * ey) * w
        hit = np.argwhere(p == want)
        return None if len(hit) == 0 else (kxs[hit[0][0]], kys[hit[0][1]])
    ky = F32(ky0)
    ey = ref_y - ky
    kxr0 = F32(q_xr) - d * np.sqrt(1.0 - split)
    kxrs = _f32_steps(kxr0, 160)
    ex = (ref_x - kxs)[:, None]; er = (F32(q_xr) - kxrs)[None, :]
    p = ((ex * ex + ey * ey) + er * er) * w
    hit = np.argwhere(p == want)
    return None if len(hit) == 0 else (kxs[hit[0][0]], ky, kxrs[hit[0][1]])


def _lattice(k, per_row, step, x0, y0):
    return F32(x0 + step * (k % per_row) + 0.375), F32(y0 + step * (k // per_row) + 0.625)


# ----------------------------------------------------------------------------------------------- the named cases
def chi2_edges(seed=51):
    """Keypoints whose gate product is exactly 5.99f and one float above it (monocular), exactly 7.8f and one float above it with
    the x_right term, on targets with different scale tables, at octaves level - 1 and level.  The edge keypoint is the nearest
    descriptor; a fallback keypoint well inside the gate wins when the edge one is rejected."""
    S = _Scene(seed)
    rng = S.rng
    specs = [dict(stereo=False, scale_factor=1.2), dict(stereo=True, scale_factor=1.5, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19, cy=185.21),
             dict(stereo=False, scale_factor=2.0, num_levels=4), dict(stereo=True, scale_factor=1.2, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19,
                                                                       cy=185.21)]
    for spec in specs:
        t = S.target(**spec)
        W = t.grid.bounds[1]
        L = len(t.sf)
        for k in range(24):
            rx, ry = _lattice(k, 8, 140.0, 150.0, 60.0) if W > 1000 else _lattice(k, 6, 90.0, 100.0, 60.0)
            stereo_edge = t.stereo and k % 4 >= 2
            want = (CHI_SQ_3D if stereo_edge else CHI_SQ_2D)
            if k % 2:
                want = np.nextafter(want, F32(np.inf))
            # (level, octave) pairs from the planned one on: not every product is reachable from float32 e^2 with every weight
            sol = None
            for j in range(2 * (L - 1)):
                level = 1 + (k + j) % (L - 1)
                o = level - ((k + j) // (L - 1)) % 2
                ref, qxr = S.reprojection(t, rx, ry)
                for tries in range(20):
                    sol = _solve_product(ref[0], ref[1], t.inv[o], want, rng.uniform(0, 2 * np.pi), qxr if stereo_edge else None)
                    if sol is not None:
                        break
                if sol is not None:
                    break
            assert sol is not None, (k, want)
            row, ref, qxr, lv = S.query(t, rx, ry, level)
            base = S.desc[row]
            t.kp(sol[0], sol[1], o, _flip(base, 5, rng), sol[2] if stereo_edge else -1.0)
            t.kp(ref[0] + F32(0.25) * t.sf[level], ref[1] - F32(0.25) * t.sf[level], level, _flip(base, 30, rng), qxr if t.stereo else -1.0)
        for k in range(60):       # clutter
            t.kp(rng.uniform(0, W), rng.uniform(0, t.grid.bounds[3]), rng.integers(0, L), rng.integers(0, 256, 32, dtype=np.uint8),
                 rng.uniform(0, W) if rng.random() < 0.5 else -1.0)
    return S.case("chi2_edges", 3.0, {"chi2_mono_equal": 12, "chi2_mono_above": 12, "chi2_stereo_equal": 6, "chi2_stereo_above": 6,
                                      "fused": 80})


def x_right(seed=52):
    """A monocular target first, then stereo ones: around each stereo query a keypoint within the monocular bound but far outside
    the stereo one (x_right -1, -0.0, 0.0 or the smallest positive float) holds the nearest descriptor, so only x_right >= 0
    decides; a fallback keypoint consistent in x_right wins otherwise.  The monocular target holds the same layout."""
    S = _Scene(seed)
    rng = S.rng
    vals = [F32(-1.0), F32(-0.0), F32(0.0), np.nextafter(F32(0), F32(1))]
    for stereo in (False, True, True):
        t = S.target(stereo=stereo, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19, cy=185.21)
        for k in range(24):
            rx, ry = _lattice(k, 8, 140.0, 120.0, 50.0)
            row, ref, qxr, lv = S.query(t, rx, ry, 2)
            base = S.desc[row]
            t.kp(ref[0] + F32(1.0), ref[1] - F32(0.5), 2, _flip(base, 4, rng), vals[k % 4])
            t.kp(ref[0] - F32(0.5), ref[1] + F32(0.5), 1, _flip(base, 20, rng), qxr - F32(0.5) if stereo else -1.0)
    return S.case("x_right", 3.0, {"xr_negative_zero": 12, "xr_positive_zero": 12, "xr_min_positive": 12, "xr_minus_one": 12,
                                   "xr_decides": 36, "target_mono": 1, "target_stereo": 2})


def levels(seed=53):
    """Keypoints on octaves level - 2 .. level + 1 around each query, the nearest descriptors on the octaves outside [level - 1,
    level], the next on level - 1: predicted level 0 (octave 0 in, 1 out), every level to the top, on targets with 1, 4, 8 and 16
    levels and scale factors 1.2, 1.5 and 2.0."""
    S = _Scene(seed)
    rng = S.rng
    for L, sfac in ((8, 1.2), (1, 1.2), (16, 1.5), (4, 2.0), (8, 1.5)):
        t = S.target(num_levels=L, scale_factor=sfac)
        for k in range(2 * L + 2):
            level = k % L
            rx, ry = _lattice(k, 8, 75.0, 40.0, 40.0)
            row, ref, qxr, lv = S.query(t, rx, ry, level)
            base = S.desc[row]
            for o, dd, off in ((level - 2, 3, (0.4, 0.1)), (level + 1, 4, (-0.4, 0.2)), (level - 1, 8, (0.2, -0.4)), (level, 12, (-0.1, -0.3))):
                if 0 <= o < L:
                    s = t.sf[o]
                    t.kp(ref[0] + F32(off[0]) * s, ref[1] + F32(off[1]) * s, o, _flip(base, dd, rng))
    return S.case("levels", 3.0, {"pred_level_zero": 10, "pred_level_top": 10, "level_in_low": 20, "level_in_high": 30, "level_out_low": 20,
                                  "level_out_high": 20, "pred_level_15": 1})


def box_and_cells(seed=54):
    """Keypoints at exactly |dx| == margin or |dy| == margin (outside, the nearest descriptor) and one float inside; windows
    clipped at each grid border; grids with a negative origin (the radial-division bounds) and with cols and rows other than
    64 x 48; query positions whose cell-range arguments are exact integers.  Margin 2, so that the box, not the gate, decides, and
    scale factors 1.5 and 2.0, so that ref +- margin is a float."""
    S = _Scene(seed)
    rng = S.rng
    margin = F32(2.0)
    for bounds, cols, rows, sfac in (((-35.5, 675.5, -20.75, 500.75), 37, 23, 1.5), ((0.0, 640.0, 0.0, 480.0), 64, 48, 2.0),
                                     ((0.0, 640.0, 0.0, 480.0), 7, 5, 1.5)):
        t = S.target(bounds=bounds, cols=cols, rows=rows, scale_factor=sfac)
        g = t.grid
        for k in range(24):
            level = k % 3
            m = F32(margin * t.sf[level])
            rx, ry = _lattice(k, 6, 90.0, 60.0, 60.0)
            row, ref, qxr, lv = S.query(t, rx, ry, level)
            base = S.desc[row]
            # the float on the box edge (|d| == m exactly) and the next one inside
            axis = k % 4
            sgn = F32(1.0) if axis < 2 else F32(-1.0)
            c = ref[axis % 2]
            e = F32(c + sgn * m)
            assert abs(F32(e - c)) == m
            inside = np.nextafter(e, c)
            for v, dd in ((e, 3), (inside, 9)):
                p = [ref[0], ref[1]]; p[axis % 2] = v
                t.kp(p[0], p[1], level, _flip(base, dd, rng))
        # clipped windows at every border and corner
        for bx, by in ((g.bounds[0] + 0.5, 200.0), (g.bounds[1] - 0.5, 200.0), (300.0, g.bounds[2] + 0.5), (300.0, g.bounds[3] - 0.5),
                       (g.bounds[0] + 0.25, g.bounds[2] + 0.25), (g.bounds[1] - 0.25, g.bounds[3] - 0.25)):
            row, ref, qxr, lv = S.query(t, F32(bx), F32(by), 1)
            t.kp(ref[0] + (F32(0.5) if ref[0] < 300 else F32(-0.5)), ref[1], 1, _flip(S.desc[row], 7, rng))
        # cell-range arguments that are exact integers: ((ref - min_x) - m) * inv_w == cx
        for k in range(12):
            level = 1
            m = F32(margin * t.sf[level])
            cxi = int(rng.integers(2, cols - 2)); cyi = int(rng.integers(1, rows - 1))
            rx = F32(g.min_x + m + F32(cxi) / g.inv_w)
            for _ in range(64):
                v = ((rx - g.min_x) - m) * g.inv_w
                if v == cxi:
                    break
                rx = np.nextafter(rx, F32(np.inf) if v < cxi else F32(-np.inf))
            ry = F32(g.min_y - m + F32(cyi) / g.inv_h)
            for _ in range(64):
                v = ((ry - g.min_y) + m) * g.inv_h
                if v == cyi:
                    break
                ry = np.nextafter(ry, F32(np.inf) if v < cyi else F32(-np.inf))
            if not (g.bounds[0] < rx < g.bounds[1] and g.bounds[2] < ry < g.bounds[3]):
                continue
            row, ref, qxr, lv = S.query(t, rx, ry, level)
            t.kp(ref[0] - F32(0.5), ref[1] + F32(0.25), level, _flip(S.desc[row], 11, rng))
        # keypoints in no cell: beyond the bounds and not finite
        for px, py in ((g.bounds[0] - 1.0, 100.0), (g.bounds[1] + 1.0, 100.0), (np.nan, 100.0), (100.0, np.inf)):
            t.kp(px, py, 0, rng.integers(0, 256, 32, dtype=np.uint8))
    return S.case("box_and_cells", float(margin), {"box_edge_exact": 60, "box_edge_inside": 60, "window_clipped": 18, "cell_edge_exact": 12,
                                                  "fused": 60})


def hamming_and_ties(seed=55):
    """Single candidates at distances 50 (accepted) and 51 (rejected); ties within one cell (the lower index is visited first);
    ties across a cell boundary where the keypoint visited first has the larger index."""
    S = _Scene(seed)
    rng = S.rng
    t = S.target()
    for k in range(48):
        rx, ry = _lattice(k, 8, 70.0, 50.0, 50.0)
        kind = k % 4
        if kind == 3:     # the query 0.25 px right of a cell boundary (cell width 10 px)
            rx = F32(np.floor(rx / 10.0) * 10.0 + 0.25)
        row, ref, qxr, lv = S.query(t, rx, ry, 1)
        base = S.desc[row]
        if kind in (0, 1):
            t.kp(ref[0] + F32(0.5), ref[1], 1, _flip(base, 50 + kind, rng))
        elif kind == 2:   # same cell, same distance: index order is visiting order
            for j in range(3):
                t.kp(ref[0] + F32(0.125 * j), ref[1] + F32(0.25), 0, _flip(base, 17, rng))
        else:             # across cells: the one in the right cell gets the smaller index, the left one is visited first
            t.kp(ref[0] + F32(1.0), ref[1], 1, _flip(base, 21, rng))
            t.kp(ref[0] - F32(1.0), ref[1], 1, _flip(base, 21, rng))
            t.kp(ref[0] + F32(0.5), ref[1] + F32(0.5), 1, _flip(base, 22, rng))
    return S.case("hamming_and_ties", 3.0, {"hamming_50_accepted": 12, "hamming_51_rejected": 12, "tie_within_cell": 12,
                                            "tie_across_cells_winner_higher_index": 12})


def rank_limit(seed=56):
    """One target with 65535 keypoints: the queries' own keypoints around them (a tie each, the first visited winning), the rest
    filling the grid, so that the winners' ranks reach past 32768 and past 65280."""
    S = _Scene(seed)
    rng = S.rng
    t = S.target()
    n_total = 65535
    for k in range(40):
        if k < 20:
            rx, ry = F32(335.0 + 2.0 * (k % 4)), F32(40.0 + 21.0 * (k // 4))
        else:
            rx, ry = F32(632.5 + 1.5 * (k % 4)), F32(380.0 + 18.0 * ((k - 20) // 4))
        row, ref, qxr, lv = S.query(t, rx, ry, 1)
        base = S.desc[row]
        t.kp(ref[0] + F32(0.75), ref[1] + F32(0.5), 1, _flip(base, 13, rng))
        t.kp(ref[0] - F32(0.75), ref[1] - F32(0.5), 0, _flip(base, 13, rng))
    n = n_total - len(t.x)
    fx = rng.uniform(0, 640, n).astype(F32); fy = rng.uniform(0, 480, n).astype(F32)
    fo = rng.integers(0, 8, n); fd = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    t.x += list(fx); t.y += list(fy); t.oct += list(fo); t.desc += list(fd); t.xr += [F32(-1)] * n
    return S.case("rank_limit", 3.0, {"rank_ge_32768": 30, "rank_ge_65280": 4, "tie": 30}, small=False)


def _populate(S, t, nq, nkp, rng, shared=(), nan_rows=0, skip=0):
    """Random queries into t with keypoints near most of them (jittered within the gate, a few bits flipped), clutter, landmarks
    shared with other targets, landmarks with a NaN position and skipped queries (q_lm = -1)."""
    b = t.grid.bounds
    L = len(t.sf)
    for k in range(nq):
        level = int(rng.integers(0, L))
        rx = F32(rng.uniform(b[0] + 5, b[1] - 5)); ry = F32(rng.uniform(b[2] + 5, b[3] - 5))
        row, ref, qxr, lv = S.query(t, rx, ry, level, z=float(rng.uniform(2.0, 12.0)), exact=False)
        if nkp and rng.random() < 0.8:
            o = int(np.clip(lv - rng.integers(0, 2), 0, L - 1))
            s = float(t.sf[o])
            kxr = (qxr + rng.normal(0, 0.8)) if (t.stereo and rng.random() < 0.7) else -1.0
            t.kp(ref[0] + rng.normal(0, 1.0) * s, ref[1] + rng.normal(0, 1.0) * s, o, _flip(S.desc[row], int(rng.integers(0, 70)), rng), kxr)
    for r in shared:
        S.query(t, 0, 0, 0, row=r)
    for _ in range(nan_rows):
        p = [np.nan, 1.0, 5.0] if rng.random() < 0.5 else [1.0, -np.inf, 5.0]
        t.queries.append(S.landmark(p, 1, 1.2, nrm=[0.0, 0.0, 1.0]))
    t.queries += [-1] * skip
    for _ in range(max(nkp - len(t.x), 0)):
        t.kp(rng.uniform(b[0], b[1]), rng.uniform(b[2], b[3]), rng.integers(0, L), rng.integers(0, 256, 32, dtype=np.uint8),
             rng.uniform(b[0], b[1]) if (t.stereo and rng.random() < 0.6) else -1.0)


def mixed_batch(seed=57):
    """One call over mono, stereo and equirectangular targets interleaved, each with its own scale table, level count and grid;
    targets without keypoints and without queries; skipped queries, one landmark queried into several targets, NaN positions."""
    S = _Scene(seed)
    rng = S.rng
    specs = [dict(), dict(stereo=True, scale_factor=1.5, num_levels=6, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19, cy=185.21, cols=80, rows=24),
             dict(model="equirectangular", scale_factor=2.0, num_levels=4), dict(num_levels=1, bounds=(-35.5, 675.5, -20.75, 500.75), cols=37, rows=23),
             dict(stereo=True, num_levels=12, scale_factor=1.2, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19, cy=185.21),
             dict(model="equirectangular", scale_factor=1.2, num_levels=8, cols=96, rows=32), dict(scale_factor=2.0, num_levels=3, cols=16, rows=12),
             dict(stereo=True, scale_factor=1.2, bounds=(0.0, 1241.0, 0.0, 376.0), cx=607.19, cy=185.21)]
    plan = [(120, 500), (150, 700), (0, 600), (100, 0), (140, 600), (130, 900), (90, 300), (110, 500)]   # (queries, keypoints)
    first_rows = []
    for k, (spec, (nq, nkp)) in enumerate(zip(specs, plan)):
        t = S.target(**spec)
        shared = first_rows[:30] if k in (4, 6, 7) else ()
        before = len(S.pos)
        _populate(S, t, nq, nkp, rng, shared=shared, nan_rows=3 if nq else 0, skip=5 if nq else 0)
        if k == 0:
            first_rows = list(range(before, before + nq))
        if nq == 0:
            t.queries.clear()
    return S.case("mixed_batch", 3.0, {"target_without_keypoints": 1, "target_without_queries": 1, "query_skipped": 30, "position_not_finite": 18,
                                       "target_mono": 3, "target_stereo": 3, "target_equirectangular": 2, "fused": 300}, small=False)


def mapping_shape(seed=58):
    """120 targets of benchmark-sized keyframes: 4000-keypoint equirectangular and 2000-keypoint perspective ones, alternating,
    with several hundred queries each."""
    S = _Scene(seed)
    rng = S.rng
    for k in range(120):
        t = S.target(model="equirectangular") if k % 2 == 0 else S.target()
        _populate(S, t, 300, 4000 if k % 2 == 0 else 2000, rng, skip=2)
    return S.case("mapping_shape", 3.0, {"fused": 15000, "target_equirectangular": 60, "target_mono": 60}, small=False)


CASES = {c.__name__: c for c in (chi2_edges, x_right, levels, box_and_cells, hamming_and_ties, rank_limit, mixed_batch, mapping_shape)}


@functools.lru_cache(maxsize=None)
def case_and_reference(name):
    """The named case and run_case's result on it, built once per process."""
    c = CASES[name]()
    return c, run_case(c)
