"""Plain numpy / math reference of the two-view triangulator of local mapping (module::two_view_triangulator::triangulate with
solve::triangulator::triangulate and keyframe::triangulate_stereo) and of create_new_landmarks' compute step.  It restates
what the reference does; it imports neither the oracle nor the library, so a slip that both of those share (a `<` for a
`<=`, the wrong octave's sigma^2, a float cast moved) shows up against it.

One pair, triangulate_pair(), with the reason and branch codes of the library (REASONS, BRANCHES):

- branch selection in scalar float64 in the device's operation order (the library is built with --fmad=false, so that
  order fixes its bits): rays r = R^T b summed in index order, cos_rays = (r1 . r2) / (|r1| |r2|); the stereo parallax
  cs = (d^2 - h^2) / (d^2 + h^2), h = true_baseline / 2, 2.0 for a monocular keypoint.  The recalled reference writes
  cos(2 atan2(h, d)), which is the same number within an ulp of 1 (test_stereo_parallax_forms_differ_by_a_few_ulp measures it);
  the closed form is what both the device and the oracle evaluate.  A keypoint is stereo when 0.0f <= x_right, so -0.0f is
  stereo.  cs1 < cs2 and cs2 < cs1 are strict: a tie takes no stereo branch;
- the two-camera point: the last right-singular vector of the 4 x 4 A from np.linalg.svd (the reference's JacobiSVD
  formulation), not a restatement of the device's Jacobi on A^T A.  With it comes `bound`, a bound on the device's error
  (point_bound());
- the stereo back-projection bit for bit: the two (float) casts of the unprojected x and y, then R^T p_c + centre, and the
  zero vector when depth <= 0;
- the gates in the device's order: cheirality (float)z > 0 of camera 1, then camera 2 (skipped for equirectangular);
  reprojection of view 1, then view 2: 5.99146f sigma^2 (mono) or 7.81473f sigma^2 (stereo, with the float term
  (float)(u - fb / z) - x_right) formed in float and compared with `<` against the double squared error; scale:
  ratio_factor = 1.5f * keyframe 1's scale_factor and ratio_octave = sf_1 / sf_2 in float, the distances and their ratio in
  double.

On the two-camera branch the gates see the SVD point, not the device's: each gate's decision is re-taken at the corners of
the cube of half-width `bound` around the point, and a decision that any corner would take differently (or whose margin is
within twice what the corners move it) is a skip.  Skips are listed with their gate (Result.skip) and the tests require none on the
constructed knife-edge cases."""
import collections
import math

import numpy as np

import candidate_lists_reference as CL
import window_match_reference as WM

F32 = np.float32
EPS = np.finfo(np.float64).eps
CHI_SQ_2D, CHI_SQ_3D = F32(5.99146), F32(7.81473)
EQUIRECTANGULAR = 1

REASONS = {0: "landmark", 1: "no branch", 2: "non-finite", 3: "cheirality 1", 4: "cheirality 2", 5: "reprojection 1",
           6: "reprojection 2", 7: "scale"}
BRANCHES = {-1: "none", 0: "two cameras", 1: "stereo 1", 2: "stereo 2"}
OK, NO_BRANCH, NON_FINITE, CHEIRALITY_1, CHEIRALITY_2, REPROJ_1, REPROJ_2, SCALE = range(8)
TWO_CAMERAS, STEREO_1, STEREO_2, NONE = 0, 1, 2, -1

# point_bound(): the Jacobi on A^T A gives the eigenvector within about eps s1^2 / (s3^2 - s4^2) (rounding of A^T A is
# ~eps s1^2, the gap to the next eigenvalue is s3^2 - s4^2); this factor covers the summation and the sweeps
BOUND_FACTOR = 64.0


def cos_threshold(rays_parallax_deg_thr):
    """cos(rays_parallax_deg_thr * pi / 180), as the host forms it once per call"""
    return math.cos(rays_parallax_deg_thr / 180.0 * math.pi)


def is_stereo(kf, i):
    return kf.stereo_x_right is not None and bool(F32(0.0) <= F32(kf.stereo_x_right[i]))


def _pose(kf):
    return [float(v) for v in kf.pose_cw]


def _centre(P):
    """-(R^T t), each component summed in index order"""
    return [-((P[i] * P[9] + P[3 + i] * P[10]) + P[6 + i] * P[11]) for i in range(3)]


def _ray(P, b):
    return [(P[i] * b[0] + P[3 + i] * b[1]) + P[6 + i] * b[2] for i in range(3)]


def stereo_cos(kf, i):
    """cos of the stereo parallax of keypoint i, closed form; 2.0 for a monocular keypoint"""
    if not is_stereo(kf, i):
        return 2.0
    h = kf.true_baseline / 2.0
    d = float(F32(kf.depths[i]))
    return (d * d - h * h) / (d * d + h * h)


def stereo_cos_atan2(kf, i):
    """the recalled reference's form cos(2 atan2(h, d))"""
    return math.cos(2.0 * math.atan2(kf.true_baseline / 2.0, float(F32(kf.depths[i])))) if is_stereo(kf, i) else 2.0


def cos_rays(kf1, i1, kf2, i2):
    r1 = _ray(_pose(kf1), [float(v) for v in kf1.bearings[i1]])
    r2 = _ray(_pose(kf2), [float(v) for v in kf2.bearings[i2]])
    n1 = math.sqrt((r1[0] * r1[0] + r1[1] * r1[1]) + r1[2] * r1[2])
    n2 = math.sqrt((r2[0] * r2[0] + r2[1] * r2[1]) + r2[2] * r2[2])
    return ((r1[0] * r2[0] + r1[1] * r2[1]) + r1[2] * r2[2]) / (n1 * n2)


def two_camera_matrix(b1, b2, P1, P2):
    """A (4 x 4): rows b_x P_r3 - b_z P_r1 and b_y P_r3 - b_z P_r2 of each view, P = [R | t]"""
    P1 = np.reshape(P1, 12); P2 = np.reshape(P2, 12)
    M1 = np.concatenate([P1[:9].reshape(3, 3), P1[9:, None]], 1); M2 = np.concatenate([P2[:9].reshape(3, 3), P2[9:, None]], 1)
    return np.array([b1[0] * M1[2] - b1[2] * M1[0], b1[1] * M1[2] - b1[2] * M1[1],
                     b2[0] * M2[2] - b2[2] * M2[0], b2[1] * M2[2] - b2[2] * M2[1]])


def point_bound(s, pos):
    """Bound on |device point - SVD point|.  The device's unit eigenvector v of A^T A is off by an angle of about
    eps s1^2 / (s3^2 - s4^2) (A's singular values s, descending); pos = v[:3] / v[3] with |v[3]| = 1 / sqrt(1 + |pos|^2)
    moves by at most that angle times (1 + |pos|^2)."""
    gap = s[2] * s[2] - s[3] * s[3]
    if not gap > 0.0:
        return math.inf
    return BOUND_FACTOR * EPS * (s[0] * s[0] / gap) * (1.0 + float(pos @ pos))


def two_cameras(kf1, i1, kf2, i2):
    """-> (point, bound, singular values); point None where the device's formulation cannot form it (A^T A overflows, or
    v[3] == 0)"""
    A = two_camera_matrix(kf1.bearings[i1], kf2.bearings[i2], kf1.pose_cw, kf2.pose_cw)
    with np.errstate(over="ignore", invalid="ignore"):
        finite = np.all(np.isfinite(A.T @ A))
    if not finite:
        return None, math.inf, None
    _, s, Vt = np.linalg.svd(A)
    v = Vt[3]
    if v[3] == 0.0:
        return None, math.inf, s
    pos = v[:3] / v[3]
    return pos, point_bound(s, pos), s


def stereo_point(kf, i):
    """keyframe::triangulate_stereo(i), perspective, bit for bit"""
    d = F32(kf.depths[i])
    if not F32(0.0) < d:
        return np.zeros(3)
    P = _pose(kf); c = kf.camera
    fx_inv, fy_inv = 1.0 / c.fx, 1.0 / c.fy
    ux = F32(((float(F32(kf.keypts["x"][i])) - c.cx) * float(d)) * fx_inv)
    uy = F32(((float(F32(kf.keypts["y"][i])) - c.cy) * float(d)) * fy_inv)
    pc = [float(ux), float(uy), float(d)]
    ctr = _centre(P)
    return np.array([((P[i_] * pc[0] + P[3 + i_] * pc[1]) + P[6 + i_] * pc[2]) + ctr[i_] for i_ in range(3)])


def camera_z(kf, p):
    P = _pose(kf)
    return ((P[6] * p[0] + P[7] * p[1]) + P[8] * p[2]) + P[11]


def cheirality_ok(kf, p):
    return kf.camera.model == EQUIRECTANGULAR or bool(F32(0.0) < F32(camera_z(kf, p)))


def reproject(kf, p):
    """(u, v), or None behind a perspective camera"""
    P = _pose(kf); c = kf.camera
    pc = [((P[3 * r] * p[0] + P[3 * r + 1] * p[1]) + P[3 * r + 2] * p[2]) + P[9 + r] for r in range(3)]
    if c.model == EQUIRECTANGULAR:
        L = math.sqrt((pc[0] * pc[0] + pc[1] * pc[1]) + pc[2] * pc[2])
        bx, by, bz = pc[0] / L, pc[1] / L, pc[2] / L
        lat, lon = -math.asin(by), math.atan2(bx, bz)
        return c.cols * (0.5 + lon / (2.0 * math.pi)), c.rows * (0.5 - lat / math.pi)
    if pc[2] <= 0.0:
        return None
    z_inv = 1.0 / pc[2]
    return c.fx * pc[0] * z_inv + c.cx, c.fy * pc[1] * z_inv + c.cy


def reprojection_margin(kf, i, p):
    """threshold - squared error (>= 0: the gate passes), -inf behind the camera"""
    uv = reproject(kf, p)
    if uv is None:
        return -math.inf
    ex, ey = uv[0] - float(F32(kf.keypts["x"][i])), uv[1] - float(F32(kf.keypts["y"][i]))
    e2 = ex * ex + ey * ey
    sig = F32(kf.level_sigma_sq[kf.keypts["octave"][i]])
    if is_stereo(kf, i):
        z = camera_z(kf, p)
        with np.errstate(over="ignore", invalid="ignore"):
            xr = F32(uv[0] - kf.camera.focal_x_baseline * (1.0 / z))
            exr = F32(xr - F32(kf.stereo_x_right[i]))
            return float(CHI_SQ_3D * sig) - (e2 + float(F32(exr * exr)))
    return float(CHI_SQ_2D * sig) - e2


def reprojection_ok(kf, i, p):
    m = reprojection_margin(kf, i, p)
    return not (m < 0.0) and m != -math.inf


def ratio_factor(kf1):
    return F32(F32(1.5) * F32(kf1.scale_factor))


def scale_margins(kf1, i1, kf2, i2, p):
    """(ratio_dists * f - ratio_octave, ratio_octave * f - ratio_dists): both >= 0 when the gate passes; None when a
    distance is 0"""
    d = []
    for kf in (kf1, kf2):
        c = _centre(_pose(kf))
        x, y, z = p[0] - c[0], p[1] - c[1], p[2] - c[2]
        d.append(math.sqrt((x * x + y * y) + z * z))
    if d[0] == 0.0 or d[1] == 0.0:
        return None
    ratio_dists = d[1] / d[0]
    f = ratio_factor(kf1)
    ro = F32(F32(kf1.scale_factors[kf1.keypts["octave"][i1]]) / F32(kf2.scale_factors[kf2.keypts["octave"][i2]]))
    return ratio_dists * float(f) - float(ro), float(F32(ro * f)) - ratio_dists


def scale_ok(kf1, i1, kf2, i2, p):
    m = scale_margins(kf1, i1, kf2, i2, p)
    return m is not None and not (m[0] < 0.0 or m[1] < 0.0)


def gates(kf1, i1, kf2, i2, p):
    """-> (reason, [(gate, passed, margin)]) for the gates in order, up to the first that fails"""
    seen = []
    for v, kf in ((0, kf1), (1, kf2)):
        if kf.camera.model != EQUIRECTANGULAR:
            z = camera_z(kf, p)
            ok = cheirality_ok(kf, p)
            seen.append(("cheirality %d" % (v + 1), ok, z))
            if not ok:
                return CHEIRALITY_1 + v, seen
    for v, (kf, i) in enumerate(((kf1, i1), (kf2, i2))):
        m = reprojection_margin(kf, i, p)
        ok = bool(not (m < 0.0) and m != -math.inf)
        seen.append(("reprojection %d %s" % (v + 1, "stereo" if is_stereo(kf, i) else "mono"), ok, m))
        if not ok:
            return REPROJ_1 + v, seen
    m = scale_margins(kf1, i1, kf2, i2, p)
    if m is None:
        seen.append(("scale distance", False, 0.0))
        return SCALE, seen
    seen.append(("scale low", not m[0] < 0.0, m[0]))
    if m[0] < 0.0:
        return SCALE, seen
    seen.append(("scale high", not m[1] < 0.0, m[1]))
    return (SCALE if m[1] < 0.0 else OK), seen


_CORNERS = np.array([[sx, sy, sz] for sx in (-1.0, 1.0) for sy in (-1.0, 1.0) for sz in (-1.0, 1.0)])


class Pair:
    """One pair's outcome: reason, branch, pos (the point of the branch taken, zeros for none), bound (0 for a stereo
    point, which is exact), skip (the first gate whose decision the bound leaves open, or None), seen (gate, passed, margin)
    and, on the two-camera branch, reach (gate -> how far the bound can move its margin)."""

    def __init__(self, reason, branch, pos, bound=0.0, skip=None, seen=(), reach=None, cos_rays=None, cs=None):
        self.reason, self.branch, self.pos, self.bound, self.skip = reason, branch, pos, bound, skip
        self.seen, self.reach, self.cos_rays, self.cs = list(seen), reach or {}, cos_rays, cs


def triangulate_pair(kf1, i1, kf2, i2, cos_thr):
    st1, st2 = is_stereo(kf1, i1), is_stereo(kf2, i2)
    cr = cos_rays(kf1, i1, kf2, i2)
    cs1, cs2 = stereo_cos(kf1, i1), stereo_cos(kf2, i2)
    cs = cs1 if cs1 < cs2 else cs2
    two = ((not st1 and not st2) and 0.0 < cr and cr < cos_thr) or ((st1 or st2) and 0.0 < cr and cr < cs)
    if two:
        pos, bound, s = two_cameras(kf1, i1, kf2, i2)
        if pos is None:
            return Pair(NON_FINITE, TWO_CAMERAS, np.full(3, np.nan), math.inf, cos_rays=cr, cs=(cs1, cs2))
        if not np.all(np.isfinite(pos)):
            return Pair(NON_FINITE, TWO_CAMERAS, pos, bound, cos_rays=cr, cs=(cs1, cs2))
        reason, seen = gates(kf1, i1, kf2, i2, pos)
        # the decisions again at the corners of the cube of half-width bound: where one differs, the bound leaves it open
        reach = collections.defaultdict(float)
        open_gate = None
        if not math.isfinite(bound) or bound >= np.linalg.norm(pos):
            open_gate = seen[0][0] if seen else "point"
        else:
            for c in _CORNERS:
                r2, seen2 = gates(kf1, i1, kf2, i2, pos + bound * c)
                for (g, ok, m), (g2, ok2, m2) in zip(seen, seen2):
                    if g != g2:
                        break
                    reach[g] = max(reach[g], abs(m2 - m)) if math.isfinite(m2 - m) else math.inf
                    if ok != ok2 and open_gate is None:
                        open_gate = g
                if r2 != reason and open_gate is None:
                    open_gate = seen[min(len(seen), len(seen2)) - 1][0]
            for g, ok, m in seen:
                if open_gate is None and abs(m) <= 2.0 * reach[g]:
                    open_gate = g
        return Pair(reason, TWO_CAMERAS, pos, bound, open_gate, seen, dict(reach), cr, (cs1, cs2))
    if st1 and cs1 < cs2:
        branch, pos = STEREO_1, stereo_point(kf1, i1)
    elif st2 and cs2 < cs1:
        branch, pos = STEREO_2, stereo_point(kf2, i2)
    else:
        return Pair(NO_BRANCH, NONE, np.zeros(3), cos_rays=cr, cs=(cs1, cs2))
    reason, seen = gates(kf1, i1, kf2, i2, pos)
    return Pair(reason, branch, pos, 0.0, None, seen, None, cr, (cs1, cs2))


class Result:
    """The reference over one problem's pairs: reason, branch (m,) int; pos (m, 3) (the branch's point, zeros for none);
    bound (m,); skip: list of (pair, gate) the bound leaves open; gates: Counter of (gate, passed) over the decisions taken;
    pairs: the Pair records."""

    def __init__(self, recs):
        self.pairs = recs
        m = len(recs)
        self.reason = np.array([r.reason for r in recs], np.int32).reshape(m)
        self.branch = np.array([r.branch for r in recs], np.int32).reshape(m)
        self.pos = np.array([r.pos for r in recs], np.float64).reshape(m, 3)
        self.bound = np.array([r.bound for r in recs], np.float64).reshape(m)
        self.skip = [(k, r.skip) for k, r in enumerate(recs) if r.skip is not None]
        self.valid = self.reason == OK
        self.gates = gate_counts(recs)


def gate_counts(recs):
    """Counter of (gate, outcome) over pairs: the branch test ("two cameras" against the parallax or the stereo parallax),
    the stereo branches, then every gate reached and whether it passed"""
    n = collections.Counter()
    for r in recs:
        if r.cs is not None:
            mono = r.cs[0] == 2.0 and r.cs[1] == 2.0
            n[("parallax" if mono else "stereo parallax", r.branch == TWO_CAMERAS)] += 1
        n[("branch", BRANCHES[r.branch])] += 1
        for g, ok, _ in r.seen:
            n[(g, ok)] += 1
    return n


def triangulate(kf1, kf2, pairs, rays_parallax_deg_thr=1.0):
    cos_thr = cos_threshold(rays_parallax_deg_thr)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    return Result([triangulate_pair(kf1, int(i1), kf2, int(i2), cos_thr) for i1, i2 in pairs])


# ------------------------------------------------------------------------------------------------ create_new_landmarks


def _stereo_flags(kf):
    if kf.stereo_x_right is None:
        return np.zeros(kf.num_keypts, np.uint8)
    return (F32(0.0) <= kf.stereo_x_right.astype(F32)).astype(np.uint8)


def create_new_landmarks(kf1, neighbours, E_12, epipole_in_2, check_orientation=False, rays_parallax_deg_thr=1.0):
    """mapping_module::create_new_landmarks' compute step: for each neighbour in order, match_for_triangulation (the
    candidate lists of candidate_lists_reference, replayed first-taker, then the orientation check) with keyframe 1's
    landmark flags as they stand, then the triangulation of its pairs in idx_1 order; a keyframe-1 keypoint that gets a
    landmark is no query for the neighbours after it.  -> records (r, 3) int32 (neighbour, idx_1, idx_2), pos_w (r, 3),
    the Pair of each record, and the number of re-queries."""
    B = len(neighbours)
    n1 = kf1.num_keypts
    cos_thr = cos_threshold(rays_parallax_deg_thr)
    q1 = CL.node_order(kf1.bow_node, kf1.has_landmark == 0)
    Q = len(q1)
    ranks = [CL.node_order(n.bow_node, n.has_landmark == 0) for n in neighbours]
    tbase = np.concatenate([[0], np.cumsum([len(r) for r in ranks])]).astype(np.int64)
    recs, pos, pairs, requeries = [], [], [], 0
    if Q == 0 or tbase[-1] == 0:
        return np.zeros((0, 3), np.int32), np.zeros((0, 3)), pairs, 0
    oct1 = kf1.keypts["octave"]
    qdesc, qbear = kf1.descriptors[q1], kf1.bearings[q1]
    qscale, qst = kf1.scale_factors[oct1[q1]].astype(F32), _stereo_flags(kf1)[q1]
    qseg = np.concatenate([CL.node_segments(kf1.bow_node[q1], n.bow_node[r]) for n, r in zip(neighbours, ranks)]).reshape(-1, 2)
    tdesc = np.concatenate([n.descriptors[r] for n, r in zip(neighbours, ranks)]).reshape(-1, 32)
    tbear = np.concatenate([n.bearings[r] for n, r in zip(neighbours, ranks)]).reshape(-1, 3)
    tst = np.concatenate([_stereo_flags(n)[r] for n, r in zip(neighbours, ranks)])
    E = np.reshape(E_12, (B, 9)); ep = np.reshape(epipole_in_2, (B, 3))
    lists = CL.triangulation_topk_batched(qdesc, qbear, qscale, qst, qseg, tdesc, tbear, tst, E, ep, tbase[:-1], Q)
    got = np.zeros(n1, bool)
    for b, n in enumerate(neighbours):
        rk = ranks[b]
        seg = qseg[b * Q:(b + 1) * Q]

        def requery(k, taken):
            return CL.triangulation_topk(qdesc[k:k + 1], qbear[k:k + 1], qscale[k:k + 1], qst[k:k + 1], seg[k:k + 1],
                                         tdesc[tbase[b]:tbase[b + 1]], tbear[tbase[b]:tbase[b + 1]], tst[tbase[b]:tbase[b + 1]],
                                         E[b], ep[b], taken=taken)[0]
        pick, _, nrq = CL.first_taker(lists[b * Q:(b + 1) * Q], requery, len(rk), skip=got[q1])
        requeries += nrq
        match = np.full(n1, -1, np.int64)
        taken_by = [k for k in range(Q) if pick[k] >= 0]
        for k in taken_by:
            match[q1[k]] = rk[pick[k]]
        if check_orientation and taken_by:
            deltas = [F32(F32(kf1.keypts["angle"][q1[k]]) - F32(n.keypts["angle"][rk[pick[k]]])) for k in taken_by]
            for k, bad in zip(taken_by, WM.angle_checker_invalid(deltas)):
                if bad:
                    match[q1[k]] = -1
        for i1 in np.flatnonzero(match >= 0):
            r = triangulate_pair(kf1, int(i1), n, int(match[i1]), cos_thr)
            if r.reason != OK:
                continue
            recs.append((b, int(i1), int(match[i1]))); pos.append(r.pos); pairs.append(r)
            got[i1] = True
    return np.array(recs, np.int32).reshape(-1, 3), np.array(pos, np.float64).reshape(-1, 3), pairs, requeries


def same_points(got, ref_pairs):
    """True when each point of `got` (r, 3) is the reference's: bit for bit on a stereo branch, within the bound on the
    two-camera branch"""
    for p, r in zip(np.asarray(got).reshape(-1, 3), ref_pairs):
        if r.branch == TWO_CAMERAS:
            if not np.linalg.norm(p - r.pos) <= r.bound:
                return False
        elif p.tobytes() != np.asarray(r.pos, np.float64).tobytes():
            return False
    return True
