"""GPU tests of the tracker's per-landmark geometry (ovs_frame_can_observe_host) and of the two composed projection searches
(ovs_projection_search_local_landmarks_host, ovs_projection_match_current_and_last_reproject_host) against the oracle and against
the matchers they wrap, fed by hand."""
import copy
import ctypes as C

import numpy as np
import pytest

import tracking_problems as TP
from openvslam_b200 import _lib, match

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 31, 32, 33, 127, 128, 129, 20000, 100000]


@pytest.fixture(scope="module")
def OT(oracle):
    from oracle import tracking
    return tracking


def _f32_ulps(a, b):
    a = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7fffffff), a); b = np.where(b < 0, -(b & 0x7fffffff), b)
    return np.abs(a - b)


def _assert_same(got, ref, equirectangular, what=""):
    ok, uv, xr, lv = got
    rok, ruv, rxr, rlv = ref
    assert np.array_equal(ok, rok), what
    assert np.array_equal(lv, rlv), what
    assert xr.tobytes() == rxr.tobytes(), what
    if equirectangular:
        d = _f32_ulps(uv, ruv)
        print("%s: %d of %d equirectangular reprojection coordinates differ from the oracle (max %d ulp)" % (what, int((d > 0).sum()), d.size,
                                                                                                          int(d.max()) if d.size else 0))
        assert d.size == 0 or d.max() <= 1, what
    else:
        assert uv.tobytes() == ruv.tobytes(), what


def _call(pj, s, usable):
    return pj.can_observe(s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5, usable)


def _oracle(OT, s, usable):
    return OT.can_observe(s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5, usable)


@pytest.mark.parametrize("name", TP.SCENES)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("masked", [False, True])
def test_can_observe_matches_the_oracle(OT, name, n, masked):
    s = TP.scene(name, n, seed=1000 + n)
    usable = s["usable"] if masked else None
    pj = match.projection()
    before = _lib.launch_count()
    got = _call(pj, s, usable)
    assert _lib.launch_count() - before == (1 if n else 0)
    _assert_same(got, _oracle(OT, s, usable), name == "equirectangular", "%s n=%d" % (name, n))
    if n >= 20000:
        assert 0.05 < got[0].mean() < 0.95 and len(np.unique(got[3][got[0]])) == TP.NUM_LEVELS
    pj.close()


@pytest.mark.parametrize("equirectangular", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_can_observe_knife_edges(OT, equirectangular, masked):
    s = TP.knife_edges(equirectangular)
    usable = None
    if masked:
        usable = np.ones(len(s["pos_w"]), np.uint8)
        usable[::3] = 0
    pj = match.projection()
    _assert_same(_call(pj, s, usable), _oracle(OT, s, usable), equirectangular, "knife edges")
    pj.close()


# ------------------------------------------------------------------ composed searches
def _clusters(s, heads, size, seed):
    """Copies each of `heads` landmarks onto size - 1 others (position, normal, distances): clusters of landmarks whose keypoints
    lie together.  _frame_for gives their descriptors the shape that exhausts candidate lists.  -> follower -> head map (-1: none)."""
    rng = np.random.default_rng(seed)
    n = len(s["pos_w"])
    pick = rng.choice(n, heads * size, replace=False).reshape(heads, size)
    head_of = np.full(n, -1, np.int64)
    for row in pick:
        for k in ("pos_w", "mean_normal", "min_valid_dist", "max_valid_dist"):
            s[k][row[1:]] = s[k][row[0]]
        head_of[row[1:]] = row[0]
    return head_of


def _frame_for(s, ok, uv, xr, lv, seed, frac_kept=0.85, frac_clutter=0.3, head_of=None):
    """Current-frame keypoints: most observable landmarks seen near their reprojection at their predicted level, with a few
    descriptor bits flipped, plus clutter.  In a cluster of m seen landmarks (head_of), keypoint i has the descriptor D with its own
    10 bits flipped; landmarks 1 .. m - 1 (in index order) carry their keypoint's descriptor and take it, and the last carries D,
    10 bits from every keypoint of the cluster, so that its candidate list is taken by the others (a re-query).  -> keypoint
    arrays, landmark descriptors, kp_has_observed_lm, the truth (landmark of each keypoint, -1 for clutter)."""
    rng = np.random.default_rng(seed)
    n = len(ok)
    lm_desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    seen = np.flatnonzero(ok)
    seen = seen[rng.random(len(seen)) < frac_kept]
    g = s["geometry"]
    nc = int(frac_clutter * len(seen)) + 5
    x = np.concatenate([uv[seen, 0] + rng.normal(0, 1.0, len(seen)), rng.uniform(g.min_x, g.max_x, nc)]).astype(np.float32)
    y = np.concatenate([uv[seen, 1] + rng.normal(0, 1.0, len(seen)), rng.uniform(g.min_y, g.max_y, nc)]).astype(np.float32)
    x = np.clip(x, g.min_x, np.nextafter(np.float32(g.max_x), np.float32(0))); y = np.clip(y, g.min_y, np.nextafter(np.float32(g.max_y), np.float32(0)))
    octave = np.concatenate([lv[seen], rng.integers(0, TP.NUM_LEVELS, nc)]).astype(np.int32)
    angle = rng.uniform(0, 360, len(x)).astype(np.float32)
    desc = np.concatenate([lm_desc[seen], rng.integers(0, 256, (nc, 32), dtype=np.uint8)])
    for i in range(len(seen)):
        for b in rng.choice(256, 6, replace=False):
            desc[i, b // 8] ^= np.uint8(1 << (b % 8))
    x_right = None
    if g.camera.focal_x_baseline > 0:
        x_right = np.concatenate([xr[seen] + rng.normal(0, 0.5, len(seen)), -np.ones(nc)]).astype(np.float32)
        x_right[rng.random(len(x_right)) < 0.2] = -1.0
    truth = np.concatenate([seen, -np.ones(nc, np.int64)])
    kp_has = (rng.random(len(x)) < 0.05).astype(np.uint8)
    if head_of is not None:
        kp_of = {int(l): j for j, l in enumerate(truth) if l >= 0}
        for h in np.unique(head_of[head_of >= 0]):
            members = sorted(int(l) for l in np.append(np.flatnonzero(head_of == h), h) if int(l) in kp_of)
            if len(members) < 5:
                continue
            D = rng.integers(0, 256, 32, dtype=np.uint8)
            bits = rng.permutation(256)
            for i, l in enumerate(members):
                k = kp_of[l]
                desc[k] = D
                for b in bits[10 * i:10 * i + 10]:
                    desc[k, b // 8] ^= np.uint8(1 << (b % 8))
                kp_has[k] = 0
                lm_desc[l] = desc[k] if i < len(members) - 1 else D
    return dict(x=x, y=y, octave=octave, angle=angle, desc=desc, x_right=x_right), lm_desc, kp_has, truth


def _index(mt, kp, g):
    return match.frame_index(mt, kp["x"], kp["y"], kp["octave"], kp["angle"], kp["x_right"], kp["desc"], match.camera_grid(g.min_x, g.max_x, g.min_y, g.max_y))


def _oracle_frame(oracle, kp, g):
    return oracle.MatchFrame(kp["x"], kp["y"], kp["octave"], kp["angle"], kp["x_right"], kp["desc"], oracle.om_grid(g.min_x, g.max_x, g.min_y, g.max_y))


@pytest.mark.parametrize("name", ["mono", "stereo", "fisheye", "equirectangular"])
@pytest.mark.parametrize("margin", [5.0, 10.0, 20.0])
@pytest.mark.parametrize("dup", [False, True])
def test_search_local_landmarks(oracle, OT, name, margin, dup):
    n = 20000 if name in ("equirectangular", "mono") else 6000
    s = TP.scene(name, n, seed=7 + int(margin))
    g = s["geometry"]
    head_of = _clusters(s, 60, 6, seed=int(margin)) if dup else None
    rok, ruv, rxr, rlv = _oracle(OT, s, s["usable"])
    kp, lm_desc, kp_has, truth = _frame_for(s, rok, ruv, rxr, rlv, seed=int(margin) + dup, head_of=head_of)
    pj = match.projection(lowe_ratio=0.8)
    fi = _index(pj, kp, g)
    args = (fi, g, TP.SCALE_FACTORS, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], lm_desc, s["usable"], kp_has, margin)
    r0 = pj.num_requeries()
    l0 = _lib.launch_count()
    nm, matched, ok, uv, xr, lv = pj.search_local_landmarks(*args)
    l1 = _lib.launch_count(); r1 = pj.num_requeries()
    # the same matcher fed by hand with the device's own can_observe outputs
    nm2, matched2 = pj.match_frame_and_landmarks(fi, TP.SCALE_FACTORS, uv, xr, lv, lm_desc, ok.astype(np.uint8), kp_has, margin)
    l2 = _lib.launch_count(); r2 = pj.num_requeries()
    assert nm == nm2 and np.array_equal(matched, matched2)
    assert r1 - r0 == r2 - r1
    assert (l1 - l0) == (l2 - l1) + 1
    if dup:
        assert r1 > r0
    # the oracle's can_observe followed by the oracle matcher
    _assert_same((ok, uv, xr, lv), (rok, ruv, rxr, rlv), name == "equirectangular", name)
    if name != "equirectangular" or uv.tobytes() == ruv.tobytes():
        fo = _oracle_frame(oracle, kp, g)
        onm, omatched = oracle.projection_match_frame_and_landmarks(fo, TP.SCALE_FACTORS, ruv, rxr, rlv, lm_desc, rok.astype(np.uint8), kp_has,
                                                                    margin, 0.8)
        assert nm == onm and np.array_equal(matched, omatched)
    # most matches are the true landmark
    m = matched >= 0
    assert nm > 0.5 * len(np.flatnonzero(truth >= 0))
    if not dup:
        assert (matched[m] == truth[m]).mean() > 0.95
    # a repeat is bit-identical
    again = pj.search_local_landmarks(*args)
    assert again[0] == nm and all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(again[1:], (matched, ok, uv, xr, lv)))
    fi.close(); pj.close()


def _motion_case(case, n, seed):
    """A last frame whose keypoints hold landmarks (some missing, some outliers, some behind the current camera) and a current
    frame moved along its optical axis so that trans_lc = (0, 0, dz)."""
    name = "mono" if case == "mono" else "stereo"
    s = TP.scene(name, n, seed=seed, frac_behind=0.1)
    tb = 0.0 if case == "mono" else 0.537
    dz = {"mono": 0.8, "forward": 0.8, "backward": -0.8, "neither": 0.3}[case]
    last_pose = s["pose_cw"].copy()
    last_pose[11] += dz
    rng = np.random.default_rng(seed)
    usable = (rng.random(n) < 0.85).astype(np.uint8)       # missing landmarks and outliers
    return s, tb, last_pose, usable, rng


@pytest.mark.parametrize("case", ["mono", "forward", "backward", "neither"])
@pytest.mark.parametrize("check_orientation", [False, True])
@pytest.mark.parametrize("n", [0, 1, 129, 1000, 20000])
def test_match_current_and_last_reproject(oracle, OT, case, check_orientation, n):
    s, tb, last_pose, usable, rng = _motion_case(case, n, seed=50 + n)
    g = s["geometry"]
    mono = case == "mono"
    fw, bw = OT.motion_direction(s["pose_cw"], last_pose, mono, tb)
    assert (fw, bw) == {"mono": (False, False), "forward": (True, False), "backward": (False, True), "neither": (False, False)}[case]
    rin, ruv, rxr = OT.reproject(g, s["pos_w"], usable)
    lv = rng.integers(0, TP.NUM_LEVELS, n).astype(np.int32)
    kp, lm_desc, kp_has, truth = _frame_for(s, rin, ruv, rxr, lv, seed=n + 3)
    last_angle = rng.uniform(0, 360, n).astype(np.float32)
    # the current keypoints' angles follow their landmark's last angle plus a common rotation, and their octave its last octave
    seen = truth >= 0
    kp["angle"][seen] = (last_angle[truth[seen]] + 20.0) % 360.0
    kp["octave"][seen] = lv[truth[seen]]
    pj = match.projection(check_orientation=check_orientation)
    fi = _index(pj, kp, g)
    l0 = _lib.launch_count()
    nm, matched, in_image, uv = pj.match_current_and_last_frames_reproject(fi, g, last_pose, TP.SCALE_FACTORS, s["pos_w"], lv, last_angle, lm_desc,
                                                                           usable, kp_has, 20.0, mono, tb)
    l1 = _lib.launch_count()
    assert np.array_equal(in_image, rin)
    if n:
        assert uv.tobytes() == ruv.tobytes()
    # the wrapped matcher fed by hand with the oracle's reprojection and direction
    nm2, matched2 = pj.match_current_and_last_frames(fi, TP.SCALE_FACTORS, TP.NUM_LEVELS, rin.astype(np.uint8), ruv, rxr, lv, last_angle, lm_desc,
                                                     kp_has, 20.0, fw, bw)
    l2 = _lib.launch_count()
    assert nm == nm2 and np.array_equal(matched, matched2)
    assert (l1 - l0) == (l2 - l1) + (1 if n else 0)
    fo = _oracle_frame(oracle, kp, g)
    onm, omatched = oracle.projection_match_current_and_last(fo, TP.SCALE_FACTORS, TP.NUM_LEVELS, rin.astype(np.uint8), ruv, rxr, lv, last_angle,
                                                             lm_desc, kp_has, 20.0, fw, bw, check_orientation)
    assert nm == onm and np.array_equal(matched, omatched)
    if n >= 1000:
        m = matched >= 0
        assert nm > 0 and (matched[m] == truth[m]).mean() > 0.95
    fi.close(); pj.close()


# ------------------------------------------------------------------ launches, errors, sharing
def test_empty_inputs_make_no_launch(OT):
    s = TP.scene("mono", 0, seed=1)
    g = s["geometry"]
    pj = match.projection()
    kp = dict(x=np.zeros(0, np.float32), y=np.zeros(0, np.float32), octave=np.zeros(0, np.int32), angle=np.zeros(0, np.float32),
              desc=np.zeros((0, 32), np.uint8), x_right=None)
    fi = _index(pj, kp, g)
    before = _lib.launch_count()
    assert len(_call(pj, s, None)[0]) == 0
    nm, matched, *_ = pj.search_local_landmarks(fi, g, TP.SCALE_FACTORS, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"],
                                                np.zeros((0, 32), np.uint8))
    assert nm == 0
    nm, matched, _, _ = pj.match_current_and_last_frames_reproject(fi, g, s["pose_cw"], TP.SCALE_FACTORS, np.zeros((0, 3)), np.zeros(0, np.int32),
                                                                   np.zeros(0, np.float32), np.zeros((0, 32), np.uint8))
    assert nm == 0
    assert _lib.launch_count() == before
    fi.close(); pj.close()


def _raw_can_observe(pj, g, n, pos, nrm, lo, hi, outs=True):
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    ok = np.zeros(max(n, 1), np.uint8); uv = np.zeros((max(n, 1), 2), np.float32); xr = np.zeros(max(n, 1), np.float32); lv = np.zeros(max(n, 1), np.int32)
    return _lib.lib().ovs_frame_can_observe_host(pj._h, C.byref(g) if g is not None else None, n, None, vp(pos), vp(nrm), vp(lo), vp(hi),
                                                 C.c_float(0.5), vp(ok) if outs else None, vp(uv), vp(xr), vp(lv))


def test_invalid_arguments_are_rejected_before_any_launch():
    s = TP.scene("mono", 50, seed=2)
    g = s["geometry"]
    pos = np.ascontiguousarray(s["pos_w"]); nrm = np.ascontiguousarray(s["mean_normal"]); lo = s["min_valid_dist"]; hi = s["max_valid_dist"]
    pj = match.projection()
    rok, ruv, rxr, rlv = _call(pj, s, None)
    kp, lm_desc, kp_has, _ = _frame_for(s, rok, ruv, rxr, rlv, seed=1)
    fi = _index(pj, kp, g)
    lv = np.zeros(50, np.int32); ang = np.zeros(50, np.float32)
    bad = []                               # geometries every entry refuses
    for field, value in (("log_scale_factor", 0.0), ("log_scale_factor", -0.2), ("log_scale_factor", float("inf")),
                         ("log_scale_factor", float("nan"))):
        b = copy.copy(g); setattr(b, field, value); bad.append(b)
    for arr in ("rot_cw", "trans_cw", "cam_center"):
        b = copy.copy(g); getattr(b, arr)[0] = float("nan"); bad.append(b)
    b = copy.copy(g); b.trans_cw[2] = float("inf"); bad.append(b)
    b = copy.copy(g); b.camera = copy.copy(g.camera); b.camera.model = 7; bad.append(b)
    before = _lib.launch_count()
    for b in bad:
        assert _raw_can_observe(pj, b, 50, pos, nrm, lo, hi) == -1
        with pytest.raises(_lib.OvsError):
            pj.search_local_landmarks(fi, b, TP.SCALE_FACTORS, pos, nrm, lo, hi, lm_desc)
        with pytest.raises(_lib.OvsError):
            pj.match_current_and_last_frames_reproject(fi, b, s["pose_cw"], TP.SCALE_FACTORS, pos, lv, ang, lm_desc)
    for levels in (0, 17):
        b = copy.copy(g); b.num_scale_levels = levels
        assert _raw_can_observe(pj, b, 50, pos, nrm, lo, hi) == -1
    assert _raw_can_observe(pj, None, 50, pos, nrm, lo, hi) == -1
    assert _raw_can_observe(pj, g, -1, pos, nrm, lo, hi) == -1
    assert _raw_can_observe(pj, g, 50, None, nrm, lo, hi) == -1
    assert _raw_can_observe(pj, g, 50, pos, None, lo, hi) == -1
    assert _raw_can_observe(pj, g, 50, pos, nrm, None, hi) == -1
    assert _raw_can_observe(pj, g, 50, pos, nrm, lo, hi, outs=False) == -1
    # the motion model: a non-finite last pose or baseline, an octave outside the scale table
    for lp, tb in ((np.where(np.arange(12) == 4, np.nan, s["pose_cw"]), 0.5), (s["pose_cw"], float("nan")), (s["pose_cw"], float("inf"))):
        with pytest.raises(_lib.OvsError):
            pj.match_current_and_last_frames_reproject(fi, g, lp, TP.SCALE_FACTORS, pos, lv, ang, lm_desc, is_monocular=False, true_baseline=tb)
    for o in (-1, TP.NUM_LEVELS):
        lvb = lv.copy(); lvb[7] = o
        with pytest.raises(_lib.OvsError):
            pj.match_current_and_last_frames_reproject(fi, g, s["pose_cw"], TP.SCALE_FACTORS, pos, lvb, ang, lm_desc)
    assert _lib.launch_count() == before
    # an unusable keypoint's octave is not read
    u = np.ones(50, np.uint8); u[7] = 0
    lvb = lv.copy(); lvb[7] = 99
    pj.match_current_and_last_frames_reproject(fi, g, s["pose_cw"], TP.SCALE_FACTORS, pos, lvb, ang, lm_desc, last_usable=u)
    fi.close(); pj.close()


def test_existing_matchers_interleaved_on_the_same_handle(OT):
    s = TP.scene("stereo", 8000, seed=99)
    g = s["geometry"]
    rok, ruv, rxr, rlv = _oracle(OT, s, s["usable"])
    kp, lm_desc, kp_has, _ = _frame_for(s, rok, ruv, rxr, rlv, seed=4)
    pj = match.projection(lowe_ratio=0.8)
    fi = _index(pj, kp, g)
    ref = pj.match_frame_and_landmarks(fi, TP.SCALE_FACTORS, ruv, rxr, rlv, lm_desc, rok.astype(np.uint8), kp_has, 5.0)
    lv = np.clip(rlv, 0, TP.NUM_LEVELS - 1)
    ref_last = pj.match_current_and_last_frames(fi, TP.SCALE_FACTORS, TP.NUM_LEVELS, rok.astype(np.uint8), ruv, rxr, lv, np.zeros(len(lv), np.float32),
                                                lm_desc, kp_has, 20.0)
    for _ in range(2):
        pj.search_local_landmarks(fi, g, TP.SCALE_FACTORS, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], lm_desc, s["usable"],
                                  kp_has, 5.0)
        pj.match_current_and_last_frames_reproject(fi, g, s["pose_cw"], TP.SCALE_FACTORS, s["pos_w"], lv, np.zeros(len(lv), np.float32), lm_desc,
                                                   s["usable"], kp_has, 20.0, False, 0.537)
        got = pj.match_frame_and_landmarks(fi, TP.SCALE_FACTORS, ruv, rxr, rlv, lm_desc, rok.astype(np.uint8), kp_has, 5.0)
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1])
        got = pj.match_current_and_last_frames(fi, TP.SCALE_FACTORS, TP.NUM_LEVELS, rok.astype(np.uint8), ruv, rxr, lv, np.zeros(len(lv), np.float32),
                                               lm_desc, kp_has, 20.0)
        assert got[0] == ref_last[0] and np.array_equal(got[1], ref_last[1])
    fi.close(); pj.close()
