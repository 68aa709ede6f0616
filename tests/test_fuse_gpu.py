"""match::fuse::replace_duplication on the device (ovs_fuse_replace_duplication_host) against the oracle (oracle/fuse_oracle.c),
query by query: best_idx and the geometry outputs, on perspective mono, stereo and equirectangular targets, from 0 to more than
100 000 queries over 1 to 120 targets, at the gates' knife edges; batches against single-target calls, repeats, launch counts,
argument checks and the other matchers of the same handle."""
import ctypes as C

import numpy as np
import pytest

from openvslam_b200 import _lib, match
from oracle import fuse as OF
from oracle import oracle as O
import fuse_problems as FP

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fz():
    m = match.fuse()
    yield m
    m.close()


def _oracle_frame(a):
    g = a["geometry"]
    return O.MatchFrame(a["x"], a["y"], a["octave"], np.zeros(len(a["x"]), np.float32), a["x_right"], a["desc"],
                        O.om_grid(g.min_x, g.max_x, g.min_y, g.max_y))


def _oracle(arrays, lms, q_off, q_lm, margin=3.0):
    Q = int(q_off[-1])
    best = np.full(Q, -1, np.int32); ok = np.zeros(Q, bool); uv = np.zeros((Q, 2), np.float32); xr = np.zeros(Q, np.float32)
    lv = np.zeros(Q, np.int32)
    for t, a in enumerate(arrays):
        s = slice(q_off[t], q_off[t + 1])
        _, best[s], ok[s], uv[s], xr[s], lv[s] = OF.replace_duplication(a["geometry"], _oracle_frame(a), FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ,
                                                                      q_lm[s], lms["pos_w"], lms["mean_normal"], lms["min_valid_dist"],
                                                                      lms["max_valid_dist"], lms["lm_desc"], margin)
    return best, ok, uv, xr, lv


def _device(fz, targets, lms, q_off, q_lm, margin=3.0):
    return fz.replace_duplication(targets, lms["pos_w"], lms["mean_normal"], lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"],
                                  q_off, q_lm, margin, geometry=True)


def _check_against_oracle(fz, scene, targets, arrays, lms, q_off, q_lm):
    num, best, ok, uv, xr, lv = _device(fz, targets, lms, q_off, q_lm)
    rbest, rok, ruv, rxr, rlv = _oracle(arrays, lms, q_off, q_lm)
    assert np.array_equal(ok, rok) and np.array_equal(lv, rlv)
    assert num == int((best >= 0).sum())
    if scene != "equirectangular":
        assert uv.tobytes() == ruv.tobytes() and xr.tobytes() == rxr.tobytes()
        assert np.array_equal(best, rbest)
    else:
        # atan2 / asin of the device: at most one float ulp on the reprojection; the search must equal the oracle's fed with the
        # device's own reprojection
        ulps = np.abs(uv.view(np.int32).astype(np.int64) - ruv.view(np.int32).astype(np.int64))
        assert ulps.max(initial=0) <= 1
        for t, a in enumerate(arrays):
            s = slice(q_off[t], q_off[t + 1])
            rows = np.maximum(q_lm[s], 0)
            _, b = O.fuse_best_keypoints(_oracle_frame(a), uv[s], xr[s], lv[s], lms["lm_desc"][rows], FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, 3.0,
                                         usable=ok[s].astype(np.uint8))
            assert np.array_equal(best[s], b), t
    return num, best


SIZES = [  # (B, queries per target, landmarks, keypoints per target, empty targets)
    (1, [0], 50, 500, ()),
    (1, [1], 50, 500, ()),
    (1, [31], 200, 800, ()),
    (2, [16, 16], 200, 800, ()),
    (1, [33], 200, 800, ()),
    (2, [127, 0], 400, 1000, ()),
    (1, [128], 400, 1000, ()),
    (2, [60, 69], 400, 1000, (1,)),
    (20, [1000] * 20, 3000, 1500, (3,)),
    (120, [850] * 119 + [0], 3000, 1200, (7, 50)),
]


@pytest.mark.parametrize("scene", sorted(FP.CAMERAS))
@pytest.mark.parametrize("size", range(len(SIZES)))
@pytest.mark.parametrize("skips", [False, True])
def test_replace_duplication_matches_oracle(fz, scene, size, skips):
    B, qpt, nlm, nkp, empty = SIZES[size]
    if B == 120 and not skips and scene != "mono":
        pytest.skip("the largest batch runs once per camera, with skips")
    targets, arrays, lms, q_off, q_lm = FP.batch(scene, B, nlm, nkp, qpt, seed=100 + size, skip_frac=0.2 if skips else 0.0, empty=empty)
    num, best = _check_against_oracle(fz, scene, targets, arrays, lms, q_off, q_lm)
    if q_off[-1] >= 1000:
        assert num > 0.05 * q_off[-1]


def test_many_queries_in_one_target(fz):
    targets, arrays, lms, q_off, q_lm = FP.batch("mono", 1, 20000, 4000, [20000], seed=8)
    num, _ = _check_against_oracle(fz, "mono", targets, arrays, lms, q_off, q_lm)
    assert num > 1000


@pytest.mark.parametrize("equirectangular", [False, True])
def test_knife_edges(fz, equirectangular):
    s = FP.knife_edges(equirectangular)
    scene = "equirectangular" if equirectangular else "mono"
    lms = dict(pos_w=s["pos_w"], mean_normal=s["mean_normal"], min_valid_dist=s["min_valid_dist"], max_valid_dist=s["max_valid_dist"])
    n = len(s["pos_w"])
    rng = np.random.default_rng(3)
    lms["lm_desc"] = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    g = s["geometry"]
    bounds = (g.min_x, g.max_x, g.min_y, g.max_y)
    # keypoints on the finite reprojections of the oracle, with the landmark's descriptor
    ok, uv, _, lv = OF.fuse_observe(g, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"])
    sel = np.flatnonzero(ok)
    x = uv[sel, 0].astype(np.float32); y = uv[sel, 1].astype(np.float32); octave = lv[sel].astype(np.int32); desc = lms["lm_desc"][sel]
    grid = match.camera_grid(*bounds)
    t = match.fuse_target(g, FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, x, y, octave, desc, grid)
    arrays = [dict(geometry=g, x=x, y=y, octave=octave, desc=desc, x_right=None, grid=grid)]
    q_off = np.array([0, n], np.int32); q_lm = np.arange(n, dtype=np.int32)
    num, best = _check_against_oracle(fz, scene, [t], arrays, lms, q_off, q_lm)
    assert num > 0
    assert (best[~np.isfinite(s["pos_w"]).all(1)] == -1).all()


def test_batch_equals_single_target_calls_and_repeats(fz):
    targets, arrays, lms, q_off, q_lm = FP.batch("stereo", 6, 2000, 1500, [400, 0, 300, 500, 1, 200], seed=12, skip_frac=0.1, empty=(2,))
    out = _device(fz, targets, lms, q_off, q_lm)
    for t in range(len(targets)):
        s = slice(q_off[t], q_off[t + 1])
        one = _device(fz, [targets[t]], lms, np.array([0, q_off[t + 1] - q_off[t]], np.int32), q_lm[s])
        for a, b in zip(out[1:], one[1:]):
            assert np.asarray(a)[s].tobytes() == np.asarray(b).tobytes()
    again = _device(fz, targets, lms, q_off, q_lm)
    assert out[0] == again[0]
    for a, b in zip(out[1:], again[1:]):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("B", [1, 2, 20, 120])
def test_launch_counts(fz, B):
    targets, arrays, lms, q_off, q_lm = FP.batch("mono", B, 500, 300, [40] * B, seed=B)
    before = _lib.launch_count()
    _device(fz, targets, lms, q_off, q_lm)
    assert 1 <= _lib.launch_count() - before <= 2
    before = _lib.launch_count()
    n, best = fz.replace_duplication(targets, lms["pos_w"], lms["mean_normal"], lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"],
                                     q_off, np.full_like(q_lm, -1))
    assert _lib.launch_count() == before and n == 0 and (best == -1).all()
    n, best = fz.replace_duplication(targets, lms["pos_w"], lms["mean_normal"], lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"],
                                     np.zeros(B + 1, np.int32), np.zeros(0, np.int32))
    assert _lib.launch_count() == before and n == 0 and len(best) == 0


def _raw(fz, B, targets, nlm, lms, q_off, q_lm, margin=3.0):
    """the C entry on raw arrays (no Python-side checks)"""
    arr = (match.FuseTarget * max(len(targets), 1))(*[t.c for t in targets])
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    Q = 0 if q_lm is None else len(q_lm)
    best = np.zeros(max(Q, 1), np.int32)
    n = C.c_int(0)
    return _lib.lib().ovs_fuse_replace_duplication_host(fz._h, B, arr if B >= 0 else None, nlm, vp(lms["pos_w"]), vp(lms["mean_normal"]),
                                                        vp(lms["min_valid_dist"]), vp(lms["max_valid_dist"]), vp(lms["lm_desc"]), vp(q_off),
                                                        vp(q_lm), C.c_float(margin), vp(best), C.byref(n), None, None, None, None)


def test_invalid_arguments_are_refused_before_any_launch(fz):
    targets, arrays, lms, q_off, q_lm = FP.batch("mono", 2, 300, 400, [50, 50], seed=5)
    lms = {k: np.ascontiguousarray(v) for k, v in lms.items()}
    INV, UNS = -1, -6
    big = (1 << 26) + 1
    before = _lib.launch_count()
    assert _raw(fz, 2, targets, 300, lms, q_off, q_lm) == 0          # the baseline call is fine (and launches)
    before = _lib.launch_count()
    cases = [
        (INV, dict(B=-1)),
        (INV, dict(margin=0.0)), (INV, dict(margin=-1.0)), (INV, dict(margin=float("nan"))), (INV, dict(margin=float("inf"))),
        (INV, dict(q_off=np.array([1, 50, 100], np.int32))), (INV, dict(q_off=np.array([0, 60, 50], np.int32))),
        (INV, dict(q_lm=np.where(np.arange(100) == 7, 300, q_lm).astype(np.int32))),
        (INV, dict(q_lm=np.where(np.arange(100) == 9, -2, q_lm).astype(np.int32))),
        (INV, dict(lms=dict(lms, pos_w=None))), (INV, dict(lms=dict(lms, lm_desc=None))),
        (INV, dict(q_off=None)), (INV, dict(q_lm=None)),
        (UNS, dict(nlm=big)),
        (UNS, dict(q_off=np.array([0, 0, big], np.int32))),
    ]
    for code, kw in cases:
        args = dict(B=2, targets=targets, nlm=300, lms=lms, q_off=q_off, q_lm=q_lm, margin=3.0)
        args.update(kw)
        assert _raw(fz, **args) == code, kw
    # per-target refusals
    t0, a0 = targets[0], arrays[0]

    def with_target(mutate):
        t = match.fuse_target(a0["geometry"], FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, a0["x"], a0["y"], a0["octave"], a0["desc"], a0["grid"])
        mutate(t)
        return _raw(fz, 2, [t, targets[1]], 300, lms, q_off, q_lm)

    def bad_octave(t):
        t.octave[5] = FP.NUM_LEVELS
    def neg_octave(t):
        t.octave[5] = -1
    def bad_grid(t):
        t.c.grid.num_grid_cols = 0
    def huge_grid(t):
        t.c.grid.num_grid_cols = 2048; t.c.grid.num_grid_rows = 1024
    def bad_model(t):
        t.c.geometry.camera.model = 9
    def nan_pose(t):
        t.c.geometry.rot_cw[4] = float("nan")
    def bad_levels(t):
        t.c.geometry.num_scale_levels = 17
    def no_scale(t):
        t.c.scale_factors = None
    def no_desc(t):
        t.c.descriptors = None
    def too_many(t):
        t.c.num_keypts = 65536
    for code, mutate in [(INV, bad_octave), (INV, neg_octave), (INV, bad_grid), (INV, huge_grid), (INV, bad_model), (INV, nan_pose),
                         (INV, bad_levels), (INV, no_scale), (INV, no_desc), (UNS, too_many)]:
        assert with_target(mutate) == code, mutate.__name__
    assert _lib.launch_count() == before


def test_other_matchers_on_the_same_handle_are_unchanged(fz):
    targets, arrays, lms, q_off, q_lm = FP.batch("stereo", 3, 1500, 1200, [800, 800, 800], seed=21)
    a = arrays[0]
    idx = match.frame_index(fz, a["x"], a["y"], a["octave"], np.zeros(len(a["x"]), np.float32), a["x_right"], a["desc"], a["grid"])
    rows = q_lm[:800]
    _, best, ok, uv, xr, lv = _device(fz, targets[:1], lms, np.array([0, 800], np.int32), rows)

    def others():
        r1 = fz.best_keypoints(idx, uv, xr, lv, lms["lm_desc"][rows], FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, 3.0, usable=ok.astype(np.uint8))
        r2 = idx.window_topk(uv, np.full(800, 10.0, np.float32), lv - 1, lv, lms["lm_desc"][rows], xr)
        return r1, r2
    r1, r2 = others()
    # the composed call gives what the matching core gives on the same reprojections
    assert np.array_equal(r1[1], best)
    _device(fz, targets, lms, q_off, q_lm)
    s1, s2 = others()
    assert r1[0] == s1[0] and np.array_equal(r1[1], s1[1])
    assert all(np.array_equal(x, y) for x, y in zip(r2, s2))
    idx.close()
