"""GPU parity of the grid-windowed matchers (match::projection, match::area) and match::stereo
against the oracle: candidate sets/order of get_keypoints_in_cell, Hamming ranks, the greedy
bookkeeping, the angle histogram, SAD sub-pixel disparities (bit-exact floats)."""
import numpy as np
import pytest

from openvslam_b200 import synth
import window_match_reference as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def frames(oracle):
    from openvslam_b200 import feature
    a = synth.frame(752, 480, seed=70)
    b = synth.shifted(a, 4, 2)
    ext = feature.orb_extractor(feature.orb_params(max_num_keypts=1000))
    ka, da = ext.extract(a)
    kb, db = ext.extract(b)
    ext.close()
    return a, b, ka, da, kb, db


def _frames(oracle, kps, desc, x_right=None, w=752, h=480):
    from openvslam_b200 import match
    mt = match.projection()
    fi = match.frame_index(mt, kps["x"], kps["y"], kps["octave"], kps["angle"], x_right, desc, match.camera_grid(0, w, 0, h))
    fo = oracle.MatchFrame(kps["x"], kps["y"], kps["octave"], kps["angle"], x_right, desc, oracle.om_grid(0, w, 0, h))
    return mt, fi, fo


def test_window_candidates_order_and_ranks(oracle, frames):
    _, _, ka, da, kb, db = frames
    mt, fi, fo = _frames(oracle, kb, db)
    rng = np.random.default_rng(0)
    nq = 300
    sel = rng.choice(len(ka), nq, replace=False)
    ref = np.stack([ka["x"][sel] + 4 + rng.normal(0, 3, nq), ka["y"][sel] + 2 + rng.normal(0, 3, nq)], 1).astype(np.float32)
    ref[:10] = [[-50, -50]] * 5 + [[900, 600]] * 5            # windows off the grid
    margin = rng.choice([3.0, 7.5, 15.0, 40.0], nq).astype(np.float32)
    lo = rng.integers(-1, 4, nq).astype(np.int32); hi = (lo + rng.integers(0, 3, nq)).astype(np.int32)
    hi[:40] = -1                                             # "no upper bound"
    idx, dist = fi.window_topk(ref, margin, lo, hi, da[sel])
    for q in range(nq):
        cand = oracle.get_keypoints_in_cell(fo, ref[q, 0], ref[q, 1], margin[q], lo[q], hi[q])
        d = np.array([oracle.hamming(da[sel[q]], db[c]) for c in cand], np.int64)
        order = np.argsort(d, kind="stable")[:4]             # stable: first visited wins ties
        want_idx = list(cand[order]) + [-1] * (4 - len(order)); want_d = list(d[order]) + [256] * (4 - len(order))
        assert list(idx[q]) == want_idx and list(dist[q]) == want_d, q
    fi.close(); mt.close()


@pytest.mark.parametrize("ratio,margin", [(0.6, 5.0), (0.8, 5.0), (0.9, 15.0)])
def test_match_frame_and_landmarks(oracle, frames, ratio, margin):
    from openvslam_b200 import match
    _, _, ka, da, kb, db = frames
    mt = match.projection(lowe_ratio=ratio)
    fi = match.frame_index(mt, kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, match.camera_grid(0, 752, 0, 480))
    fo = oracle.MatchFrame(kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, oracle.om_grid(0, 752, 0, 480))
    rng = np.random.default_rng(1)
    sf = oracle.scale_factors(1.2, 8)
    # landmarks: frame A's keypoints (x3, so that several landmarks compete for one keypoint)
    rep = np.tile(np.arange(len(ka)), 3)
    reproj = np.stack([ka["x"][rep] + 4 + rng.normal(0, 1.0, len(rep)), ka["y"][rep] + 2 + rng.normal(0, 1.0, len(rep))], 1).astype(np.float32)
    usable = (rng.random(len(rep)) < 0.9).astype(np.uint8)
    has = (rng.random(len(kb)) < 0.1).astype(np.uint8)
    n, m = mt.match_frame_and_landmarks(fi, sf, reproj, None, ka["octave"][rep], da[rep], usable, has, margin)
    on, om = oracle.projection_match_frame_and_landmarks(fo, sf, reproj, None, ka["octave"][rep], da[rep], usable, has, margin, ratio)
    assert n == on and np.array_equal(m, om) and n > 200
    fi.close(); mt.close()


@pytest.mark.parametrize("forward,backward,check", [(False, False, True), (True, False, True), (False, True, False)])
def test_match_current_and_last_frames(oracle, frames, forward, backward, check):
    from openvslam_b200 import match
    _, _, ka, da, kb, db = frames
    mt = match.projection(check_orientation=check)
    rng = np.random.default_rng(2)
    xr = np.where(rng.random(len(kb)) < 0.5, kb["x"] - 10, -1).astype(np.float32)     # stereo frame: half the keypoints have x_right
    fi = match.frame_index(mt, kb["x"], kb["y"], kb["octave"], kb["angle"], xr, db, match.camera_grid(0, 752, 0, 480))
    fo = oracle.MatchFrame(kb["x"], kb["y"], kb["octave"], kb["angle"], xr, db, oracle.om_grid(0, 752, 0, 480))
    sf = oracle.scale_factors(1.2, 8)
    reproj = np.stack([ka["x"] + 4 + rng.normal(0, 2.0, len(ka)), ka["y"] + 2 + rng.normal(0, 2.0, len(ka))], 1).astype(np.float32)
    rxr = (reproj[:, 0] - 10 + rng.normal(0, 3.0, len(ka))).astype(np.float32)
    usable = (rng.random(len(ka)) < 0.85).astype(np.uint8)
    n, m = mt.match_current_and_last_frames(fi, sf, 8, usable, reproj, rxr, ka["octave"], ka["angle"], da, None, 20.0, forward, backward)
    on, om = oracle.projection_match_current_and_last(fo, sf, 8, usable, reproj, rxr, ka["octave"], ka["angle"], da, None, 20.0, forward, backward, check)
    assert n == on and np.array_equal(m, om) and n > 100
    fi.close(); mt.close()


@pytest.mark.parametrize("thr,check", [(50, True), (100, False), (70, True)])
def test_match_frame_and_keyframe_and_sim3(oracle, frames, thr, check):
    """projection::match_frame_and_keyframe / match_by_Sim3_transform (relocalisation / loop closure callers)."""
    from openvslam_b200 import match
    _, _, ka, da, kb, db = frames
    mt = match.projection(check_orientation=check)
    fi = match.frame_index(mt, kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, match.camera_grid(0, 752, 0, 480))
    fo = oracle.MatchFrame(kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, oracle.om_grid(0, 752, 0, 480))
    rng = np.random.default_rng(8)
    sf = oracle.scale_factors(1.2, 8)
    reproj = np.stack([ka["x"] + 4 + rng.normal(0, 2.0, len(ka)), ka["y"] + 2 + rng.normal(0, 2.0, len(ka))], 1).astype(np.float32)
    lvl = np.clip(ka["octave"] + rng.integers(-1, 2, len(ka)), 0, 7).astype(np.int32)
    usable = (rng.random(len(ka)) < 0.8).astype(np.uint8)
    has = (rng.random(len(kb)) < 0.15).astype(np.uint8)
    n, m = mt.match_frame_and_keyframe(fi, sf, reproj, lvl, ka["angle"], da, usable, has, 10.0, thr)
    on, om = oracle.projection_match_best(fo, reproj, None, np.float32(10.0) * sf[lvl], lvl - 1, lvl + 1, ka["angle"], da, usable, has, thr, check)
    assert n == on and np.array_equal(m, om) and n > 50
    n, m = mt.match_by_Sim3_transform(fi, sf, reproj, lvl, da, usable, has, 7.5)
    on, om = oracle.projection_match_best(fo, reproj, None, np.float32(7.5) * sf[lvl], lvl - 1, lvl, np.zeros(len(ka), np.float32), da, usable, has, 50, False)
    assert n == on and np.array_equal(m, om)
    fi.close(); mt.close()


@pytest.mark.parametrize("margin", [7.5, 15.0])
def test_match_keyframes_mutually(oracle, frames, margin):
    """projection::match_keyframes_mutually (loop closure): independent best match per landmark in both directions + cross-check."""
    from openvslam_b200 import match
    _, _, ka, da, kb, db = frames
    mt = match.projection()
    grid = match.camera_grid(0, 752, 0, 480)
    f1 = match.frame_index(mt, ka["x"], ka["y"], ka["octave"], ka["angle"], None, da, grid)
    f2 = match.frame_index(mt, kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, grid)
    o1 = oracle.MatchFrame(ka["x"], ka["y"], ka["octave"], ka["angle"], None, da, oracle.om_grid(0, 752, 0, 480))
    o2 = oracle.MatchFrame(kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, oracle.om_grid(0, 752, 0, 480))
    rng = np.random.default_rng(21)
    sf = oracle.scale_factors(1.2, 8)
    # frame b is frame a shifted by (3, 1): the "Sim3" reprojections are the keypoint positions moved by the shift plus noise
    r12 = np.stack([ka["x"] + 3 + rng.normal(0, 1.5, len(ka)), ka["y"] + 1 + rng.normal(0, 1.5, len(ka))], 1).astype(np.float32)
    r21 = np.stack([kb["x"] - 3 + rng.normal(0, 1.5, len(kb)), kb["y"] - 1 + rng.normal(0, 1.5, len(kb))], 1).astype(np.float32)
    l12 = np.clip(ka["octave"] + rng.integers(0, 2, len(ka)), 0, 7).astype(np.int32)
    l21 = np.clip(kb["octave"] + rng.integers(0, 2, len(kb)), 0, 7).astype(np.int32)
    u1 = (rng.random(len(ka)) < 0.85).astype(np.uint8); u2 = (rng.random(len(kb)) < 0.85).astype(np.uint8)
    n, m = mt.match_keyframes_mutually(f1, f2, sf, u1, r12, l12, da, u2, r21, l21, db, margin)
    on, om = oracle.projection_match_keyframes_mutually(o1, o2, sf, u1, r12, l12, da, u2, r21, l21, db, margin)
    assert n == on and np.array_equal(m, om) and n > 50
    assert (m[u1 == 0] == -1).all()
    f1.close(); f2.close(); mt.close()


@pytest.mark.parametrize("margin,ratio", [(50, 0.9), (100, 0.9), (30, 0.7)])
def test_area_match_in_consistent_area(oracle, frames, margin, ratio):
    from openvslam_b200 import match
    _, _, ka, da, kb, db = frames
    mt = match.area(lowe_ratio=ratio)
    fi = match.frame_index(mt, kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, match.camera_grid(0, 752, 0, 480))
    f1 = oracle.MatchFrame(ka["x"], ka["y"], ka["octave"], ka["angle"], None, da, oracle.om_grid(0, 752, 0, 480))
    f2 = oracle.MatchFrame(kb["x"], kb["y"], kb["octave"], kb["angle"], None, db, oracle.om_grid(0, 752, 0, 480))
    prev = np.stack([ka["x"], ka["y"]], 1).astype(np.float32)
    n, m, p = mt.match_in_consistent_area(fi, ka["octave"], ka["angle"], da, prev, margin)
    on, om, op = oracle.area_match_in_consistent_area(f1, f2, prev, margin, ratio, True)
    assert n == on and np.array_equal(m, om) and np.array_equal(p, op) and n > 50
    fi.close(); mt.close()


def test_greedy_requery_paths(oracle):
    """Many near-identical descriptors inside one window: the top-4 lists get exhausted by claimed
    keypoints and the GPU re-query path must reproduce the sequential reference."""
    from openvslam_b200 import match
    rng = np.random.default_rng(5)
    n = 600
    base = rng.integers(0, 256, (6, 32), dtype=np.uint8)
    desc = base[rng.integers(0, 6, n)].copy()
    desc[:, 0] ^= rng.integers(0, 4, n).astype(np.uint8)      # tiny perturbations: lots of ties
    x = rng.uniform(100, 400, n).astype(np.float32); y = rng.uniform(100, 300, n).astype(np.float32)
    octv = rng.integers(0, 3, n).astype(np.int32); ang = rng.uniform(0, 360, n).astype(np.float32)
    mt = match.projection(lowe_ratio=0.95)
    fi = match.frame_index(mt, x, y, octv, ang, None, desc, match.camera_grid(0, 752, 0, 480))
    fo = oracle.MatchFrame(x, y, octv, ang, None, desc, oracle.om_grid(0, 752, 0, 480))
    sf = oracle.scale_factors(1.2, 8)
    nl = 1500
    lmd = base[rng.integers(0, 6, nl)].copy()
    reproj = np.stack([rng.uniform(100, 400, nl), rng.uniform(100, 300, nl)], 1).astype(np.float32)
    lvl = rng.integers(0, 3, nl).astype(np.int32)
    fr = R.Frame(x, y, octv, ang, None, desc, R.Grid(0, 752, 0, 480))
    before = mt.num_requeries()
    n1, m1 = mt.match_frame_and_landmarks(fi, sf, reproj, None, lvl, lmd, None, None, 40.0)
    o1, om1 = oracle.projection_match_frame_and_landmarks(fo, sf, reproj, None, lvl, lmd, None, None, 40.0, 0.95)
    r1, rm1, _ = R.match_frame_and_landmarks(fr, sf, reproj, None, lvl, lmd, None, None, 40.0, 0.95)
    assert n1 == o1 == r1 and np.array_equal(m1, om1) and np.array_equal(m1, rm1)
    assert mt.num_requeries() > before
    usable = np.ones(nl, np.uint8)
    last_angle = rng.uniform(0, 360, nl).astype(np.float32)
    before = mt.num_requeries()
    n2, m2 = mt.match_current_and_last_frames(fi, sf, 8, usable, reproj, None, lvl, last_angle, lmd, None, 40.0)
    o2, om2 = oracle.projection_match_current_and_last(fo, sf, 8, usable, reproj, None, lvl, last_angle, lmd, None, 40.0, False, False, True)
    r2, rm2, _ = R.match_current_and_last_frames(fr, sf, 8, usable, reproj, None, lvl, last_angle, lmd, None, 40.0)
    assert n2 == o2 == r2 and np.array_equal(m2, om2) and np.array_equal(m2, rm2) and n2 > 0
    assert mt.num_requeries() > before
    fi.close(); mt.close()


def test_angle_checker(oracle):
    rng = np.random.default_rng(3)
    d = np.concatenate([rng.normal(20, 5, 300), rng.uniform(-360, 720, 100)]).astype(np.float32)
    inv = oracle.angle_checker_invalid(d)
    assert inv[:300].mean() < 0.2 and inv[300:].mean() > 0.5


def test_stereo_compute_bit_exact(oracle):
    from openvslam_b200 import feature, match
    left = synth.frame(1241, 376, seed=90)
    rng = np.random.default_rng(4)
    right = np.empty_like(left)
    # piecewise-constant disparity (three depth planes): rows shifted by d in {6, 18, 41}
    for (y0, y1, d) in [(0, 130, 6), (130, 260, 18), (260, 376, 41)]:
        right[y0:y1] = np.roll(left[y0:y1], -d, axis=1)
    right = np.clip(right.astype(np.int16) + rng.integers(-2, 3, right.shape), 0, 255).astype(np.uint8)
    el = feature.orb_extractor(feature.orb_params(max_num_keypts=2000)); er = feature.orb_extractor(feature.orb_params(max_num_keypts=2000))
    kl, dl = el.extract(left); kr, dr = er.extract(right)
    st = match.stereo()
    fxb, bl = 386.1448, 0.5372
    xr, dp, nm = st.compute(el, er, kl, dl, kr, dr, fxb, bl)
    P = oracle.params(2000)
    oxr, odp, onm = oracle.stereo_compute(oracle.build_pyramid(left, P), oracle.build_pyramid(right, P), oracle.scale_factors(1.2, 8), kl, dl, kr, dr, fxb, bl)
    assert nm == onm and np.array_equal(xr.view(np.uint32), oxr.view(np.uint32)) and np.array_equal(dp.view(np.uint32), odp.view(np.uint32))
    ok = xr >= 0
    assert ok.sum() > 300
    disp = kl["x"][ok] - xr[ok]
    truth = np.where(kl["y"][ok] < 130, 6, np.where(kl["y"][ok] < 260, 18, 41))
    assert np.mean(np.abs(disp - truth) < 1.5) > 0.85
    # empty sides
    z = np.zeros(0, kl.dtype)
    xr0, _, n0 = st.compute(el, er, kl, dl, z, np.zeros((0, 32), np.uint8), fxb, bl)
    assert n0 == 0 and (xr0 == -1).all()
    el.close(); er.close(); st.close()


def test_frame_index_from_device_output(oracle):
    """SURVEY 8f rank 1: the frame index built from the extractor's device output (descriptors never visit the host)
    answers every windowed query exactly like the index built from host arrays."""
    import torch
    from openvslam_b200 import feature, match, synth
    img = synth.frame(752, 480, seed=41)
    ext = feature.orb_extractor(feature.orb_params(max_num_keypts=1500))
    kps, desc = ext.extract(img)
    dev = torch.device("cuda", 0)
    d_img = torch.from_numpy(img).to(dev)
    cap = ext._cap
    d_kps = torch.zeros((cap, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((cap, 32), dtype=torch.uint8, device=dev)
    n = ext.extract_device(d_img.data_ptr(), 752, 480, 752, d_kps.data_ptr(), d_desc.data_ptr(), cap)
    assert n == len(kps)
    mt = match.projection()
    grid = match.camera_grid(0, 752, 0, 480)
    fd = match.frame_index.from_device(mt, n, d_kps.data_ptr(), d_desc.data_ptr(), grid)
    fh = match.frame_index(mt, kps["x"], kps["y"], kps["octave"], kps["angle"], None, desc, grid)
    rng = np.random.default_rng(3)
    nq = 1200
    sel = rng.integers(0, n, nq)
    ref = np.stack([kps["x"][sel] + rng.normal(0, 3, nq), kps["y"][sel] + rng.normal(0, 3, nq)], 1).astype(np.float32)
    margin = rng.uniform(5, 25, nq).astype(np.float32)
    lo = np.clip(kps["octave"][sel] - 1, 0, 7).astype(np.int32); hi = (lo + 2).astype(np.int32)
    q = desc[sel].copy(); q[:, 0] ^= rng.integers(0, 256, nq).astype(np.uint8)
    i_d, d_d = fd.window_topk(ref, margin, lo, hi, q)
    i_h, d_h = fh.window_topk(ref, margin, lo, hi, q)
    assert np.array_equal(i_d, i_h) and np.array_equal(d_d, d_h) and (i_h[:, 0] >= 0).mean() > 0.9
    # and a full matcher call on top of it
    sf = oracle.scale_factors(1.2, 8)
    usable = np.ones(nq, np.uint8); has = np.zeros(n, np.uint8)
    lvl = np.clip(kps["octave"][sel], 0, 7).astype(np.int32)
    nd, md = mt.match_frame_and_landmarks(fd, sf, ref, None, lvl, q, usable, has, 5.0)
    nh, mh = mt.match_frame_and_landmarks(fh, sf, ref, None, lvl, q, usable, has, 5.0)
    assert nd == nh and np.array_equal(md, mh) and nd > 100
    fd.close(); fh.close(); mt.close(); ext.close()


@pytest.mark.parametrize("n,nq,stereo,seed", [(2000, 6000, False, 1), (4000, 20000, True, 2)])
def test_fuse_best_keypoints(oracle, n, nq, stereo, seed):
    """match::fuse matching core: window + per-octave chi-square gate on the reprojection error + nearest descriptor
    (first in visiting order on ties) at <= HAMMING_DIST_THR_LOW, for every landmark independently."""
    from openvslam_b200 import match
    rng = np.random.default_rng(seed)
    W, H = 1241, 376
    x = rng.uniform(0, W, n).astype(np.float32); y = rng.uniform(0, H, n).astype(np.float32)
    octv = rng.integers(0, 8, n).astype(np.int32); ang = rng.uniform(0, 360, n).astype(np.float32)
    xr = np.where(rng.random(n) < 0.7, x - rng.uniform(1, 40, n), -1).astype(np.float32) if stereo else None
    base = rng.integers(0, 256, (64, 32), dtype=np.uint8)
    desc = base[rng.integers(0, 64, n)].copy(); desc[:, 7] ^= rng.integers(0, 4, n).astype(np.uint8)
    sf = oracle.scale_factors(1.2, 8); inv_sigma = (1.0 / (sf * sf)).astype(np.float32)
    sel = rng.integers(0, n, nq)
    ref = np.stack([x[sel] + rng.normal(0, 1.5, nq), y[sel] + rng.normal(0, 1.5, nq)], 1).astype(np.float32)
    rxr = (ref[:, 0] - rng.uniform(1, 40, nq)).astype(np.float32) if stereo else None
    if stereo:
        hit = xr[sel] >= 0
        rxr[hit] = (xr[sel][hit] + rng.normal(0, 1.0, hit.sum())).astype(np.float32)
    lvl = np.clip(octv[sel] + rng.integers(0, 2, nq), 0, 7).astype(np.int32)
    q = desc[sel].copy(); q[:, 1] ^= rng.integers(0, 8, nq).astype(np.uint8)
    usable = (rng.random(nq) < 0.9).astype(np.uint8)
    grid = match.camera_grid(0, W, 0, H)
    fz = match.fuse()
    f = match.frame_index(fz, x, y, octv, ang, xr, desc, grid)
    num, best = fz.best_keypoints(f, ref, rxr, lvl, q, sf, inv_sigma, 3.0, usable)
    fo = oracle.MatchFrame(x, y, octv, ang, xr, desc, oracle.om_grid(0, W, 0, H))
    onum, obest = oracle.fuse_best_keypoints(fo, ref, rxr, lvl, q, sf, inv_sigma, 3.0, usable)
    assert num == onum and np.array_equal(best, obest) and num > nq // 4
    f.close(); fz.close()
