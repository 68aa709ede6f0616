"""bench.py --dump-outputs: what the value path returned in its last timed step lands as float32 / float64 .npy files within
64 MB; the arrays are those of the frame that step processed (checked against the CPU oracle and against direct calls of the
library on the same inputs); two runs with the same arguments write the same arrays."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

WARMUP, STEPS, STREAMS = 3, 2, 2
LAST = WARMUP + STEPS - 1          # step index of the last timed step (the value leg starts at step 0)


def _run(out_dir, config, steps=STEPS):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--config", str(config), "--steps", str(steps),
                        "--warmup", str(WARMUP), "--streams", str(STREAMS), "--no-cpu-baseline", "--no-latency", "--dump-outputs", str(out_dir)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return {f[:-4]: np.load(os.path.join(out_dir, f)) for f in sorted(os.listdir(out_dir))}


def _workload(config):
    cfg = bench.CONFIGS[config]
    ring = bench.default_ring(cfg)
    return cfg, bench.make_workload(cfg, 0, ring), ring


def _check_common(d, prefix, O, cfg, frame):
    """keypoints / descriptors against the oracle's extract of `frame`; returns the oracle's (kps, desc)."""
    assert all(v.dtype in (np.float32, np.float64) for v in d.values())
    assert sum(v.nbytes for v in d.values()) <= 64 << 20
    kps, desc, _ = O.extract(frame, O.params(cfg["NKP"]))
    got = d[prefix + "keypoints"]
    assert got.shape == (len(kps), 7)
    for c, f in enumerate(("x", "y", "size", "angle", "response", "octave")):
        assert np.array_equal(got[:, c], kps[f].astype(np.float32)), f
    assert np.array_equal(d[prefix + "descriptors"], desc.astype(np.float32))
    return kps, desc


def _check_pose(d, prefix, wl, stereo):
    from openvslam_b200 import optimize
    p = wl["pose"]
    po = optimize.pose_optimizer()
    ninl, pose, flags, _ = po.optimize(optimize.camera(**p["cam"]), not stereo, p["pts_w"], p["obs_xy"], p["obs_xr"] if stereo else None,
                                       p["inv_sigma_sq"], p["poses"][0])
    po.close()
    assert np.array_equal(d[prefix + "pose"], np.asarray(pose, np.float64))
    assert np.array_equal(d[prefix + "pose_outliers"], np.asarray(flags).astype(np.float32))
    assert d[prefix + "pose_num_inliers"][0] == ninl


@pytest.mark.gpu
def test_dump_config4_is_the_last_frame_and_reproducible(tmp_path, oracle):
    O = oracle
    a = _run(tmp_path / "a", 4)
    names = {"keypoints", "descriptors", "bf_matches", "projection_matches", "pose", "pose_outliers", "pose_num_inliers",
             "ba_poses", "ba_points", "ba_outliers"}
    assert set(a) == {"r0_s%d_%s" % (s, n) for s in range(STREAMS) for n in names}
    cfg, wl, ring = _workload(4)
    i, prev = bench.frame_of_step(LAST, 0, ring), bench.frame_of_step(LAST - 1, 0, ring)
    kps, desc = _check_common(a, "r0_s0_", O, cfg, wl["frames"][i])
    _, desc_prev, _ = O.extract(wl["frames"][prev], O.params(cfg["NKP"]))
    assert np.array_equal(a["r0_s0_bf_matches"], O.robust_brute_force_match(desc, desc_prev, None, 0.75).astype(np.float32))
    # projection match against the same landmark construction, made from the oracle's extraction
    s = bench.oracle_landmark_sets(cfg, wl, O, O.params(cfg["NKP"]))[i % wl["nbase"]]
    xy = s["xy"].copy(); xy[:, 0] = (xy[:, 0] + wl["shifts"][i]) % cfg["W"]
    frm = O.MatchFrame(kps["x"], kps["y"], kps["octave"], kps["angle"], None, desc, O.om_grid(0, cfg["W"], 0, cfg["H"]))
    sf = np.array([1.2 ** k for k in range(8)], np.float32)
    _, want = O.projection_match_frame_and_landmarks(frm, sf, xy, None, s["level"], s["desc"], None, None, 5.0)
    assert np.array_equal(a["r0_s0_projection_matches"], want.astype(np.float32))
    _check_pose(a, "r0_s0_", wl, False)
    from openvslam_b200 import optimize
    ba = wl["ba"]
    lba = optimize.local_bundle_adjuster()
    lba.set_cluster_width(2)                  # the bench's width for several streams (the result does not depend on it)
    poses, points, outl, _ = lba.optimize(optimize.camera(**ba["cam"]), True, ba["poses"], ba["fixed"], ba["points"], ba["obs_kf"], ba["obs_lm"],
                                          ba["obs_xy"], None, ba["inv_sigma_sq"])
    lba.close()
    assert np.array_equal(a["r0_s0_ba_poses"], poses) and np.array_equal(a["r0_s0_ba_points"], points)
    assert np.array_equal(a["r0_s0_ba_outliers"], np.asarray(outl).astype(np.float32))
    b = _run(tmp_path / "b", 4)
    assert set(a) == set(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    # one more step: the last step ran on the next frame
    c = _run(tmp_path / "c", 4, STEPS + 1)
    _check_common(c, "r0_s0_", O, cfg, wl["frames"][bench.frame_of_step(LAST + 1, 0, ring)])


@pytest.mark.gpu
def test_dump_config2_projection_branch(tmp_path, oracle):
    O = oracle
    d = _run(tmp_path / "d", 2)
    names = {"keypoints", "descriptors", "projection_matches", "pose", "pose_outliers", "pose_num_inliers"}
    assert set(d) == {"r0_s%d_%s" % (s, n) for s in range(STREAMS) for n in names}
    cfg, wl, ring = _workload(2)
    lmsets = bench.oracle_landmark_sets(cfg, wl, O, O.params(cfg["NKP"]))
    for sid in range(STREAMS):
        i = bench.frame_of_step(LAST, sid, ring)
        kps, desc = _check_common(d, "r0_s%d_" % sid, O, cfg, wl["frames"][i])
        s = lmsets[i % wl["nbase"]]
        xy = s["xy"].copy(); xy[:, 0] = (xy[:, 0] + wl["shifts"][i]) % cfg["W"]
        frm = O.MatchFrame(kps["x"], kps["y"], kps["octave"], kps["angle"], None, desc, O.om_grid(0, cfg["W"], 0, cfg["H"]))
        sf = np.array([1.2 ** k for k in range(8)], np.float32)
        _, want = O.projection_match_current_and_last(frm, sf, 8, np.ones(len(xy), np.uint8), xy, None, s["level"], s["angle"], s["desc"], None, 20.0)
        assert np.array_equal(d["r0_s%d_projection_matches" % sid], want.astype(np.float32))
    _check_pose(d, "r0_s0_", wl, False)


@pytest.mark.gpu
def test_dump_config3_stereo_branch(tmp_path, oracle):
    O = oracle
    d = _run(tmp_path / "e", 3)
    names = {"keypoints", "descriptors", "stereo_x_right", "stereo_depth", "pose", "pose_outliers", "pose_num_inliers"}
    assert set(d) == {"r0_s%d_%s" % (s, n) for s in range(STREAMS) for n in names}
    cfg, wl, ring = _workload(3)
    i = bench.frame_of_step(LAST, 0, ring)
    P = O.params(cfg["NKP"])
    kps, desc = _check_common(d, "r0_s0_", O, cfg, wl["frames"][i])
    kps_r, desc_r, _ = O.extract(wl["frames_right"][i], P)
    cam = wl["pose"]["cam"]
    sf = O.scale_factors(1.2, 8)           # the extractors' own scale factors (float products), which stereo::compute uses
    xr, depth, _ = O.stereo_compute(O.build_pyramid(wl["frames"][i], P), O.build_pyramid(wl["frames_right"][i], P), sf, kps, desc, kps_r, desc_r,
                                    cam["focal_x_baseline"], cam["focal_x_baseline"] / cam["fx"])
    assert np.array_equal(d["r0_s0_stereo_x_right"], xr.astype(np.float32)) and np.array_equal(d["r0_s0_stereo_depth"], depth.astype(np.float32))
    _check_pose(d, "r0_s0_", wl, True)
