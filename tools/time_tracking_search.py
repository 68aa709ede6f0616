"""Times the tracker's two projection searches with the per-landmark geometry on the device against the shape they replace, at
bench.py's shapes:

  config 4  equirectangular 1920 x 960, 4000 keypoints, 20 000 local landmarks: tracking_module::search_local_landmarks
  config 5  perspective 1920 x 1080, 2000 keypoints, 20 000 local landmarks: the same
  config 2  perspective 752 x 480 monocular, 1000 keypoints: the motion model (match_current_and_last_frames)

Three numbers per configuration:
  host_loop_plus_matcher_ms  the oracle's C loop (frame::can_observe, or reproject_to_image and the direction, one landmark after the
                             other in one thread, on arrays marshalled once) followed by the existing GPU matcher call;
  composed_ms                the composed call (ovs_projection_search_local_landmarks_host or
                             ovs_projection_match_current_and_last_reproject_host);
  kernel_us                  the geometry kernel alone (CUDA events around its launch, ovs_frame_can_observe_host; for config 2 the
                             same kernel over the last frame's 1000 landmarks).
The call times are medians over warm calls of the host clock around one call (each ends with a device synchronise).  The GPU's name
and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE` also writes them there.

    python tools/time_tracking_search.py [--calls 50] [--out results.jsonl]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tracking_problems as TP  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def median_ms(fn, calls):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def scene(model, W, H, n, seed):
    """n landmarks spread over the whole view (the local map), about half of them observable"""
    rng = np.random.default_rng(seed)
    from openvslam_b200.match import frame_geometry
    from openvslam_b200.optimize import camera
    if model == "equirectangular":
        cam = camera("equirectangular", cols=float(W), rows=float(H))
    else:
        f = 0.8 * W
        cam = camera("perspective", fx=f, fy=f, cx=W / 2.0, cy=H / 2.0)
    R = TP.rotation(rng); t = rng.normal(size=3)
    g = frame_geometry(cam, (0.0, float(W), 0.0, float(H)), TP.pose12(R, t), TP.NUM_LEVELS, TP.LOG_SCALE_FACTOR)
    center = -(R.T @ t)
    d = rng.normal(size=(n, 3))
    if model != "equirectangular":
        d[:, 2] = np.abs(d[:, 2]) * 1.5
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dist = rng.uniform(1.0, 30.0, n)
    pos = center + (d * dist[:, None]) @ R
    nrm = (pos - center) / dist[:, None] + rng.normal(scale=0.5, size=(n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    hi = (dist * rng.uniform(0.7, 2.0, n)).astype(np.float32)
    lo = (hi / np.float32(TP.SCALE_FACTOR ** 7) * rng.uniform(0.8, 2.0, n)).astype(np.float32)
    return dict(geometry=g, pos_w=pos, mean_normal=nrm, min_valid_dist=lo, max_valid_dist=hi, usable=np.ones(n, np.uint8), pose_cw=TP.pose12(R, t))


def frame(s, ok, uv, lv, nkp, seed):
    """nkp keypoints: observable landmarks near their reprojection with a few bits flipped, the rest clutter"""
    rng = np.random.default_rng(seed)
    g = s["geometry"]
    n = len(ok)
    lm_desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    seen = rng.permutation(np.flatnonzero(ok))[: int(0.7 * nkp)]
    nc = nkp - len(seen)
    x = np.clip(np.concatenate([uv[seen, 0] + rng.normal(0, 1, len(seen)), rng.uniform(g.min_x, g.max_x, nc)]), g.min_x, g.max_x - 1e-3)
    y = np.clip(np.concatenate([uv[seen, 1] + rng.normal(0, 1, len(seen)), rng.uniform(g.min_y, g.max_y, nc)]), g.min_y, g.max_y - 1e-3)
    octave = np.concatenate([lv[seen], rng.integers(0, TP.NUM_LEVELS, nc)]).astype(np.int32)
    desc = np.concatenate([lm_desc[seen], rng.integers(0, 256, (nc, 32), dtype=np.uint8)])
    desc[: len(seen), 0] ^= np.uint8(0x11)
    return dict(x=x.astype(np.float32), y=y.astype(np.float32), octave=octave, angle=rng.uniform(0, 360, nkp).astype(np.float32), desc=desc), lm_desc


def host_can_observe(OT, s):
    """the oracle's C loop on arrays marshalled once, as a C++ caller would run it"""
    lib = OT.lib()
    n = len(s["pos_w"])
    pos = np.ascontiguousarray(s["pos_w"]); nrm = np.ascontiguousarray(s["mean_normal"])
    lo = s["min_valid_dist"]; hi = s["max_valid_dist"]; u = s["usable"]
    ok = np.zeros(n, np.uint8); uv = np.zeros((n, 2), np.float32); xr = np.zeros(n, np.float32); lv = np.zeros(n, np.int32)
    args = [C.byref(s["geometry"]), n] + [a.ctypes.data_as(C.c_void_p) for a in (u, pos, nrm, lo, hi)] + [C.c_float(0.5)] + \
        [a.ctypes.data_as(C.c_void_p) for a in (ok, uv, xr, lv)]
    return lambda: lib.ott_can_observe_all(*args), (ok, uv, xr, lv)


def host_reproject(OT, s):
    lib = OT.lib()
    n = len(s["pos_w"])
    pos = np.ascontiguousarray(s["pos_w"])
    ok = np.zeros(n, np.uint8); uv = np.zeros((n, 2), np.float32); xr = np.zeros(n, np.float32)
    args = [C.byref(s["geometry"]), n, s["usable"].ctypes.data_as(C.c_void_p)] + [a.ctypes.data_as(C.c_void_p) for a in (pos, ok, uv, xr)]
    return lambda: lib.ott_reproject_all(*args), (ok, uv, xr)


def local_map_search(pj, OT, model, W, H, nkp, nlm, calls):
    from openvslam_b200 import match
    s = scene(model, W, H, nlm, seed=nkp)
    g = s["geometry"]
    loop, (ok, uv, xr, lv) = host_can_observe(OT, s)
    loop()
    kp, lm_desc = frame(s, ok.astype(bool), uv, lv, nkp, seed=1)
    fi = match.frame_index(pj, kp["x"], kp["y"], kp["octave"], kp["angle"], None, kp["desc"], match.camera_grid(g.min_x, g.max_x, g.min_y, g.max_y))
    args = (fi, g, TP.SCALE_FACTORS, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], lm_desc, s["usable"], None, 5.0)
    res = pj.search_local_landmarks(*args)
    ref = pj.match_frame_and_landmarks(fi, TP.SCALE_FACTORS, uv, xr, lv, lm_desc, ok, None, 5.0)
    assert res[0] == ref[0] and np.array_equal(res[1], ref[1])

    def host():
        loop()
        pj.match_frame_and_landmarks(fi, TP.SCALE_FACTORS, uv, xr, lv, lm_desc, ok, None, 5.0)
    host_ms = median_ms(host, calls)
    composed_ms = median_ms(lambda: pj.search_local_landmarks(*args), calls)
    kus = []
    for _ in range(calls):
        pj.can_observe(g, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5, s["usable"])
        kus.append(pj.last_kernel_us())
    fi.close()
    return dict(landmarks=nlm, observable=int(ok.sum()), matches=int(res[0]), host_loop_plus_matcher_ms=round(host_ms, 3),
                composed_ms=round(composed_ms, 3), kernel_us=round(float(np.median(kus)), 2))


def motion_model(pj, OT, W, H, nkp, calls):
    from openvslam_b200 import match
    s = scene("perspective", W, H, nkp, seed=2)
    g = s["geometry"]
    last_pose = s["pose_cw"].copy(); last_pose[11] += 0.05
    loop, (ok, uv, xr) = host_reproject(OT, s)
    loop()
    lv = np.random.default_rng(3).integers(0, TP.NUM_LEVELS, nkp).astype(np.int32)
    kp, lm_desc = frame(s, ok.astype(bool), uv, lv, nkp, seed=4)
    ang = np.zeros(nkp, np.float32)
    fi = match.frame_index(pj, kp["x"], kp["y"], kp["octave"], kp["angle"], None, kp["desc"], match.camera_grid(g.min_x, g.max_x, g.min_y, g.max_y))
    args = (fi, g, last_pose, TP.SCALE_FACTORS, s["pos_w"], lv, ang, lm_desc, s["usable"], None, 20.0, True, 0.0)
    res = pj.match_current_and_last_frames_reproject(*args)
    ref = pj.match_current_and_last_frames(fi, TP.SCALE_FACTORS, TP.NUM_LEVELS, ok, uv, xr, lv, ang, lm_desc, None, 20.0)
    assert res[0] == ref[0] and np.array_equal(res[1], ref[1])

    def host():
        loop()
        fw, bw = OT.motion_direction(s["pose_cw"], last_pose, True, 0.0)
        pj.match_current_and_last_frames(fi, TP.SCALE_FACTORS, TP.NUM_LEVELS, ok, uv, xr, lv, ang, lm_desc, None, 20.0, fw, bw)
    host_ms = median_ms(host, calls)
    composed_ms = median_ms(lambda: pj.match_current_and_last_frames_reproject(*args), calls)
    kus = []
    for _ in range(calls):
        pj.can_observe(g, s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5, s["usable"])
        kus.append(pj.last_kernel_us())
    fi.close()
    return dict(landmarks=nkp, in_image=int(ok.sum()), matches=int(res[0]), host_loop_plus_matcher_ms=round(host_ms, 3),
                composed_ms=round(composed_ms, 3), kernel_us=round(float(np.median(kus)), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from openvslam_b200 import match
    from oracle import oracle as O
    from oracle import tracking as OT
    O.build()
    name, power = gpu_info()
    pj = match.projection(lowe_ratio=0.8, check_orientation=True)
    lines = []
    for cfg, run in ((4, lambda: local_map_search(pj, OT, "equirectangular", 1920, 960, 4000, 20000, args.calls)),
                     (5, lambda: local_map_search(pj, OT, "perspective", 1920, 1080, 2000, 20000, args.calls)),
                     (2, lambda: motion_model(pj, OT, 752, 480, 1000, args.calls))):
        line = dict(tool="time_tracking_search", gpu=name, power_limit=power, config=cfg,
                    search="motion model" if cfg == 2 else "local map", keypoints={4: 4000, 5: 2000, 2: 1000}[cfg])
        line.update(run())
        print(json.dumps(line), flush=True)
        lines.append(line)
    pj.close()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
