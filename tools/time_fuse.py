"""Times mapping_module::fuse_landmark_duplication's compute (match::fuse::replace_duplication, forward into every target and
backward into the current keyframe) with ovs_fuse_replace_duplication_host against what a caller does without it, at bench.py's
shapes:

  config 4  equirectangular 1920 x 960, 4000 keypoints per keyframe
  config 5  perspective 1920 x 1080, 2000 keypoints per keyframe

each at 20 and 120 target keyframes.  The current keyframe holds 1500 landmarks (forward: every one listed for every target); the
backward pass queries 20 000 landmarks, the union of the targets' landmarks.  Four numbers per configuration:
  (a) per_target_ms   the oracle's C geometry loop (reproject_to_image, the two gates, predict_scale_level, one landmark after the
                      other on one thread) plus, per target and for the backward pass, one ovs_frame_index_create,
                      ovs_fuse_best_keypoints_host and ovs_frame_index_destroy: the caller's shape today;
  (b) composed_ms     the two calls of ovs_fuse_replace_duplication_host (B targets, then B = 1);
  (c) kernel_us       their two kernels by CUDA events (the handle's last_kernel_us of each call, summed);
  (d) h2d_ms, h2d_share  a pinned host-to-device copy of the two calls' staged inputs (their byte count, measured alone with CUDA
                      events) and its share of (b).
The call times are medians over warm calls of the host clock around the whole sequence (each call ends with a device wait).  The
GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE` also writes them there.

    python tools/time_fuse.py [--calls 20] [--out results.jsonl]
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

import fuse_problems as FP  # noqa: E402
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


def make(config, B, seed):
    from openvslam_b200 import match
    if config == 4:
        FP.CAMERAS["bench4"] = ("equirectangular", dict(cols=1920.0, rows=960.0), (0.0, 1920.0, 0.0, 960.0), False)
        scene, nkp = "bench4", 4000
    else:
        FP.CAMERAS["bench5"] = ("perspective", dict(fx=1000.0, fy=1000.0, cx=960.0, cy=540.0), (0.0, 1920.0, 0.0, 1080.0), False)
        scene, nkp = "bench5", 2000
    rng = np.random.default_rng(seed)
    lms = FP.landmarks(20000, rng, config == 4)
    targets, arrays = [], []
    for _ in range(B):
        t, a = FP.target(scene, lms, nkp, rng)
        targets.append(t); arrays.append(a)
    cur, cur_a = FP.target(scene, lms, nkp, rng, pose=TP.pose12(np.eye(3), np.zeros(3)))
    cur_rows = rng.choice(20000, 1500, replace=False).astype(np.int32)
    fwd_off = (np.arange(B + 1) * 1500).astype(np.int32)
    fwd_lm = np.tile(cur_rows, B)
    bwd_lm = np.arange(20000, dtype=np.int32)
    return match, targets, arrays, cur, cur_a, lms, fwd_off, fwd_lm, bwd_lm


def staged_bytes(B, nkp_total, ncells_total, nlm, nq):
    # inputs of one call as fuse.cu stages them: targets, (target, row) per query, the landmark table, the keypoints in rank order
    # and the cell starts (each buffer 256-byte aligned: ignored)
    return B * 400 + 8 * nq + (24 + 24 + 4 + 4 + 32) * nlm + (4 + 4 + 4 + 1 + 32) * nkp_total + 4 * ncells_total


def run(config, B, calls, name, power):
    import torch
    from openvslam_b200 import _lib
    from oracle import oracle as O
    match, targets, arrays, cur, cur_a, lms, fwd_off, fwd_lm, bwd_lm = make(config, B, seed=config * 1000 + B)
    fz = match.fuse()
    L = _lib.lib()
    lm_args = (lms["pos_w"], lms["mean_normal"], lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"])
    out = {}

    def composed():
        n1, _ = fz.replace_duplication(targets, *lm_args, fwd_off, fwd_lm)
        k1 = fz.last_kernel_us()
        n2, _ = fz.replace_duplication([cur], *lm_args, np.array([0, len(bwd_lm)], np.int32), bwd_lm)
        out.update(fused=n1 + n2, kernel_us=k1 + fz.last_kernel_us())

    # (a): the oracle's geometry on one thread, then one index build and one matching-core call per target
    from oracle import fuse as OF
    lib_o = O.lib()
    f_obs = lib_o.ott_fuse_observe
    f_obs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    pos = np.ascontiguousarray(lms["pos_w"]); nrm = np.ascontiguousarray(lms["mean_normal"])
    lo = lms["min_valid_dist"]; hi = lms["max_valid_dist"]
    vp = lambda a: a.ctypes.data_as(C.c_void_p)

    def geometry_c(a, rows):
        # the C loop of the oracle over the queries (one ctypes call per target: ott_fuse_replace_duplication_all's geometry part is
        # the same loop; its search is replaced here by the GPU core)
        n = len(rows)
        ok = np.zeros(n, np.uint8); uv = np.zeros((n, 2), np.float32); xr = np.zeros(n, np.float32); lv = np.zeros(n, np.int32)
        best = np.zeros(n, np.int32)
        empty = O.MatchFrame(np.zeros(0, np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32), np.zeros(0, np.float32), None,
                             np.zeros((0, 32), np.uint8), O.om_grid(a["geometry"].min_x, a["geometry"].max_x, a["geometry"].min_y, a["geometry"].max_y))
        OF_lib = lib_o.ott_fuse_replace_duplication_all
        OF_lib.argtypes = [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 6 + [C.c_float] + [C.c_void_p] * 5
        sf = FP.SCALE_FACTORS; iw = FP.INV_LEVEL_SIGMA_SQ
        OF_lib(C.addressof(a["geometry"]), C.addressof(empty.c), vp(sf), vp(iw), n, vp(rows), vp(pos), vp(nrm), vp(lo), vp(hi), vp(lms["lm_desc"]),
               3.0, vp(best), vp(ok), vp(uv), vp(xr), vp(lv))
        return ok, uv, xr, lv

    def per_target():
        total = 0
        for a, rows in [(a, fwd_lm[:1500]) for a in arrays] + [(cur_a, bwd_lm)]:
            ok, uv, xr, lv = geometry_c(a, rows)
            idx = match.frame_index(fz, a["x"], a["y"], a["octave"], np.zeros(len(a["x"]), np.float32), a["x_right"], a["desc"], a["grid"])
            n, _ = fz.best_keypoints(idx, uv, xr, lv, lms["lm_desc"][rows], FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, 3.0, usable=ok)
            idx.close()
            total += n
        out["fused_per_target"] = total

    composed_ms = median_ms(composed, calls)
    per_target_ms = median_ms(per_target, max(3, calls // 4))
    nkp = sum(t.n for t in targets)
    nbytes = staged_bytes(B, nkp, B * (64 * 48 + 1), 20000, len(fwd_lm)) + staged_bytes(1, cur.n, 64 * 48 + 1, 20000, len(bwd_lm))
    h = torch.empty(nbytes, dtype=torch.uint8).pin_memory(); d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(10):
        e0.record(); d.copy_(h, non_blocking=True); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    h2d_ms = float(np.median(ts[2:]))
    composed()
    rec = {"tool": "time_fuse", "gpu": name, "power_limit": power, "config": config, "targets": B, "keypoints_per_keyframe": int(targets[0].n),
           "current_landmarks": 1500, "backward_landmarks": int(len(bwd_lm)), "queries": int(len(fwd_lm) + len(bwd_lm)), "fused": int(out["fused"]),
           "fused_per_target_shape": int(out["fused_per_target"]), "per_target_ms": round(per_target_ms, 3), "composed_ms": round(composed_ms, 3),
           "kernel_us": round(out["kernel_us"], 1), "staged_mb": round(nbytes / 1e6, 2), "h2d_ms": round(h2d_ms, 3),
           "h2d_share": round(h2d_ms / composed_ms, 3)}
    fz.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    name, power = gpu_info()
    lines = []
    for config in (4, 5):
        for B in (20, 120):
            rec = run(config, B, args.calls, name, power)
            print(json.dumps(rec), flush=True)
            lines.append(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
