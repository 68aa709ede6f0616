#!/usr/bin/env python
"""Per-kernel device time of the flagship workload (bench.py config 4, value leg: every input resident in HBM, eight camera
streams on one GPU, each on its own host thread), measured with torch.profiler (CUDA activities) in a run of its own.

Prints one table: for every kernel, its device time per frame (summed over the eight streams' launches, divided by the frames
of all streams), launches per frame and share of the total; then one JSON line with the same numbers, the GPU's name and its
power limit.  Profiling slows the host side, so frames/s belong to bench.py; the per-kernel device times are what this is for.

  python tools/profile_ba_kernels.py [--steps 20] [--warmup 3] [--streams 8] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def gpu_info(index):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, plim, clk = [c.strip() for c in r.stdout.strip().split(",")[:3]]
        return dict(name=name, power_limit=plim, sm_max_clock=clk)
    except Exception as e:  # noqa: BLE001
        return dict(name="unknown", error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="profiled frames per stream")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--top", type=int, default=40, help="kernels listed in the table")
    ap.add_argument("--out", default="", help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from openvslam_b200 import _lib, feature

    cfg = bench.CONFIGS[4]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    S = args.streams
    ring = bench.default_ring(cfg)
    wl = bench.make_workload(cfg, 0, ring)
    W, H, NKP = cfg["W"], cfg["H"], cfg["NKP"]
    _lib.lib().ovs_set_wait_mode(0 if S <= max(1, bench.host_cores() - 2) else 2)   # as bench.py --wait auto
    h = torch.empty((ring, H, W), dtype=torch.uint8).pin_memory()
    for i, f in enumerate(wl["frames"]):
        h[i].copy_(torch.from_numpy(f))
    d_frames = h.to(dev)
    torch.cuda.synchronize()
    ext0 = feature.orb_extractor(feature.orb_params(max_num_keypts=NKP), device=0)
    lmsets = bench.make_landmark_sets(cfg, wl, ext0)
    ext0.close()
    cluster = 8 if S == 1 else 2                  # bench.py's default for one / several streams
    cams = [bench.CameraStream(cfg, sid, 0, dev, d_frames, h.numpy(), None, None, wl, lmsets, ring, 4, cluster) for sid in range(S)]

    def run_all(lo, hi):
        errs = []

        def work(cs):
            try:
                torch.cuda.set_device(0)
                for i in range(lo, hi):
                    cs.step_device(i)
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        ths = [threading.Thread(target=work, args=(cs,)) for cs in cams]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        if errs:
            raise errs[0]

    run_all(0, args.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        run_all(args.warmup, args.warmup + args.steps)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    frames = S * args.steps
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        if name.startswith("Memcpy") or name.startswith("Memset"):
            name = name.split(" ")[0] + " " + (name.split(" ")[1] if " " in name else "")
        else:
            for tok in ("(anonymous namespace)::", "void "):
                name = name.replace(tok, "")
            name = name.split("(")[0]
        d = per.setdefault(name, [0.0, 0])
        d[0] += us
        d[1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(((k, v[0] / frames, v[1] / frames) for k, v in per.items()), key=lambda r: -r[1])
    info = gpu_info(0)
    print("GPU: %s, power limit %s, max SM clock %s" % (info.get("name"), info.get("power_limit"), info.get("sm_max_clock")))
    print("config 4 value leg, %d streams x %d frames (profiled, wall %.2f s)" % (S, args.steps, wall))
    print("%-40s %12s %10s %7s" % ("kernel", "us/frame", "launches", "share"))
    for k, us, n in rows[:args.top]:
        print("%-40s %12.1f %10.1f %6.1f%%" % (k[:40], us, n, 100.0 * us / (total / frames)))
    print("%-40s %12.1f" % ("total device time", total / frames))
    ba = sum(us for k, us, _ in rows if k.startswith(("k_ba_", "k_chol_", "k_lm_")))
    print("%-40s %12.1f" % ("of which local BA kernels", ba))
    res = dict(gpu=info, streams=S, steps=args.steps, device_us_per_frame=total / frames, ba_us_per_frame=ba,
               kernels={k: dict(us_per_frame=round(us, 2), launches_per_frame=round(n, 2)) for k, us, n in rows})
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    for cs in cams:
        cs.close()


if __name__ == "__main__":
    main()
