"""Times util::stereo_rectifier on the device at three stereo shapes:

  euroc    752 x 480 gray pair (EuRoC)
  config3  1241 x 376 gray pair (bench.py configuration 3)
  config5  1920 x 1080 BGR pair (bench.py configuration 5)

Per shape:
  remap_us_per_pair     device time of the two remap kernels of one ovs_stereo_rectify_host call (channels kept), from
                        torch.profiler's kernel records over warm calls, in a profiled run of its own;
  remap_gray_us         device time of the fused remap + gray kernel of one ovs_extract_host_rectified call (one side);
  bytes_per_pair        what the remap has to move, from the shapes: per side the 8-byte fixed-point map entry, the source
                        pixel and the output pixel (channels each); achieved bytes/s = bytes_per_pair / remap time, against the
                        H100 SXM data sheet's 3.35 TB/s;
  extract_rectified_ms  median host time of one ovs_extract_host_rectified call (one side; it ends in a device synchronise);
  host_remap_plus_extract_ms  what a user does without it: cv2.remap on the host (cv2's own threads) and then ovs_extract_host
                        (gray) or ovs_extract_host_color (BGR) on the remapped image;
  host_remap_ms         the cv2.remap alone.
The GPU's name and power limit are read in the same run.  Prints one JSON line per shape; `--out FILE` also writes them there.

    python tools/time_stereo_rectify.py [--calls 100] [--out results/h100_stereo_rectify.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rectify_cases as RC  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = [("euroc", 752, 480, 1), ("config3", 1241, 376, 1), ("config5", 1920, 1080, 3)]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def median_ms(fn, calls):
    for _ in range(5):
        fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def kernel_us(fn, calls, gray):
    """mean device time per call of the remap kernels `fn` launches (the gray variant or the channel-keeping one)"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
    tot, n = 0.0, 0
    for e in prof.key_averages():
        if "k_stereo_remap" in e.key and (("true" in e.key) == gray):
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total")
            n += e.count
    if n == 0:
        raise RuntimeError("no k_stereo_remap kernel in the profile")
    return tot / calls, n / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--out")
    a = ap.parse_args()
    import cv2
    from openvslam_b200 import feature, synth, util
    name, power = gpu_info()
    lines = []
    for tag, W, H, ch in SHAPES:
        r = RC.rig("perspective", W, H, seed=W + H, rot=0.02)
        rect = util.stereo_rectifier(W, H, r["K_rect"], r["K_l"], r["D_l"], r["R_l"], r["K_r"], r["D_r"], r["R_r"])
        gray_l, gray_r = synth.frame(W, H, seed=1), synth.frame(W, H, seed=2)
        if ch == 1:
            il, ir = gray_l, gray_r
        else:
            il = np.ascontiguousarray(np.stack([gray_l, 255 - gray_l, gray_l // 2 + 64], 2))
            ir = np.ascontiguousarray(np.stack([gray_r, 255 - gray_r, gray_r // 2 + 64], 2))
        remap_us, per_call = kernel_us(lambda: rect.rectify(il, ir), a.calls, gray=False)
        ext = feature.orb_extractor(feature.orb_params(max_num_keypts=2000 if W > 1000 else 1000))
        gray_us, _ = kernel_us(lambda: ext.extract(il, rectifier=rect, side=0), a.calls, gray=True)
        mx, my = rect.maps(0)
        t_rect = median_ms(lambda: ext.extract(il, rectifier=rect, side=0), a.calls)
        t_host = median_ms(lambda: ext.extract(cv2.remap(il, mx, my, cv2.INTER_LINEAR)), a.calls)
        t_remap = median_ms(lambda: cv2.remap(il, mx, my, cv2.INTER_LINEAR), a.calls)
        nbytes = 2 * W * H * (8 + ch + ch)
        line = dict(shape=tag, width=W, height=H, channels=ch, remap_kernels_per_call=per_call, remap_us_per_pair=round(remap_us, 2),
                    remap_gray_us=round(gray_us, 2), bytes_per_pair=nbytes,
                    achieved_TBps=round(nbytes / (remap_us * 1e-6) / 1e12, 3),
                    share_of_3_35_TBps=round(nbytes / (remap_us * 1e-6) / HBM_BYTES_PER_S, 3),
                    extract_rectified_ms=round(t_rect, 3), host_remap_plus_extract_ms=round(t_host, 3), host_remap_ms=round(t_remap, 3),
                    cv2_threads=cv2.getNumThreads(), calls=a.calls, gpu=name, power_limit=power)
        print(json.dumps(line), flush=True)
        lines.append(line)
        ext.close(); rect.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
