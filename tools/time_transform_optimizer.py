"""Times optimize::transform_optimizer on the GPU (ovs_transform_optimize_host, one k_sim3_optimize launch per call).

For n in {100, 1000} pairs (perspective, free scale, 15 % wrong pairs, the reference's 5 + 10 iterations): the median and the
spread of the call's own device time (stats["device_us"], CUDA events around the kernel) over warm calls on one problem.  The
GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE` also writes them there.

    python tools/time_transform_optimizer.py [--calls 50] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sim3_problems as sp  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from openvslam_b200 import optimize
    name, power = gpu_info()
    opt = optimize.transform_optimizer(False)
    lines = []
    for n in (100, 1000):
        p = sp.problem(n, seed=100 + n)
        cam = optimize.camera(**p["cam"])
        for _ in range(a.warmup):
            opt.optimize(cam, cam, *sp.args(p))
        us = [opt.optimize(cam, cam, *sp.args(p))[3]["device_us"] for _ in range(a.calls)]
        line = dict(metric="transform_optimizer_device_us", n=n, median_us=float(np.median(us)), min_us=float(np.min(us)),
                    max_us=float(np.max(us)), calls=a.calls, gpu=name, power_limit=power)
        print(json.dumps(line), flush=True)
        lines.append(line)
    opt.close()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
