"""Times solve::pnp_solver.find_via_ransac on the GPU (ovs_pnp_solve_ransac_host) against the C oracle on one host thread.

For B in {1, 8, 32} relocalisation candidates of n in {50, 300, 2000} correspondences (25 % wrong landmarks, bearing noise of 1e-3
rad, 30 hypotheses, recompute on): the median over warm calls of the host clock around one call (the call ends with a device
synchronise, so this is the device timeline plus the one copy each way), and the oracle's time for the same B problems, one
after another.  The GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE`
also writes them there.

    python tools/time_pnp_solver.py [--calls 30] [--out results.jsonl]
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

import pnp_problems as pp  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--oracle-calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from openvslam_b200 import solve
    from oracle import oracle as O
    from oracle import pnp_solver as ps
    O.build()
    name, power = gpu_info()
    solver = solve.pnp_solver(10)
    lines = []
    for n in (50, 300, 2000):
        for B in (1, 8, 32):
            probs = [pp.problem(n, wrong=0.25, noise=1e-3, seed=100 * b + n) for b in range(B)]
            gp = [pp.gpu_problem(p) for p in probs]
            seeds = list(range(B))
            for _ in range(3):
                out = solver.find_via_ransac(gp, 30, True, seeds)
            ts = []
            for _ in range(a.calls):
                t0 = time.perf_counter()
                solver.find_via_ransac(gp, 30, True, seeds)
                ts.append(time.perf_counter() - t0)
            to = []
            for _ in range(a.oracle_calls):
                t0 = time.perf_counter()
                for b, p in enumerate(probs):
                    o = ps.pnp_solve_ransac(*pp.args(p), min_num_inliers=10, max_num_iter=30, recompute=True, seed=b)
                to.append(time.perf_counter() - t0)
            assert o["num_inliers"] == out[-1]["num_inliers"] and np.array_equal(o["pose_cw"], out[-1]["pose_cw"])
            line = dict(metric="pnp_solver_call_ms", B=B, n=n, hypotheses=30, gpu_ms_median=1e3 * float(np.median(ts)),
                        gpu_ms_min=1e3 * float(np.min(ts)), oracle_one_thread_ms=1e3 * float(np.median(to)), calls=a.calls, gpu=name,
                        power_limit=power)
            print(json.dumps(line), flush=True)
            lines.append(line)
    solver.close()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
