"""Times solve::essential_solver.find_via_ransac on the GPU (ovs_essential_solve_ransac_host) against the C oracle on one host thread.

For B = 1 problem of n in {300, 2000, 4000} matches and B = 32 problems of 300 and of 2000 (25 % wrong matches, bearing noise of
1e-3 rad, 50 hypotheses, recompute on and off): the median over warm calls of the host clock around one call (the call ends with a
device synchronise, so this is the device timeline plus the one copy each way), and the oracle's time for the same B problems, one
after another.  The GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE` also
writes them there.

    python tools/time_essential_solver.py [--calls 30] [--out results.jsonl]
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

import essential_problems as ep  # noqa: E402


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
    from oracle import essential_solver as es
    O.build()
    name, power = gpu_info()
    solver = solve.essential_solver()
    lines = []
    H = 50
    for B, n in ((1, 300), (1, 2000), (1, 4000), (32, 300), (32, 2000)):
        for recompute in (True, False):
            probs = [ep.problem(n, model="equirectangular" if b % 2 else "perspective", wrong=0.25, noise=1e-3, seed=100 * b + n)
                     for b in range(B)]
            gp = [ep.gpu_problem(p) for p in probs]
            seeds = list(range(B))
            for _ in range(3):
                out = solver.find_via_ransac(gp, H, recompute, seeds)
            ts = []
            for _ in range(a.calls):
                t0 = time.perf_counter()
                solver.find_via_ransac(gp, H, recompute, seeds)
                ts.append(time.perf_counter() - t0)
            to = []
            for _ in range(a.oracle_calls):
                t0 = time.perf_counter()
                for b, p in enumerate(probs):
                    o = es.essential_solve_ransac(p["bearings_1"], p["bearings_2"], H, recompute=recompute, seed=b)
                to.append(time.perf_counter() - t0)
            assert o["num_inliers"] == out[-1]["num_inliers"] and np.array_equal(o["E_21"], out[-1]["E_21"])
            line = dict(metric="essential_solver_call_ms", B=B, n=n, hypotheses=H, recompute=recompute,
                        gpu_ms_median=1e3 * float(np.median(ts)), gpu_ms_min=1e3 * float(np.min(ts)),
                        oracle_one_thread_ms=1e3 * float(np.median(to)), calls=a.calls, gpu=name, power_limit=power)
            print(json.dumps(line), flush=True)
            lines.append(line)
    solver.close()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
