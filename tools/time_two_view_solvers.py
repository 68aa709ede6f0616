"""Times solve::homography_solver and solve::fundamental_solver .find_via_ransac on the GPU (ovs_homography_solve_ransac_host,
ovs_fundamental_solve_ransac_host) against the C oracle on one host thread.

For B = 1 problem of m in {300, 1000, 4000} matches (2000 keypoints per view, 4000 at m = 4000) and B = 8 and 32 problems of 1000
matches (25 % wrong matches, 1 px of noise, 100 and 200 hypotheses, recompute on, both models): the median over warm calls of the
host clock around one call (the call ends with a device synchronise, so this is the device timeline plus the one copy each way),
and the oracle's time for the same B problems, one after another.  The GPU's name and power limit are read in the same run.
Prints one JSON line per configuration; `--out FILE` also writes them there.

    python tools/time_two_view_solvers.py [--calls 20] [--out results.jsonl]
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

import two_view_problems as tp  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--oracle-calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from openvslam_b200 import solve
    from oracle import oracle as O
    from oracle import two_view_solver as tv
    O.build()
    name, power = gpu_info()
    solvers = {"H": solve.homography_solver(), "F": solve.fundamental_solver()}
    key = {"H": "H_21", "F": "F_21"}
    lines = []
    for B, m in ((1, 300), (1, 1000), (1, 4000), (8, 1000), (32, 1000)):
        nk = 4000 if m == 4000 else 2000
        probs = [tp.problem(m, scene="planar" if b % 2 else "general", wrong=0.25, noise=1.0, seed=100 * b + m, n1=nk, n2=nk)
                 for b in range(B)]
        gp = [tp.gpu_problem(p) for p in probs]
        seeds = list(range(B))
        for model in ("H", "F"):
            for H in (100, 200):
                s = solvers[model]
                for _ in range(3):
                    out = s.find_via_ransac(gp, H, True, seeds)
                ts = []
                for _ in range(a.calls):
                    t0 = time.perf_counter()
                    s.find_via_ransac(gp, H, True, seeds)
                    ts.append(time.perf_counter() - t0)
                to = []
                for _ in range(a.oracle_calls):
                    t0 = time.perf_counter()
                    for b, p in enumerate(probs):
                        o = tv.solve_ransac(model, p["keypts_1"], p["keypts_2"], p["matches_12"], H, recompute=True, seed=b)
                    to.append(time.perf_counter() - t0)
                assert o["num_inliers"] == out[-1]["num_inliers"] and np.array_equal(o["M"], out[-1][key[model]])
                line = dict(metric="two_view_solver_call_ms", model=model, B=B, matches=m, keypoints_per_view=nk, hypotheses=H,
                            recompute=True, gpu_ms_median=1e3 * float(np.median(ts)), gpu_ms_min=1e3 * float(np.min(ts)),
                            oracle_one_thread_ms=1e3 * float(np.median(to)), calls=a.calls, gpu=name, power_limit=power)
                print(json.dumps(line), flush=True)
                lines.append(line)
    for s in solvers.values():
        s.close()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
