"""Times perspective map initialisation on the GPU (ovs_initialize_perspective_host: both RANSAC solvers, the model choice, the
decomposition, check_pose on every hypothesis and the choice, in one call) against
  - the two solver calls alone on the GPU (ovs_homography_solve_ransac_host + ovs_fundamental_solve_ransac_host on the same
    matches and seeds): what a caller ran on the device before, with the reconstruct still to do on the host;
  - the oracle's reconstruct on one CPU thread: the oracle's whole initialize (C, -O3) minus its two solves, both timed on the
    same problems (the reconstruct is what the composed call adds to the two solver calls).
For m in {300, 1000, 4000} matches (general scenes of tests/initializer_problems.py, 20 % wrong matches, 1 px noise, 100 RANSAC
iterations) and B in {1, 8} problems: the median over warm calls of the host clock around one call (each GPU call ends with a
device synchronise).  The GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out
FILE` also writes them there.

    python tools/time_initializer.py [--calls 20] [--oracle-calls 3] [--out results.jsonl]
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

import initializer_problems as IP  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def median_ms(fn, calls):
    fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--oracle-calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from openvslam_b200 import initialize, optimize, solve
    from oracle import oracle as O
    from oracle.oracle import lib as olib
    import oracle.initializer as OI
    O.build()
    name, power = gpu_info()
    init = initialize.perspective(None)
    hs, fs = solve.homography_solver(), solve.fundamental_solver()
    cam = optimize.camera("perspective", fx=500.0, fy=500.0, cx=320.0, cy=240.0, cols=640.0, rows=480.0)
    lines = []
    for m in (300, 1000, 4000):
        for B in (1, 8):
            ps = [IP.problem(m, wrong=0.2, noise=1.0, seed=1000 * m + b) for b in range(B)]
            seeds = np.arange(B, dtype=np.uint64)
            views = [dict(ref=initialize.view(cam, p["keypts_ref"], p["bearings_ref"]), cur=initialize.view(cam, p["keypts_cur"], p["bearings_cur"]),
                          ref_matches_with_cur=p["ref_matches_with_cur"]) for p in ps]
            tv = []
            for p in ps:
                ri = np.nonzero(p["ref_matches_with_cur"] >= 0)[0]
                tv.append(dict(keypts_1=p["keypts_ref"], keypts_2=p["keypts_cur"], matches_12=np.stack([ri, p["ref_matches_with_cur"][ri]], 1)))
            got = init.initialize_batch(views, seeds)
            composed = median_ms(lambda: init.initialize_batch(views, seeds), args.calls)
            solvers = median_ms(lambda: (hs.find_via_ransac(tv, 100, True, seeds), fs.find_via_ransac(tv, 100, True, seeds)), args.calls)

            def oracle_init():
                for b, p in enumerate(ps):
                    OI.initialize(*IP.oracle_args(p), seed=b)

            def oracle_solves():
                L = olib()
                for b, p in enumerate(ps):
                    k1 = np.ascontiguousarray(p["keypts_ref"]); k2 = np.ascontiguousarray(p["keypts_cur"])
                    pr = np.ascontiguousarray(tv[b]["matches_12"], np.int32)
                    M = np.zeros(9); fl = np.zeros(len(pr), np.uint8)
                    v, n, bi, sc = C.c_int(), C.c_int(), C.c_int(), C.c_double()
                    vp = lambda a: a.ctypes.data_as(C.c_void_p)
                    for model in (0, 1):
                        L.ot_solve_ransac(model, len(k1), vp(k1), len(k2), vp(k2), len(pr), vp(pr), C.c_float(1.0), 100, 1, C.c_uint64(b),
                                          vp(M), C.byref(v), C.byref(n), C.byref(bi), C.byref(sc), vp(fl), None, None, None, None)
            o_init = median_ms(oracle_init, args.oracle_calls)
            o_solve = median_ms(oracle_solves, args.oracle_calls)
            line = dict(tool="time_initializer", gpu=name, power_limit=power, m=m, B=B, ok=sum(g["ok"] for g in got),
                        models="".join(str(g["model"] or "-") for g in got), composed_ms=round(composed, 3),
                        h_plus_f_solver_calls_ms=round(solvers, 3), oracle_initialize_ms=round(o_init, 3),
                        oracle_solves_ms=round(o_solve, 3), oracle_reconstruct_ms=round(o_init - o_solve, 3))
            print(json.dumps(line), flush=True)
            lines.append(line)
    init.close(); hs.close(); fs.close()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
