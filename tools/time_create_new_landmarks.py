"""Times the compute step of mapping_module::create_new_landmarks on the GPU (ovs_create_new_landmarks_host: every neighbour's
triangulation matcher and triangulator in one call) against the shape it replaces: B single match_for_triangulation calls on the GPU
(ovs_robust_match_for_triangulation_host), each followed by the oracle's host triangulation of its pairs, with keyframe 1's landmark
flags carried from one neighbour to the next.  The oracle's keyframe records are built once, outside the timed calls, so the
baseline's host side is the matcher's Python wrapper and the C triangulation; the composed call's includes its Python wrapper
(module.create_new_landmarks, which flattens every keyframe on each call).

For B in {1, 10, 20} neighbours and n1 in {1500, 4000} keypoints (the scenes of tests/triangulation_problems.py, 30 % stereo
keypoints, orientation check on): the median over warm calls of the host clock around one call (each ends with a device
synchronise).  The GPU's name and power limit are read in the same run.  Prints one JSON line per configuration; `--out FILE` also
writes them there.

    python tools/time_create_new_landmarks.py [--calls 20] [--out results.jsonl]
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

import triangulation_problems as tp  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: no GPU to time on")
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return name, power


def marshal(OT, keyframes):
    """the oracle's keyframe records, built once: the timed loop then pays only the C triangulation, as a C++ caller would"""
    keep = []
    return [OT._kf(k, keep) for k in keyframes], keep


def loop_of_single_calls(mt, OT, kf1, nbs, E, ep, recs):
    """the per-neighbour shape: one GPU matcher call and the oracle's C triangulation of its pairs per neighbour"""
    import ctypes as C
    lib = OT.lib()
    r1 = recs[0]
    has = kf1.has_landmark.copy()
    st1 = (kf1.stereo_x_right >= 0).astype(np.uint8)
    cos_thr = C.c_double(1.0)
    num = 0
    for b, n in enumerate(nbs):
        st2 = (n.stereo_x_right >= 0).astype(np.uint8)
        _, m = mt.match_for_triangulation(kf1.descriptors, kf1.bearings, kf1.keypts["octave"], kf1.keypts["angle"], has, st1, kf1.bow_node,
                                          n.descriptors, n.bearings, n.keypts["angle"], n.has_landmark, st2, n.bow_node, E[b], ep[b],
                                          kf1.scale_factors)
        i1 = np.flatnonzero(m >= 0)
        pairs = np.ascontiguousarray(np.stack([i1, m[i1]], 1), np.int32)
        k = max(len(pairs), 1)
        valid = np.zeros(k, np.uint8); pos = np.zeros((k, 3)); reason = np.zeros(k, np.int32); branch = np.zeros(k, np.int32)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        lib.otr_two_view_triangulate(C.byref(r1), C.byref(recs[1 + b]), len(pairs), vp(pairs), cos_thr, vp(valid), vp(pos), vp(reason),
                                     vp(branch))
        ok = valid[:len(pairs)].astype(bool)
        has[i1[ok]] = 1
        num += int(ok.sum())
    return num


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
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from openvslam_b200 import match, module
    from oracle import oracle as O
    from oracle import triangulation as OT
    O.build()
    name, power = gpu_info()
    mt = match.robust(check_orientation=True)
    lines = []
    for n1 in (1500, 4000):
        for B in (1, 10, 20):
            kf1, nbs, E, ep = tp.neighbourhood(1000 + n1 + B, n1, B, stereo_frac=0.3)
            rec, _ = module.create_new_landmarks(mt, kf1, nbs, E, ep, True)
            recs, _keep = marshal(OT, [kf1] + nbs)
            n_loop = loop_of_single_calls(mt, OT, kf1, nbs, E, ep, recs)
            assert n_loop == len(rec)
            composed = median_ms(lambda: module.create_new_landmarks(mt, kf1, nbs, E, ep, True), args.calls)
            single = median_ms(lambda: loop_of_single_calls(mt, OT, kf1, nbs, E, ep, recs), max(3, args.calls // 4))
            line = dict(tool="time_create_new_landmarks", gpu=name, power_limit=power, n1=n1, B=B, landmarks=len(rec),
                        composed_ms=round(composed, 3), single_calls_plus_host_triangulation_ms=round(single, 3))
            print(json.dumps(line), flush=True)
            lines.append(line)
    mt.close()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
