#!/usr/bin/env python
"""Generates tests/golden/ba_edge_record_golden.npz: local and global bundle-adjuster results of the CUDA path on seeded graphs of
tests/ba_graphs.py, stored bit for bit.  The vectors pin the adjusters' arithmetic: a change to how the per-edge blocks are stored
or accumulated that keeps every sum in its order must reproduce them exactly (tests/test_ba_edge_record_gpu.py).
The graphs cover 2-row edges only (mono, equirectangular), 2- and 3-row edges in one problem (stereo with monocular keyframes),
outliers leaving the graph between the two rounds of the local adjuster, and a landmark observed by more than 128 keyframes.
Made on an H100 by the revision before the compact edge record (git revision stored in the file).
Re-run (needs a GPU): python tests/golden/make_ba_edge_record_golden.py [OUT]"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ba_graphs as bg  # noqa: E402

# name -> (kind, graph arguments); kind "local" = local_bundle_adjuster(5, 10), "global" = global_bundle_adjuster(10, huber)
CASES = {
    "mono": ("local", dict(num_free=16, num_fixed=3, num_landmarks=500, seed=31)),
    "stereo_mono": ("local", dict(num_free=10, num_fixed=3, fixed="first", num_landmarks=400, stereo=True, mono_keyframes=(0, 4, 5, 9, 11),
                                  behind=6, seed=32)),
    "equirectangular": ("local", dict(num_free=12, num_fixed=2, fixed="first", num_landmarks=400, model="equirectangular", seed=33)),
    "outliers": ("local", dict(num_free=20, num_fixed=4, fixed="interleaved", num_landmarks=600, outlier_frac=0.2, seed=34)),
    "seen_by_140_global": ("global", dict(num_free=140, num_fixed=6, num_landmarks=700, views=(2, 6), seen_by_all=2, seed=35)),
    "seen_by_140_local": ("local", dict(num_free=140, num_fixed=6, num_landmarks=700, views=(2, 6), seen_by_all=2, seed=35)),
}


def run_case(name):
    """-> dict of arrays: poses, points, outliers (local only), num_iterations, num_trials"""
    from openvslam_b200 import optimize
    kind, kw = CASES[name]
    g = bg.graph(**kw)
    cam = optimize.camera(**g["cam"])
    if kind == "local":
        ba = optimize.local_bundle_adjuster(5, 10)
        poses, points, outl, st = ba.optimize(cam, g["setup_is_mono"], *bg.args(g))
    else:
        ba = optimize.global_bundle_adjuster(10, True)
        poses, points, st = ba.optimize(cam, g["setup_is_mono"], *bg.args(g))
        outl = np.zeros(0, bool)
    ba.close()
    return dict(poses=poses, points=points, outliers=outl, num_iterations=np.array(st["num_iterations"]),
                num_trials=np.array(st["num_trials"]))


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ba_edge_record_golden.npz")
    vec = {}
    for name in CASES:
        for k, v in run_case(name).items():
            vec[name + "/" + k] = v
    try:
        rev = subprocess.run(["git", "rev-parse", "HEAD"], cwd=ROOT, capture_output=True, text=True).stdout.strip()
    except OSError:
        rev = ""
    vec["revision"] = np.array(rev or os.environ.get("OVS_GOLDEN_REVISION", "unknown"))
    np.savez_compressed(out, **vec)
    print(out)


if __name__ == "__main__":
    main()
