"""Re-query and launch counts of the greedy replays, call by call: every window_match_reference case (the synthetic ones and
bench2 / bench4), and the inputs of the re-query tests of bow_tree, match_for_triangulation, create_new_landmarks and
robust::brute_force_match.  Each line: the call, its num_requeries() and _lib.launch_count() deltas and a digest of its
result.  Two revisions compute the same matches with the same GPU work when they print the same lines; run the other
revision's package first on PYTHONPATH:

    python tools/count_requeries.py [--out FILE]
    PYTHONPATH=<other tree> python tools/count_requeries.py [--out FILE]
"""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path += [ROOT, os.path.join(ROOT, "tests")]   # appended: a package on PYTHONPATH comes first


def digest(res):
    h = hashlib.sha1()
    for a in (res if isinstance(res, tuple) else (res,)):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import openvslam_b200
    import torch
    from openvslam_b200 import _lib, feature, match, module, synth
    from oracle import oracle as O
    import window_match_reference as R
    import test_window_match_reference_gpu as TW
    import test_match_gpu as TM
    import test_two_view_triangulator_gpu as TT
    import triangulation_problems as TP

    lines = []

    def record(name, mt, fn):
        r0, l0 = mt.num_requeries(), _lib.launch_count()
        res = fn()
        line = {"call": name, "requeries": mt.num_requeries() - r0, "launches": _lib.launch_count() - l0, "result": digest(res)}
        lines.append(line)
        print(json.dumps(line), flush=True)

    def window_case(case):
        for i, (kind, kw) in enumerate(case.calls):
            if kind == "angles":
                continue
            l0 = _lib.launch_count()
            res, nrq = TW.run_gpu(case, kind, kw)   # a matcher and an index of its own: nrq is this call's
            line = {"call": "%s/%d/%s" % (case.name, i, kind), "requeries": nrq, "launches": _lib.launch_count() - l0, "result": digest(res)}
            lines.append(line)
            print(json.dumps(line), flush=True)

    for name in sorted(R.SYNTHETIC_CASES):
        window_case(R.SYNTHETIC_CASES[name]())
    a = synth.frame(752, 480, seed=200)
    ka, da, _ = O.extract(a, O.params(1000))
    kb, db, _ = O.extract(synth.shifted(a, 3, 0), O.params(1000))
    window_case(R.bench2(ka, da, kb, db))
    ext = feature.orb_extractor(feature.orb_params(max_num_keypts=4000))
    kps, desc = ext.extract(synth.frame(1920, 960, seed=400))
    ext.close()
    window_case(R.bench4(kps, desc))

    for n, seed, nodes, dup in ((1500, 1, 40, False), (3000, 3, 3, False), (600, 4, 2, True)):
        p, v1, v2 = TM._bow_problem(n, seed, nodes, dup)
        mt = match.bow_tree(lowe_ratio=0.75 if dup else 0.6, check_orientation=True)
        record("bow_tree.match_keyframes/%d" % seed, mt, lambda: mt.match_keyframes(
            p["desc_1"], p["angle_1"], v1, p["bow_node_1"], p["desc_2"], p["angle_2"], v2, p["bow_node_2"]))
        record("bow_tree.match_frame_and_keyframe/%d" % seed, mt, lambda: mt.match_frame_and_keyframe(
            p["desc_1"], p["angle_1"], v1, p["bow_node_1"], p["desc_2"], p["angle_2"], p["bow_node_2"]))
        mt.close()

    # test_match_for_triangulation_tiny_nodes_exhaust_the_candidate_lists
    p = synth.triangulation_problem(500, 7, n_nodes=2)
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (3, 32), dtype=np.uint8)
    p["desc_1"] = base[rng.integers(0, 3, len(p["desc_1"]))]
    p["desc_2"] = base[rng.integers(0, 3, len(p["desc_2"]))]
    p["E_12"] = np.zeros((3, 3)); p["E_12"][2, 2] = 1.0
    for k, z in (("bearing_1", -0.5), ("bearing_2", 0.5)):
        b = p[k].copy(); b[:, 2] = z * np.linalg.norm(b[:, :2], axis=1); b /= np.linalg.norm(b, axis=1, keepdims=True); p[k] = b
    p["epipole_in_2"] = np.array([0.0, 0.0, -1.0])
    keys = ("desc_1", "bearing_1", "octave_1", "angle_1", "has_lm_1", "is_stereo_1", "bow_node_1",
            "desc_2", "bearing_2", "angle_2", "has_lm_2", "is_stereo_2", "bow_node_2", "E_12", "epipole_in_2")
    for orient in (False, True):
        mt = match.robust(check_orientation=orient)
        record("robust.match_for_triangulation/%d" % orient, mt, lambda: mt.match_for_triangulation(*[p[k] for k in keys], O.scale_factors(1.2, 8)))
        mt.close()

    for orient in (False, True):
        kf1, nbs, E, ep = TT._planar_neighbourhood(8, 600, 3)
        mt = match.robust(check_orientation=orient)
        record("create_new_landmarks/planar/%d" % orient, mt, lambda: module.create_new_landmarks(mt, kf1, nbs, E, ep, orient))
        mt.close()
    kf1, nbs, E, ep = TP.neighbourhood(9, 1500, 10, stereo_frac=0.3)
    mt = match.robust(check_orientation=True)
    record("create_new_landmarks/neighbourhood", mt, lambda: module.create_new_landmarks(mt, kf1, nbs, E, ep, True))
    mt.close()

    # test_robust_greedy_uniqueness_requery and test_brute_force_match_on_device_resident_descriptors
    rng = np.random.default_rng(9)
    base = TM._rand_desc(rng, 40)
    frm = np.concatenate([TM._noisy_copy(rng, base, 3) for _ in range(8)])
    kf = np.concatenate([TM._noisy_copy(rng, base, 2) for _ in range(12)])
    for ratio in (0.6, 0.9, 1.0):
        mt = match.robust(lowe_ratio=ratio)
        record("robust.brute_force_match/%g" % ratio, mt, lambda: mt.brute_force_match(frm, kf))
        mt.close()
    rng = np.random.default_rng(5)
    base = rng.integers(0, 256, (3000, 32), dtype=np.uint8)
    d1 = base.copy(); d2 = base[rng.permutation(3000)[:2500]].copy()
    d2 ^= (rng.integers(0, 256, d2.shape, dtype=np.uint8) & rng.integers(0, 256, d2.shape, dtype=np.uint8)
           & rng.integers(0, 256, d2.shape, dtype=np.uint8) & rng.integers(0, 256, d2.shape, dtype=np.uint8))
    valid = (rng.random(len(d2)) < 0.9).astype(np.uint8)
    t1 = torch.from_numpy(d1).cuda(); t2 = torch.from_numpy(d2).cuda()
    mt = match.robust(lowe_ratio=0.75)
    record("robust.brute_force_match_device", mt, lambda: mt.brute_force_match_device(t1.data_ptr(), len(d1), t2.data_ptr(), len(d2), valid))
    record("robust.brute_force_match_host", mt, lambda: mt.brute_force_match(d1, d2, valid))
    mt.close()

    print("package: %s" % os.path.dirname(openvslam_b200.__file__), file=sys.stderr)
    if args.out:
        with open(args.out, "w") as fh:
            fh.writelines(json.dumps(l) + "\n" for l in lines)


if __name__ == "__main__":
    main()
