#!/usr/bin/env python
"""One hot-path step (extract, brute-force match, pose optimiser, local BA) to run under a profiler (e.g. torch.profiler).
usage: python tools/profile_step.py [ba|extract|match|pose|all] [repeat]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openvslam_b200 import feature, match, optimize, synth  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "all"
rep = int(sys.argv[2]) if len(sys.argv) > 2 else 1
if what in ("extract", "match", "all"):
    a = synth.frame(1920, 960, seed=1); b = synth.shifted(a, 3, 1)
    ext = feature.orb_extractor(feature.orb_params(max_num_keypts=4000))
    for _ in range(rep + 1):
        ka, da = ext.extract(a)
    kb, db = ext.extract(b)
    if what in ("match", "all"):
        mt = match.robust(lowe_ratio=0.75)
        for _ in range(rep):
            mt.brute_force_match(da, db)
if what in ("pose", "all"):
    p = synth.pose_problem(4000, model="equirectangular", seed=3, stereo=False)
    po = optimize.pose_optimizer()
    for _ in range(rep):
        po.optimize(optimize.camera(**p["cam"]), True, p["pts_w"], p["obs_xy"], None, p["inv_sigma_sq"], p["poses"][0])
if what in ("ba", "all"):
    q = synth.ba_problem(50, 10, 20000, model="equirectangular", seed=4)
    ba = optimize.prepared_local_ba(optimize.camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                    q["obs_xy"], None, q["inv_sigma_sq"])
    for _ in range(rep):
        st = ba.run()
        poses, points, outl = ba.fetch()
        print('run: trials', st['num_trials'], 'last_chi2', st['last_chi2'], 'chi2 of fetched state (inliers)',
              synth.reprojection_chi2(q['cam'], poses, points, q['obs_kf'], q['obs_lm'], q['obs_xy'], None, q['inv_sigma_sq'], ~outl), 'outliers', int(outl.sum()))
    print(st)
