#!/usr/bin/env python
"""One hot-path step (extract, brute-force match, pose optimiser, local BA) to run under a profiler (e.g. torch.profiler).
usage: python tools/profile_step.py [ba|extract|match|pose|all] [repeat]"""
import os, sys
import numpy as np
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
    print('cholesky cluster width', ba.cluster_width())
    clk = ba.debug_clocks()
    import numpy as np
    c = clk[:50].reshape(10, 5)
    print('cholesky phase cycles per block step [panel load, panel solve, look-ahead (warp 0), barrier] and step totals:')
    for b in range(10):
        if c[b, 0] == 0: break
        print(b, [int(c[b, k + 1] - c[b, k]) for k in range(4) if c[b, k + 1] > 0], int((c[b + 1, 0] if b < 9 and c[b + 1, 0] > 0 else clk[95]) - c[b, 0]))
    print('total cycles', int(clk[95] - clk[0]))
    print('look-ahead detail per step [tile update, factor loop]:', [(int(clk[168 + 2 * b] - c[b, 2]), int(clk[169 + 2 * b] - clk[168 + 2 * b])) for b in range(10) if clk[168 + 2 * b] > 0])
    print('back-substitution: start->first block ready', int(clk[96] - clk[94]), 'per block [matvec, update, wait next]:',
          [(int(clk[97 + 3 * j] - clk[96 + 3 * j]), int(clk[98 + 3 * j] - clk[97 + 3 * j]), int(clk[99 + 3 * j] - clk[98 + 3 * j]) if clk[99 + 3 * j] > 0 and j < 9 else 0) for j in range(10) if clk[96 + 3 * j] > 0])
    for b in range(9):
        q = clk[50 + 4 * b: 54 + 4 * b]
        if q[0] == 0: break
        print('tile0 of step', b, 'since panel solved', int(q[0] - c[b, 2]), 'loads', int(q[1] - q[0]), 'kloop', int(q[2] - q[1]), 'stores', int(q[3] - q[2]))
