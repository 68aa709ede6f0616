"""The array-pass formulation of distribute_keypoints_via_tree that k_tree_distribute implements (tests/tree_device_model.py:
serial numbers instead of list links, speculative child counts + prefix search in the largest-first phase, one sort at the
end) against the oracle's list-based tree, on the CPU.  The kernel itself is checked on the GPU (tests/test_extractor_gpu.py)."""
import numpy as np
import pytest

from openvslam_b200 import synth

import extractor_limit_cases as lc
import tree_device_model as tm


@pytest.mark.parametrize("w,h,seed", [(800, 500, 5), (300, 600, 6), (333, 333, 7), (1000, 112, 8), (1241, 376, 9)])
def test_model_equals_oracle_tree(oracle, w, h, seed):
    img = synth.frame(w, h, seed=seed)
    cands = oracle.fast_detect(np.ascontiguousarray(img[19:-19, 19:-19]), 20)
    for N in (1, 2, 7, 50, 217, 869, 2500, 10 ** 6):
        ref = oracle.distribute_via_tree(cands, 19, w - 19, 19, h - 19, N)
        got = tm.distribute(cands["x"], cands["y"], cands["score"], 19, w - 19, 19, h - 19, N)
        assert len(got) == len(ref) and np.array_equal(got, ref), (w, h, N)


def test_model_ties_and_clusters(oracle):
    rng = np.random.default_rng(3)
    n = 3000
    xy = rng.choice(600 * 400, n, replace=False)
    cands = np.zeros(n, oracle.FASTPT_DTYPE)
    cands["x"] = xy % 600; cands["y"] = xy // 600; cands["score"] = rng.integers(20, 23, n)
    cands = cands[np.lexsort((cands["x"], cands["y"]))]
    for N in (10, 100, 400, 1000):
        ref = oracle.distribute_via_tree(cands, 19, 619, 19, 419, N)
        got = tm.distribute(cands["x"], cands["y"], cands["score"], 19, 619, 19, 419, N)
        assert np.array_equal(got, ref)
    # a dense cluster: chains of splits with a single non-empty child
    xs, ys = np.meshgrid(np.arange(300, 340, 2), np.arange(200, 240, 2))
    cl = np.zeros(xs.size + 5, oracle.FASTPT_DTYPE)
    cl["x"][:xs.size] = xs.ravel(); cl["y"][:xs.size] = ys.ravel()
    cl["x"][xs.size:] = [5, 580, 10, 570, 299]; cl["y"][xs.size:] = [5, 5, 390, 390, 100]
    cl["score"] = rng.integers(20, 200, len(cl))
    cl = cl[np.lexsort((cl["x"], cl["y"]))]
    for N in (3, 8, 30, 200, 1000):
        ref = oracle.distribute_via_tree(cl, 19, 619, 19, 419, N)
        got = tm.distribute(cl["x"], cl["y"], cl["score"], 19, 619, 19, 419, N)
        assert np.array_equal(got, ref), N


@pytest.mark.parametrize("case", list(lc.TREE_CASES))
def test_limit_cases_reach_their_sort_branch(oracle, case):
    """Each tree case of the GPU limit tests reaches the sort branch it is there for: the kernel sorts the largest-first pool and
    the final selection in shared memory up to SORT_SMEM keys and in global scratch beyond.  The model also equals the oracle's
    list-based tree at these sizes."""
    make, n, levels, pool_global, fin_global = lc.TREE_CASES[case]
    img = make()
    P = oracle.params(n, num_levels=levels)
    pyr = oracle.build_pyramid(img, P)
    sf = oracle.scale_factors(1.2, levels)
    target = oracle.keypts_per_level(n, 1.2, levels)
    stats = []
    for l in range(levels):
        h, w = pyr[l].shape
        c = oracle.level_candidates(P, pyr[l], float(sf[l]))
        st = {}
        got = tm.distribute(c["x"], c["y"], c["score"], 19, w - 19, 19, h - 19, int(target[l]), stats=st)
        assert np.array_equal(got, oracle.distribute_via_tree(c, 19, w - 19, 19, h - 19, int(target[l]))), (case, l)
        assert st["nfin"] == len(got)
        stats.append(st)
    assert stats[0]["pool_m"] > 0, stats                    # the largest-first phase is reached
    assert tuple(l for l, st in enumerate(stats) if st["pool_m"] > lc.SORT_SMEM) == pool_global, stats
    assert tuple(l for l, st in enumerate(stats) if st["nfin"] > lc.SORT_SMEM) == fin_global, stats
    if case == "noise1920-n9000":
        assert stats[0]["pool_m"] == lc.SORT_SMEM          # the largest pool that still sorts in shared memory
