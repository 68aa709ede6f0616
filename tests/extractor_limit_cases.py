"""Images and budgets that take the ORB extractor to its size-driven limits: the global-memory sorts of the tree distribution,
dense-corner images and the 12-bit candidate coordinates.  The GPU parity tests (test_extractor_limits_gpu.py) run them against
the oracle; the CPU tests (test_tree_device_model.py) check with the numpy tree model that every tree case reaches the branch it
is meant to cover."""
import numpy as np

from openvslam_b200 import synth

SORT_SMEM = 8192        # keys k_tree_distribute sorts in shared memory (kTreeSortSmem); a larger sort runs in global scratch


def noise(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def lattice(w, h, inverse=False):
    """0 / 255 image, bright where (x + 2 y) % 4 == 0 (dark there if `inverse`): nearly every fourth pixel is a FAST corner."""
    y, x = np.mgrid[0:h, 0:w]
    bright = (x + 2 * y) % 4 == 0
    return np.where(bright != inverse, 255, 0).astype(np.uint8)


def sparse(w, h, seed, density=0.05):
    """isolated bright pixels on black"""
    return np.where(np.random.default_rng(seed).random((h, w)) < density, 255, 0).astype(np.uint8)


# id -> (image, max_num_keypts, num_levels, levels whose largest-first pool is sorted in global memory,
#        levels whose final selection is sorted in global memory)
TREE_CASES = {
    # control: pool (2048) and selection (8000) both sorted in shared memory
    "noise1920-n8000": (lambda: noise(1920, 960, 1), 8000, 1, (), ()),
    # the pool exactly fills shared memory (8192 keys); the selection (9002) goes to global memory
    "noise1920-n9000": (lambda: noise(1920, 960, 1), 9000, 1, (), (0,)),
    "noise1920-n40000": (lambda: noise(1920, 960, 1), 40000, 1, (0,), (0,)),
    # a natural image: pool of 10716 nodes
    "synth3840-n20000": (lambda: synth.frame(3840, 1920, seed=3), 20000, 1, (0,), (0,)),
    # several CTAs sort their selections in global scratch at once (levels 0-2: 13031, 10859, 9050 keypoints)
    "noise3840-n60000-l8": (lambda: noise(3840, 1920, 4), 60000, 8, (), (0, 1, 2)),
    # two CTAs sort pools of 32768 nodes in global scratch at once
    "noise3840-n80000-l2": (lambda: noise(3840, 1920, 4), 80000, 2, (0, 1), (0, 1)),
}

# (width, height, max_num_keypts) of the dense-corner images: the sizes and budgets of BASELINE configs[1] and [3]
DENSE_SIZES = [(752, 480, 1000), (1920, 960, 4000)]
# id -> (image factory (w, h), extra orb_params)
DENSE_IMAGES = {
    "lattice": (lambda w, h: lattice(w, h), {}),
    "lattice-inverse": (lambda w, h: lattice(w, h, inverse=True), {}),
    "noise-thr20-7": (lambda w, h: noise(w, h, 5), {}),
    "noise-thr7-7": (lambda w, h: noise(w, h, 5), dict(ini_fast_thr=7, min_fast_thr=7)),
    "sparse": (lambda w, h: sparse(w, h, 6), {}),
}
