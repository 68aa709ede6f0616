"""The bundle adjusters against committed results of the CUDA path (tests/golden/ba_edge_record_golden.npz, made by
tests/golden/make_ba_edge_record_golden.py before the per-edge blocks were replaced by one compact record per edge): how the
normal equations' per-edge blocks are stored and where they are formed must not change a single bit of the result.  The graphs
cover 2-row and mixed 2- / 3-row problems, the equirectangular model, outliers leaving the graph between the rounds, and a
landmark with more than 128 edges (a linearisation block of its own, walked in passes)."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_ba_edge_record_golden", os.path.join(ROOT, "tests", "golden", "make_ba_edge_record_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.fixture(scope="module")
def vec():
    return np.load(os.path.join(ROOT, "tests", "golden", "ba_edge_record_golden.npz"))


@pytest.mark.parametrize("name", list(G.CASES))
def test_ba_matches_golden_bit_for_bit(vec, name):
    res = G.run_case(name)
    for key in ("poses", "points", "outliers", "num_iterations", "num_trials"):
        assert np.array_equal(res[key], vec[name + "/" + key]), key
