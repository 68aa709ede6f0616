"""solve._batch, the batching every RANSAC solver class passes to the C ABI: what it hands over by pointer is contiguous."""
import numpy as np
import pytest


@pytest.mark.parametrize("take", [slice(None, None, 2), slice(None, None, -2), slice(1, None, 2)])
def test_seeds_views_are_passed_by_value_as_contiguous_arrays(take):
    from openvslam_b200.solve import _batch
    seeds = np.arange(100, 106, dtype=np.uint64)[take]
    t = _batch("solver", 3, seeds, {"x": ([np.zeros((2, 3))] * 3, (3,), np.float64)}, 9)
    assert t.seeds.flags.c_contiguous and t.seeds.dtype == np.uint64 and np.array_equal(t.seeds, seeds)
    assert all(a.flags.c_contiguous for a in [*t.off.values(), *t.cat.values()])
    assert np.array_equal(t.off["x"], [0, 2, 4, 6]) and t.cat["x"].shape == (6, 3)
