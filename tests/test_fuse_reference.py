"""The fuse oracle (oracle/fuse_oracle.c, one call per target) against the numpy reference of tests/fuse_reference.py, bit for bit,
on every named case and on the seeded scenes of fuse_problems; the reference's window against a grid-free scan; every case
reaching the edges it is named for.  CPU only."""
import numpy as np
import pytest

from oracle import fuse as OF
from oracle import oracle as O
import fuse_problems as FP
import fuse_reference as R
import window_match_reference as WR

case = R.case_and_reference


def oracle_frame(t):
    f, g = t.frame, t.frame.grid
    return O.MatchFrame(f.x, f.y, f.octave, f.angle, f.x_right, f.desc, O.om_grid(*g.bounds, g.cols, g.rows))


def run_oracle(c):
    Q = int(c.q_off[-1])
    best = np.full(Q, -1, np.int32); ok = np.zeros(Q, bool); uv = np.zeros((Q, 2), np.float32); xr = np.zeros(Q, np.float32)
    lv = np.zeros(Q, np.int32)
    num = 0
    for k, t in enumerate(c.targets):
        s = slice(c.q_off[k], c.q_off[k + 1])
        n, best[s], ok[s], uv[s], xr[s], lv[s] = OF.replace_duplication(t.geometry, oracle_frame(t), t.scale_factors, t.inv_level_sigma_sq,
                                                                        c.q_lm[s], c.lms["pos_w"], c.lms["mean_normal"], c.lms["min_valid_dist"],
                                                                        c.lms["max_valid_dist"], c.lms["lm_desc"], c.margin)
        num += n
    return num, best, ok, uv, xr, lv


def same(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("name", sorted(R.CASES))
def test_oracle_equals_reference(name):
    c, ref = case(name)
    got = run_oracle(c)
    assert got[0] == ref[0]
    for label, a, b in zip(("best_idx", "passed", "reproj_xy", "x_right", "pred_level"), got[1:], ref[1:6]):
        assert same(a, b), label


@pytest.mark.parametrize("name", sorted(R.CASES))
def test_case_reaches_its_edges(name):
    c, ref = case(name)
    st = ref[6]
    missing = {k: (st[k], v) for k, v in c.expect.items() if st[k] < v}
    assert not missing, missing


@pytest.mark.parametrize("scene", sorted(FP.CAMERAS))
def test_oracle_equals_reference_on_fuse_problems(scene):
    targets, arrays, lms, q_off, q_lm = FP.batch(scene, 4, 2000, 1200, [600, 0, 500, 700], seed=61, skip_frac=0.1, empty=(2,))
    total = 0
    for k, a in enumerate(arrays):
        s = slice(q_off[k], q_off[k + 1])
        g = a["geometry"]
        grid = WR.Grid(g.min_x, g.max_x, g.min_y, g.max_y)
        t = R.Target(g, FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, a["x"], a["y"], a["octave"], a["desc"], grid, a["x_right"])
        ref = R.replace_duplication(t, lms, q_lm[s])
        got = OF.replace_duplication(g, oracle_frame(t), FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, q_lm[s], lms["pos_w"], lms["mean_normal"],
                                     lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"])
        assert got[0] == ref[0]
        for label, x, y in zip(("best_idx", "passed", "reproj_xy", "x_right", "pred_level"), got[1:], ref[1:6]):
            assert same(x, y), (k, label)
        total += ref[0]
    assert total > 100


def scan(t, ref_xy, level, margin):
    """get_keypoints_in_cell without the grid: every keypoint in a cell, inside the box and the level range, by index."""
    f = t.frame
    m = np.float32(np.float32(margin) * t.scale_factors[level])
    dx = np.abs(f.x - np.float32(ref_xy[0])); dy = np.abs(f.y - np.float32(ref_xy[1]))
    ok = f.in_grid & (dx < m) & (dy < m) & (f.octave <= level) & (f.octave >= level - 1)
    return np.flatnonzero(ok)


@pytest.mark.parametrize("name", ["chi2_edges", "x_right", "levels", "box_and_cells", "hamming_and_ties"])
def test_window_equals_grid_free_scan(name):
    c, ref = case(name)
    assert c.small
    _, best, ok, uv, xr, lv, _ = ref
    checked = 0
    for k, t in enumerate(c.targets):
        f = t.frame
        for q in range(c.q_off[k], c.q_off[k + 1]):
            if not ok[q]:
                continue
            m = np.float32(np.float32(c.margin) * t.scale_factors[lv[q]])
            ranks = WR.window(f, uv[q, 0], uv[q, 1], m, lv[q] - 1, lv[q])
            assert sorted(f.rank_to_idx[ranks].tolist()) == scan(t, uv[q], lv[q], c.margin).tolist(), (k, q)
            checked += 1
    assert checked >= 40
