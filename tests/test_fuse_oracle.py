"""The geometry of match::fuse::replace_duplication in the oracle (oracle/fuse_oracle.c: ott_fuse_observe) against a numpy
restatement, bit for bit, on seeded scenes and at the knife edges of its gates; and the oracle's batched loop against that geometry
fed to the fuse matching core of the match oracle.  CPU only."""
import numpy as np
import pytest

from oracle import fuse as OF
from oracle import oracle as O
import fuse_problems as FP
from fuse_reference import fuse_observe_reference
import tracking_problems as TP
import tracking_reference as REF


def _same_bits(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _check(s):
    args = (s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"])
    ok, uv64, xr, lv = OF.fuse_observe(*args)
    got = (ok, np.where(ok[:, None], uv64.astype(np.float32), np.float32(0)).astype(np.float32), xr, lv)
    ref = fuse_observe_reference(*args)
    for name, a, b in zip(("passed", "reproj_xy", "x_right", "pred_level"), got, ref):
        assert _same_bits(a, b), name
    return got


@pytest.mark.parametrize("name", TP.SCENES)
def test_fuse_observe_scenes(name):
    s = TP.scene(name, 3000, seed=23)
    ok, uv, xr, lv = _check(s)
    assert 0 < ok.sum() < len(ok)
    assert len(np.unique(lv[ok])) >= 3


@pytest.mark.parametrize("equirectangular", [False, True])
def test_fuse_observe_knife_edges(equirectangular):
    s = FP.knife_edges(equirectangular)
    ok, uv, xr, lv = _check(s)
    P = s["pos_w"]
    # the non-finite positions are rejected, whatever the gates say
    assert not ok[~np.isfinite(P).all(1)].any()
    if not equirectangular:
        # the fuse gates' own edges (appended last): on each bound passes, one double ulp outside fails
        n_extra = 4 * 2 * 3 + 4
        dist_ok = ok[-n_extra:-4].reshape(4, 2, 3)
        assert dist_ok[:, 0, :].tolist() == [[False, True, True]] * 4     # 0.7 min: below fails, on and above pass
        assert dist_ok[:, 1, :].tolist() == [[True, True, False]] * 4     # 1.3 max: on and below pass, above fails
        assert ok[-4:].tolist() == [True, False, True, False]               # v . n == 0.5 dist passes, just below fails


def test_fuse_observe_differs_from_can_observe():
    """The fuse gates compare the double distance with the float bounds; can_observe compares the float distance: a landmark one
    double ulp beyond (double)(float)(1.3 max) passes can_observe and fails fuse_observe."""
    s = FP.knife_edges(False)
    ok_f = _check(s)[0]
    ok_c = REF.can_observe(s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5)[0]
    assert (ok_c & ~ok_f).any()


@pytest.mark.parametrize("scene", sorted(FP.CAMERAS))
def test_oracle_loop_is_geometry_then_core(scene):
    targets, arrays, lms, q_off, q_lm = FP.batch(scene, 2, 3000, 1500, [2500, 2500], seed=4, skip_frac=0.1)
    total = 0
    for t, a in enumerate(arrays):
        ql = q_lm[q_off[t]:q_off[t + 1]]
        frame = O.MatchFrame(a["x"], a["y"], a["octave"], np.zeros(len(a["x"]), np.float32), a["x_right"], a["desc"],
                             O.om_grid(*(a["geometry"].min_x, a["geometry"].max_x, a["geometry"].min_y, a["geometry"].max_y)))
        num, best, ok, uv, xr, lv = OF.replace_duplication(a["geometry"], frame, FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, ql, lms["pos_w"],
                                                           lms["mean_normal"], lms["min_valid_dist"], lms["max_valid_dist"], lms["lm_desc"])
        rows = np.maximum(ql, 0)
        ok2, uv2, xr2, lv2 = fuse_observe_reference(a["geometry"], lms["pos_w"][rows], lms["mean_normal"][rows], lms["min_valid_dist"][rows],
                                                    lms["max_valid_dist"][rows])
        ok2 &= ql >= 0
        assert np.array_equal(ok, ok2) and np.array_equal(lv, np.where(ok2, lv2, 0))
        n2, best2 = O.fuse_best_keypoints(frame, uv, xr, lv, lms["lm_desc"][rows], FP.SCALE_FACTORS, FP.INV_LEVEL_SIGMA_SQ, 3.0,
                                          usable=ok.astype(np.uint8))
        assert num == n2 and np.array_equal(best, best2)
        total += num
    assert total > 100
