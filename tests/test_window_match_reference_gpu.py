"""The GPU windowed matchers (csrc/match_window.cu: k_window_topk + the sequential replays with re-queries) against the
numpy restatement in window_match_reference.py and the oracle, bit for bit in the match arrays and counts, on the named
cases: the benchmark's shapes (config 4 on a host-built index and on one built from the extractor's device output,
config 2), an offset grid, window and level edges, thresholds, ties, contention, the angle histogram and x_right."""
import numpy as np
import pytest

import window_match_reference as R

pytestmark = pytest.mark.gpu


def _grid(case):
    from openvslam_b200 import match
    return match.camera_grid(*case.frame.grid.args())


def _index(mt, case):
    from openvslam_b200 import match
    f = case.frame
    return match.frame_index(mt, f.x, f.y, f.octave, f.angle, f.x_right, f.desc, _grid(case))


def run_gpu(case, kind, kw, fi=None):
    """One call of the case on the GPU -> (result tuple, re-queries it issued).  With an index of its own the call counts
    the re-queries of its matcher; a given index (fi) belongs to another matcher, and the count is not read."""
    from openvslam_b200 import match
    if kind == "area":
        mt = match.area(lowe_ratio=kw.get("lowe_ratio", 0.9), check_orientation=kw.get("check_orientation", True))
    else:
        mt = match.projection(lowe_ratio=kw.get("lowe_ratio", 0.6), check_orientation=kw.get("check_orientation", True))
    own = fi is None
    if own:
        fi = _index(mt, case)
    before = mt.num_requeries()
    try:
        if kind == "landmarks":
            res = mt.match_frame_and_landmarks(fi, kw["scale_factors"], kw["reproj_xy"], kw["x_right_in_tracking"], kw["pred_level"], kw["lm_desc"],
                                               kw.get("lm_usable"), kw.get("kp_has_observed_lm"), kw.get("margin", 5.0))
        elif kind == "current_and_last":
            res = mt.match_current_and_last_frames(fi, kw["scale_factors"], kw["num_scale_levels"], kw["last_usable"], kw["reproj_xy"],
                                                   kw["reproj_x_right"], kw["last_level"], kw["last_angle"], kw["lm_desc"], kw.get("kp_has_observed_lm"),
                                                   kw.get("margin", 20.0), kw.get("assume_forward", False), kw.get("assume_backward", False))
        elif kind == "frame_and_keyframe":
            res = mt.match_frame_and_keyframe(fi, kw["scale_factors"], kw["reproj_xy"], kw["pred_level"], kw["keyfrm_angle"], kw["lm_desc"], kw["usable"],
                                              kw["kp_has_lm"], kw["margin"], kw["hamm_dist_thr"])
        elif kind == "sim3":
            res = mt.match_by_Sim3_transform(fi, kw["scale_factors"], kw["reproj_xy"], kw["pred_level"], kw["lm_desc"], kw["usable"],
                                             kw["kp_already_matched"], kw["margin"])
        elif kind == "best":
            res = mt.match_best(fi, kw["ref_xy"], kw["ref_x_right"], kw["margin"], kw["min_level"], kw["max_level"], kw["q_angle"], kw["q_desc"],
                                kw.get("usable"), kw.get("kp_unavailable"), kw.get("hamm_dist_thr", R.THR_HIGH))
        elif kind == "area":
            res = mt.match_in_consistent_area(fi, kw["octave_1"], kw["angle_1"], kw["desc_1"], kw["prev_matched_xy"], kw.get("margin", 100))
        elif kind == "topk":
            res = fi.window_topk(kw["ref_xy"], kw["margin"], kw["min_level"], kw["max_level"], kw["q_desc"])
        else:
            raise ValueError(kind)
        return res, mt.num_requeries() - before
    finally:
        if own:
            fi.close()
        mt.close()


def assert_same(case, i, kind, got, want):
    what = "%s call %d (%s)" % (case.name, i, kind)
    if kind == "topk":
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), what
    else:
        assert got[0] == want[0], (what, got[0], want[0])
        assert np.array_equal(got[1], want[1]), (what, np.flatnonzero(got[1] != want[1])[:10])
        if kind == "area":
            assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32)), what


def check_case(oracle, case, fi=None):
    """GPU == reference == oracle for every call (the oracle's equality with the reference is also a CPU test; repeated
    here so that a GPU run alone shows all three agree)."""
    requeries = []
    for i, (kind, kw) in enumerate(case.calls):
        want = R.run_reference(case, kind, kw)
        if kind == "angles":
            assert np.array_equal(R.run_oracle(oracle, case, kind, kw)[0], want[0])
            requeries.append(0)
            continue
        got, nrq = run_gpu(case, kind, kw, fi)
        assert_same(case, i, kind, got, want)
        if not (kind == "topk" and case.frame.x_right is not None):
            assert_same(case, i, kind, R.run_oracle(oracle, case, kind, kw), want)
        requeries.append(nrq)
    return requeries


@pytest.mark.parametrize("name", sorted(R.SYNTHETIC_CASES))
def test_gpu_matches_reference(oracle, name):
    case = R.SYNTHETIC_CASES[name]()
    requeries = check_case(oracle, case)
    if name == "contention":
        # every replay (match_frame_and_landmarks, match_best, area) reached its undecided branches and asked the GPU again
        kinds = [k for k, _ in case.calls]
        assert kinds == ["landmarks", "best", "area"] and all(r > 0 for r in requeries), requeries


def test_gpu_matches_reference_bench2(oracle):
    from openvslam_b200 import synth
    a = synth.frame(752, 480, seed=200)
    ka, da, _ = oracle.extract(a, oracle.params(1000))
    kb, db, _ = oracle.extract(synth.shifted(a, 3, 0), oracle.params(1000))
    check_case(oracle, R.bench2(ka, da, kb, db))


def test_gpu_matches_reference_bench4_host_and_device_index(oracle):
    """Config 4: the keypoints of extract_device, indexed once from host arrays and once by frame_index.from_device."""
    import torch
    from openvslam_b200 import feature, match, synth
    W, H = 1920, 960
    img = synth.frame(W, H, seed=400)
    ext = feature.orb_extractor(feature.orb_params(max_num_keypts=4000))
    dev = torch.device("cuda", 0)
    d_img = torch.from_numpy(img).to(dev)
    cap = ext._cap
    d_kps = torch.zeros((cap, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((cap, 32), dtype=torch.uint8, device=dev)
    n = ext.extract_device(d_img.data_ptr(), W, H, W, d_kps.data_ptr(), d_desc.data_ptr(), cap)
    kps, desc = ext.extract(img)
    assert n == len(kps) and n >= 3900
    assert np.array_equal(d_desc[:n].cpu().numpy(), desc)
    case = R.bench4(kps, desc)
    check_case(oracle, case)
    mt = match.projection()
    fd = match.frame_index.from_device(mt, n, d_kps.data_ptr(), d_desc.data_ptr(), _grid(case))
    try:
        check_case(oracle, case, fd)
    finally:
        fd.close(); mt.close(); ext.close()
