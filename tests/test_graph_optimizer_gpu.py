"""The pose-graph optimiser on the GPU (ovs_graph_optimize_host, optimize.graph_optimizer) against the CPU oracle
(oracle/graph_oracle.c), the numpy float64 step of tests/pose_graphs.py and the ground truth of the generated loops."""
import ctypes as C
import statistics
import subprocess

import numpy as np
import pytest

import pose_graphs as pg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G(oracle):
    from oracle import graph
    return graph


@pytest.fixture(scope="module")
def gopt():
    from openvslam_b200 import optimize
    return optimize


def _run(gopt, g, num_iter=50, S=None, lm=None, ref=None, opt=None):
    o = opt or gopt.graph_optimizer(g["fix_scale"], num_iter)
    out = o.optimize(g["start"] if S is None else S, g["fixed"], g["edge_i"], g["edge_j"], g["meas"], lm, ref)
    if opt is None:
        o.close()
    return out


def _step_err(a, b, x):
    return np.abs(a - b).max() / max(np.abs(x).max(), 1e-300)


@pytest.mark.parametrize("fix_scale", [False, True])
@pytest.mark.parametrize("nfree", [10, 98, 99, 150])
def test_converged_matches_oracle(gopt, G, nfree, fix_scale):
    g = pg.loop_graph(nfree, seed=nfree, fix_scale=fix_scale, num_landmarks=200)
    S, pose, lm, st = _run(gopt, g, lm=g["lm"], ref=g["lm_ref"])
    So, _, _, sto = G.graph_optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"], fix_scale, 50)
    print("nfree %d fix_scale %d: GPU %d iterations / %d trials, oracle %d / %d" % (nfree, fix_scale, st["num_iterations"], st["num_trials"],
                                                                                 sto["num_iterations"], sto["num_trials"]))
    # 1e-8 where the oracle's run ends by g2o's stop rule (ten rejected trials, or rho == 0) before the 50-iteration budget.
    # Exception: the fixed-scale graphs at 98 and 150 free vertices use the whole budget.  A fixed scale drops sigma from the
    # 7-wide step, and these runs descend slowly: between its iterations 49 and 50 the oracle still moves 3.3e-9 (98) and
    # 3.4e-5 (150), and chi2 falls a further 0.5 % (98) and 2.4 % (150) over the next 50 iterations.  The result is a snapshot
    # in mid-descent, so a trial decided differently at rounding level (98: 99 GPU trials against 98) moves it by more than
    # 1e-8; these two are compared within 1e-6.
    tol = 1e-8 if sto["num_iterations"] < 50 else 1e-6
    if sto["num_iterations"] >= 50:
        assert fix_scale and nfree in (98, 150), "an unexpected budget-limited run"
    assert np.abs(S - So).max() <= tol
    assert abs(st["final_chi2"] - sto["final_chi2"]) <= tol * sto["final_chi2"]
    assert st["lambda_init"] == [1e-16] and st["reduced_dim"] == 7 * nfree
    assert np.abs(pose - pg.pose_of(S)).max() <= 1e-12
    ref = pg.corrected_landmarks(g["start"], S, g["lm"], g["lm_ref"])
    assert np.abs(lm - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    keep = g["lm_ref"] < 0
    assert np.array_equal(lm[keep], g["lm"][keep])
    fixed = g["fixed"] == 1
    assert np.array_equal(S[fixed], g["start"][fixed])
    if fix_scale:
        assert np.array_equal(S[:, 12], g["start"][:, 12])


def _irregular(nfree, seed, fix_scale=False):
    """duplicate edges, i > j orientations, an edge between two fixed vertices, an isolated free vertex, a vertex tied only to
    fixed ones and interleaved fixed vertices"""
    g = pg.loop_graph(nfree, seed=seed, fix_scale=fix_scale, fixed_every=4, drift=(0.01, 0.02, 0.02))
    K = len(g["start"])
    rng = np.random.default_rng(seed)
    ei, ej, meas = list(g["edge_i"]), list(g["edge_j"]), list(g["meas"])
    # an isolated free vertex and one tied only to the fixed vertices 0 and 4
    iso = len(g["start"])
    lone = iso + 1
    true = np.vstack([g["true"], g["true"][1:3]])
    start = np.vstack([g["start"], g["start"][1:3]])
    fixed = np.append(g["fixed"], [0, 0]).astype(np.uint8)
    for (i, j) in [(lone, 0), (4, lone), (0, 4), (4, 0), (ei[0], ej[0]), (ej[1], ei[1])]:
        ei.append(i); ej.append(j)
        meas.append(pg.relative(true[j], true[i]))
    g.update(true=true, start=start, fixed=fixed, edge_i=np.array(ei, np.int32), edge_j=np.array(ej, np.int32), meas=np.array(meas))
    return g


def _one_step(gopt, G, g, with_oracle=True, first_trial=True):
    """num_iter = 1 against the oracle (equal trial counts, 1e-10 of the step) and, when the first trial is the accepted one,
    against the numpy step.  first_trial: the numpy step must lower chi2 (so g2o's rho test accepts it: its denominator is
    positive), and the device must then have taken exactly that one trial."""
    S, _, _, st = _run(gopt, g, num_iter=1)
    if first_trial:
        x, ref = pg.lm_first_step(g, g["start"])
        assert pg.chi2(g, ref) < pg.chi2(g, g["start"])
        assert st["num_trials"] == 1
        assert _step_err(S, ref, x) <= 1e-10
    else:
        x = S - g["start"]
    if with_oracle:
        So, _, _, sto = G.graph_optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"], g["fix_scale"], 1)
        assert st["num_trials"] == sto["num_trials"]
        assert _step_err(S, So, x) <= 1e-10
    return S, st


@pytest.mark.parametrize("nfree", [1, 2, 23, 97, 98, 99, 300, 857])   # 23, 97: odd 7 n_free on the cluster solver (padded row)
def test_one_step(gopt, G, nfree):
    g = pg.loop_graph(nfree, seed=nfree + 7, cov_step=(2, 3, 4))
    S, st = _one_step(gopt, G, g, with_oracle=nfree <= 300)
    assert st["reduced_dim"] == 7 * nfree and st["lambda_init"] == [1e-16]


@pytest.mark.parametrize("fix_scale", [False, True])
def test_one_step_irregular_graph(gopt, G, fix_scale):
    g = _irregular(20, 31, fix_scale)
    S, st = _one_step(gopt, G, g)
    iso = len(g["start"]) - 2
    assert np.array_equal(S[iso], g["start"][iso])         # the free vertex without an edge keeps its bits
    assert not np.array_equal(S[iso + 1], g["start"][iso + 1])
    nfree = int(((pg.free_index(len(S), g["fixed"], g["edge_i"], g["edge_j"])) >= 0).sum())
    assert st["reduced_dim"] == 7 * nfree


def test_first_iteration_with_more_than_four_rejected_trials(gopt, G):
    g = pg.loop_graph(12, seed=2, drift=(0.3, 0.5, 0.3), noise=0.05)
    S, st = _one_step(gopt, G, g, first_trial=False)
    assert st["num_trials"] > 4 and st["solver_trials"] >= st["num_trials"]


def test_noise_free_graph_converges_to_truth(gopt):
    g = pg.loop_graph(40, seed=9, noise=0.0, drift=(0.01, 0.02, 0.02))
    S, _, _, st = _run(gopt, g)
    assert np.abs(S - g["true"]).max() <= 1e-9, st


def test_drifted_monocular_loop_improves(gopt):
    g = pg.loop_graph(60, seed=10, drift=(0.003, 0.01, 0.02))
    S, _, _, _ = _run(gopt, g)
    before, after = pg.trajectory_error(g["start"], g["true"]), pg.trajectory_error(S, g["true"])
    print("trajectory error %.4g -> %.4g" % (before, after))
    assert after * 5 <= before


def test_interface_edges(gopt):
    from openvslam_b200 import _lib
    o = gopt.graph_optimizer(False)
    rc_bad = []
    h = o._h
    g = pg.loop_graph(10, seed=1)
    for mutate in ["range", "self", "scale", "meas_scale"]:
        S, ei, ej, meas = g["start"].copy(), g["edge_i"].copy(), g["edge_j"].copy(), g["meas"].copy()
        if mutate == "range": ej[0] = len(S)
        if mutate == "self": ej[0] = ei[0]
        if mutate == "scale": S[3, 12] = -1.0
        if mutate == "meas_scale": meas[2, 12] = np.inf
        fixed = np.ascontiguousarray(g["fixed"], np.uint8)
        ei = np.ascontiguousarray(ei, np.int32); ej = np.ascontiguousarray(ej, np.int32); meas = np.ascontiguousarray(meas)
        rc = _lib.lib().ovs_graph_optimize_host(h, len(S), S.ctypes.data_as(C.c_void_p), fixed.ctypes.data_as(C.c_void_p), len(ei),
                                                ei.ctypes.data_as(C.c_void_p), ej.ctypes.data_as(C.c_void_p), meas.ctypes.data_as(C.c_void_p),
                                                0, 50, 0, None, None, None, None)
        rc_bad.append(rc)
    assert rc_bad == [-1, -1, -1, -1]
    # 858 free vertices -> OVS_ERR_UNSUPPORTED
    g = pg.loop_graph(858, seed=1, cov_step=(2,))
    S = np.ascontiguousarray(g["start"]); fixed = np.ascontiguousarray(g["fixed"], np.uint8)
    ei = np.ascontiguousarray(g["edge_i"], np.int32); ej = np.ascontiguousarray(g["edge_j"], np.int32); meas = np.ascontiguousarray(g["meas"])
    rc = _lib.lib().ovs_graph_optimize_host(h, len(S), S.ctypes.data_as(C.c_void_p), fixed.ctypes.data_as(C.c_void_p), len(ei),
                                            ei.ctypes.data_as(C.c_void_p), ej.ctypes.data_as(C.c_void_p), meas.ctypes.data_as(C.c_void_p),
                                            0, 50, 0, None, None, None, None)
    assert rc == -6
    # E == 0: no Levenberg launch, the estimates come back unchanged
    g = pg.loop_graph(10, seed=1)
    before = _lib.launch_count()
    S, pose, _, st = o.optimize(g["start"], g["fixed"], np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 13)))
    assert _lib.launch_count() - before <= 1 and st["num_iterations"] == 0 and st["solver_launches"] == 0
    assert np.array_equal(S, g["start"])
    o.close()


def test_repeated_calls_bit_identical(gopt):
    g = pg.loop_graph(120, seed=12, num_landmarks=100)
    o = gopt.graph_optimizer(False)
    a = o.optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"], g["lm"], g["lm_ref"])
    b = o.optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"], g["lm"], g["lm_ref"])
    o.close()
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)
    assert a[3]["num_trials"] == b[3]["num_trials"] and a[3]["final_chi2"] == b[3]["final_chi2"]


def test_invalidates_prepared_local_ba(gopt):
    from openvslam_b200 import optimize, synth
    q = synth.ba_problem(6, 2, 300, model="perspective", seed=6)
    pre = optimize.prepared_local_ba(optimize.camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                     q["obs_xy"], None, q["inv_sigma_sq"])
    pre.run()
    g = pg.loop_graph(10, seed=1)
    graph = gopt.graph_optimizer.__new__(gopt.graph_optimizer)
    graph._h = pre._h; graph.fix_scale_ = False; graph.num_iter_ = 50
    graph.optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"])
    with pytest.raises(Exception):
        pre.run()
    graph._h = None
    pre.close()


def test_cpp_class_layer(tmp_path):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_graph_optimizer")
    from openvslam_b200 import build
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "test_graph_optimizer.cpp"),
                           "-o", exe, "-L", os.path.dirname(build.SO), "-lovs_b200", "-Wl,-rpath," + os.path.dirname(build.SO)])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    print(out.stdout)


def test_timing(gopt, G):
    import time
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception:
        pl = "unknown"
    print("\n%s, power limit %s" % (name, pl))
    for nfree in [50, 98, 99, 300, 857]:
        g = pg.loop_graph(nfree, seed=nfree, cov_step=(2, 3, 4, 5), extra_loops=3)
        o = gopt.graph_optimizer(False)
        ts = []
        for k in range(23):
            _, _, _, st = o.optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"])
            if k >= 3:
                ts.append(st["device_us"])
        o.close()
        oracle_us = "not measured"
        if nfree <= 300:       # the oracle's naive dense Cholesky takes minutes at 857
            t0 = time.perf_counter()
            G.graph_optimize(g["start"], g["fixed"], g["edge_i"], g["edge_j"], g["meas"], False, 50)
            oracle_us = "%.0f us" % ((time.perf_counter() - t0) * 1e6)
        print("nfree %4d edges %5d: device_us median %.0f (iterations %d, trials %d, solver launches %d); C oracle single thread %s" %
              (nfree, len(g["edge_i"]), statistics.median(ts), st["num_iterations"], st["num_trials"], st["solver_launches"], oracle_us), flush=True)


def test_statistics_when_nothing_is_optimised(gopt):
    """edges only between fixed vertices, and num_iter == 0: the estimates come back unchanged, one round of no iterations,
    final_chi2 = chi2 at the returned estimates"""
    g = pg.loop_graph(10, seed=4)
    want = pg.chi2(g, g["start"])
    for fixed, num_iter in [(np.ones(len(g["start"]), np.uint8), 50), (g["fixed"], 0)]:
        o = gopt.graph_optimizer(False, num_iter)
        S, _, _, st = o.optimize(g["start"], fixed, g["edge_i"], g["edge_j"], g["meas"])
        o.close()
        assert np.array_equal(S, g["start"])
        assert st["num_rounds"] == 1 and st["num_iterations"] == 0 and st["num_trials"] == 0 and st["solver_launches"] == 0
        assert abs(st["final_chi2"] - want) <= 1e-10 * want
