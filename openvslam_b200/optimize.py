"""Host-side mirror of openvslam::optimize::{pose_optimizer, local_bundle_adjuster, global_bundle_adjuster,
transform_optimizer} (src/openvslam/optimize/*.h; names as in SURVEY.md 8a)
over the C ABI of libovs_b200.so.  The reference classes take data::frame / data::keyframe; here the
same quantities are passed as flat arrays (see include/ovs_b200.h for the field-by-field mapping)."""
import ctypes as C
import numpy as np

from . import _lib

CAMERA_PERSPECTIVE, CAMERA_EQUIRECTANGULAR, CAMERA_FISHEYE, CAMERA_RADIAL_DIVISION = 0, 1, 2, 3
_MODEL_ID = {"perspective": 0, "equirectangular": 1, "fisheye": 2, "radial_division": 3}


class Camera(C.Structure):
    _fields_ = [("model", C.c_int32), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("cols", C.c_double), ("rows", C.c_double)]


class BaStats(C.Structure):
    _fields_ = [("num_rounds", C.c_int32), ("num_iterations", C.c_int32), ("num_trials", C.c_int32),
                ("round_iterations", C.c_int32 * 8), ("lambda_init", C.c_double * 8),
                ("last_lambda", C.c_double), ("last_chi2", C.c_double), ("final_chi2", C.c_double), ("device_us", C.c_float),
                ("solver_us", C.c_float), ("solver_launches", C.c_int32), ("solver_trials", C.c_int32), ("reduced_dim", C.c_int32),
                ("schur_us", C.c_float), ("co_observations", C.c_int32)]


def camera(model="perspective", fx=0.0, fy=0.0, cx=0.0, cy=0.0, focal_x_baseline=0.0, cols=0.0, rows=0.0):
    """model: "perspective" | "equirectangular"; "fisheye" / "radial_division" for feature.undistort_keypoints only (the
    matchers and optimisers work on the undistorted keypoints with the perspective model, as the reference)."""
    return Camera(_MODEL_ID[model], fx, fy, cx, cy, focal_x_baseline, cols, rows)


def _stats(st):
    return dict(num_rounds=st.num_rounds, num_iterations=st.num_iterations, num_trials=st.num_trials,
                round_iterations=list(st.round_iterations)[:st.num_rounds], lambda_init=list(st.lambda_init)[:st.num_rounds],
                last_lambda=st.last_lambda, last_chi2=st.last_chi2, final_chi2=st.final_chi2, device_us=st.device_us,
                solver_us=st.solver_us, solver_launches=st.solver_launches, solver_trials=st.solver_trials, reduced_dim=st.reduced_dim,
                schur_us=st.schur_us, co_observations=st.co_observations)


def _p(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a, a.ctypes.data_as(C.c_void_p)


class _optimizer_handle:
    def __init__(self, device=0):
        self._h = C.c_void_p()
        _lib.check(_lib.lib().ovs_optimizer_create(int(device), C.byref(self._h)))

    def set_speculation(self, width):
        """local BA: LM trials evaluated per launch sequence (1..4); same result for every width."""
        _lib.check(_lib.lib().ovs_optimizer_set_speculation(self._h, int(width)))

    def set_second_batch(self, width):
        """local BA: a second trial batch of `width` damping values enqueued statically behind the first (0 = off); same result."""
        _lib.check(_lib.lib().ovs_optimizer_set_second_batch(self._h, int(width)))

    def set_graphs(self, enable=True):
        """local BA: replay the (static) launch sequence of an LM iteration as one CUDA graph per iteration."""
        _lib.check(_lib.lib().ovs_optimizer_set_graphs(self._h, 1 if enable else 0))

    def set_cluster_width(self, width):
        """local / global BA: CTAs per cluster of the reduced-system solver (1, 2, 4, 8): 8 = lowest latency, 2 = most calls per
        second when several optimisers share the GPU.  Same results."""
        _lib.check(_lib.lib().ovs_optimizer_set_cluster_width(self._h, int(width)))

    def set_host_sync(self, mode=-1):
        """local BA: 1 = the host reads the device's Levenberg decision after every trial batch (skips unneeded launches),
        0 = never synchronise, -1 = automatic.  Same results."""
        _lib.check(_lib.lib().ovs_optimizer_set_host_sync(self._h, int(mode)))

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib().ovs_optimizer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class pose_optimizer(_optimizer_handle):
    """openvslam::optimize::pose_optimizer(num_trials = 4, num_each_iter = 10)."""

    def __init__(self, num_trials=4, num_each_iter=10, device=0):
        super().__init__(device)
        self.num_trials_ = int(num_trials)
        self.num_each_iter_ = int(num_each_iter)

    def optimize(self, cam, setup_is_mono, pts_w, obs_xy, obs_x_right, inv_sigma_sq, pose_cw):
        """-> (num_inliers, pose_cw[12], outlier_flags[n], stats)."""
        pts_w, pp = _p(pts_w, np.float64); obs_xy, po = _p(obs_xy, np.float32); inv_sigma_sq, pi = _p(inv_sigma_sq, np.float32)
        n = len(inv_sigma_sq)
        px = None
        if obs_x_right is not None:
            obs_x_right, px = _p(obs_x_right, np.float32)
        pose = np.array(pose_cw, np.float64).reshape(12).copy()
        flags = np.zeros(max(n, 1), np.uint8)
        ninl = C.c_int(0); st = BaStats()
        _lib.check(_lib.lib().ovs_pose_optimize_host(self._h, C.byref(cam), int(setup_is_mono), n, pp, po, px, pi,
                                                     pose.ctypes.data_as(C.c_void_p), flags.ctypes.data_as(C.c_void_p),
                                                     self.num_trials_, self.num_each_iter_, C.byref(ninl), C.byref(st)))
        return ninl.value, pose, flags[:n].astype(bool), _stats(st)


class local_bundle_adjuster(_optimizer_handle):
    """openvslam::optimize::local_bundle_adjuster(num_first_iter = 5, num_second_iter = 10)."""

    def __init__(self, num_first_iter=5, num_second_iter=10, device=0):
        super().__init__(device)
        self.num_first_iter_ = int(num_first_iter)
        self.num_second_iter_ = int(num_second_iter)

    def optimize(self, cam, setup_is_mono, poses, fixed, points, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq,
                 force_stop_flag=None):
        """-> (poses[K,12], points[L,3], outlier[M], stats)."""
        poses = np.array(poses, np.float64).reshape(-1, 12).copy(); points = np.array(points, np.float64).reshape(-1, 3).copy()
        fixed, pf = _p(fixed, np.uint8); obs_kf, pk = _p(obs_kf, np.int32); obs_lm, pl = _p(obs_lm, np.int32)
        obs_xy, po = _p(obs_xy, np.float32); inv_sigma_sq, pi = _p(inv_sigma_sq, np.float32)
        px = None
        if obs_x_right is not None:
            obs_x_right, px = _p(obs_x_right, np.float32)
        M = len(obs_kf)
        out = np.zeros(max(M, 1), np.uint8)
        st = BaStats()
        fs = None
        if force_stop_flag is not None:
            fs = C.c_uint8(int(bool(force_stop_flag)))
        _lib.check(_lib.lib().ovs_local_ba_host(self._h, C.byref(cam), int(setup_is_mono), len(poses), poses.ctypes.data_as(C.c_void_p), pf,
                                                len(points), points.ctypes.data_as(C.c_void_p), M, pk, pl, po, px, pi,
                                                self.num_first_iter_, self.num_second_iter_, C.byref(fs) if fs is not None else None,
                                                out.ctypes.data_as(C.c_void_p), C.byref(st)))
        return poses, points, out[:M].astype(bool), _stats(st)


class global_bundle_adjuster(_optimizer_handle):
    """openvslam::optimize::global_bundle_adjuster(map_db, num_iter = 10, use_huber_kernel = true)."""

    def __init__(self, num_iter=10, use_huber_kernel=True, device=0):
        super().__init__(device)
        self.num_iter_ = int(num_iter)
        self.use_huber_kernel_ = bool(use_huber_kernel)

    def optimize(self, cam, setup_is_mono, poses, fixed, points, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq, force_stop_flag=None):
        """-> (poses[K,12], points[L,3], stats)."""
        poses = np.array(poses, np.float64).reshape(-1, 12).copy(); points = np.array(points, np.float64).reshape(-1, 3).copy()
        fixed, pf = _p(fixed, np.uint8); obs_kf, pk = _p(obs_kf, np.int32); obs_lm, pl = _p(obs_lm, np.int32)
        obs_xy, po = _p(obs_xy, np.float32); inv_sigma_sq, pi = _p(inv_sigma_sq, np.float32)
        px = None
        if obs_x_right is not None:
            obs_x_right, px = _p(obs_x_right, np.float32)
        st = BaStats()
        fs = C.c_uint8(int(bool(force_stop_flag))) if force_stop_flag is not None else None
        _lib.check(_lib.lib().ovs_global_ba_host(self._h, C.byref(cam), int(setup_is_mono), len(poses), poses.ctypes.data_as(C.c_void_p), pf,
                                                 len(points), points.ctypes.data_as(C.c_void_p), len(obs_kf), pk, pl, po, px, pi, self.num_iter_,
                                                 int(self.use_huber_kernel_), C.byref(fs) if fs is not None else None, C.byref(st)))
        return poses, points, _stats(st)


class transform_optimizer(_optimizer_handle):
    """openvslam::optimize::transform_optimizer(fix_scale, num_iter = 10): the Sim3 refinement of a loop candidate.
    num_first_iter is the first round's iteration count (the reference's 5)."""

    def __init__(self, fix_scale, num_iter=10, num_first_iter=5, device=0):
        super().__init__(device)
        self.fix_scale_ = bool(fix_scale)
        self.num_iter_ = int(num_iter)
        self.num_first_iter_ = int(num_first_iter)

    def optimize(self, cam_1, cam_2, pose_1w, pose_2w, pos_w_1, obs_xy_1, inv_sigma_sq_1, pos_w_2, obs_xy_2, inv_sigma_sq_2, sim3_12,
                 chi_sq=10.0):
        """One row per correspondence (see include/ovs_b200.h); sim3_12 = {R row-major (9), t (3), s}.
        -> (num_inliers, sim3_12[13] (the input when num_inliers == 0), inlier_flags[n], stats)."""
        p1 = np.array(pose_1w, np.float64).reshape(12); p2 = np.array(pose_2w, np.float64).reshape(12)
        w1, pw1 = _p(np.asarray(pos_w_1).reshape(-1, 3), np.float64); x1, px1 = _p(obs_xy_1, np.float32); s1, ps1 = _p(inv_sigma_sq_1, np.float32)
        w2, pw2 = _p(np.asarray(pos_w_2).reshape(-1, 3), np.float64); x2, px2 = _p(obs_xy_2, np.float32); s2, ps2 = _p(inv_sigma_sq_2, np.float32)
        n = len(s1)
        if not (len(w1) == len(w2) == len(s2) == n and x1.size == x2.size == 2 * n):
            raise ValueError("transform_optimizer: every per-pair array needs n rows")
        S = np.array(sim3_12, np.float64).reshape(13).copy()
        flags = np.zeros(max(n, 1), np.uint8)
        ninl = C.c_int(0); st = BaStats()
        _lib.check(_lib.lib().ovs_transform_optimize_host(self._h, C.byref(cam_1), C.byref(cam_2), p1.ctypes.data_as(C.c_void_p),
                                                          p2.ctypes.data_as(C.c_void_p), n, pw1, px1, ps1, pw2, px2, ps2,
                                                          int(self.fix_scale_), C.c_float(chi_sq), self.num_first_iter_, self.num_iter_,
                                                          S.ctypes.data_as(C.c_void_p), flags.ctypes.data_as(C.c_void_p), C.byref(ninl),
                                                          C.byref(st)))
        return ninl.value, S, flags[:n].astype(bool), _stats(st)


class graph_optimizer(_optimizer_handle):
    """openvslam::optimize::graph_optimizer(fix_scale, num_iter = 50): the loop-closure pose graph over Sim3 vertices."""

    def __init__(self, fix_scale, num_iter=50, device=0):
        super().__init__(device)
        self.fix_scale_ = bool(fix_scale)
        self.num_iter_ = int(num_iter)

    def optimize(self, sim3_cw, fixed, edge_i, edge_j, meas_ji, lm_pos_w=None, lm_ref=None):
        """sim3_cw[K, 13] = S_iw {R row-major (9), t (3), s}; edges (i, j) with measurements S_ji[E, 13]; landmarks corrected through
        their reference vertex lm_ref (-1: unchanged).  See include/ovs_b200.h.
        -> (sim3_cw[K, 13], pose_cw[K, 12], lm_pos_w[L, 3], stats)."""
        S = np.array(sim3_cw, np.float64).reshape(-1, 13).copy()
        K = len(S)
        fixed, pf = _p(np.asarray(fixed).reshape(-1), np.uint8)
        ei, pi = _p(np.asarray(edge_i).reshape(-1), np.int32); ej, pj = _p(np.asarray(edge_j).reshape(-1), np.int32)
        meas, pm = _p(np.asarray(meas_ji, np.float64).reshape(-1, 13), np.float64)
        E = len(ei)
        if not (len(fixed) == K and len(ej) == E and len(meas) == E):
            raise ValueError("graph_optimizer: fixed needs K rows, edge_j and meas_ji need E rows")
        lm = np.zeros((0, 3)) if lm_pos_w is None else np.array(lm_pos_w, np.float64).reshape(-1, 3).copy()
        L = len(lm)
        ref, pr = _p(np.full(L, -1, np.int32) if lm_ref is None else np.asarray(lm_ref).reshape(-1), np.int32)
        if len(ref) != L:
            raise ValueError("graph_optimizer: lm_ref needs one entry per landmark")
        pose = np.zeros((K, 12))
        st = BaStats()
        _lib.check(_lib.lib().ovs_graph_optimize_host(self._h, K, S.ctypes.data_as(C.c_void_p), pf, E, pi if E else None, pj if E else None,
                                                      pm if E else None, int(self.fix_scale_), self.num_iter_, L,
                                                      lm.ctypes.data_as(C.c_void_p) if L else None, pr if L else None,
                                                      pose.ctypes.data_as(C.c_void_p), C.byref(st)))
        return S, pose, lm, _stats(st)


class prepared_local_ba(_optimizer_handle):
    """A local-BA problem kept resident on the device: prepare once, run many times (bench.py's
    device-resident leg), fetch the result of the last run."""

    def __init__(self, cam, setup_is_mono, poses, fixed, points, obs_kf, obs_lm, obs_xy, obs_x_right, inv_sigma_sq, device=0):
        super().__init__(device)
        poses, pp = _p(np.asarray(poses).reshape(-1, 12), np.float64); points, pq = _p(np.asarray(points).reshape(-1, 3), np.float64)
        fixed, pf = _p(fixed, np.uint8); obs_kf, pk = _p(obs_kf, np.int32); obs_lm, pl = _p(obs_lm, np.int32)
        obs_xy, po = _p(obs_xy, np.float32); inv_sigma_sq, pi = _p(inv_sigma_sq, np.float32)
        px = None
        if obs_x_right is not None:
            obs_x_right, px = _p(obs_x_right, np.float32)
        self.K, self.L, self.M = len(poses), len(points), len(obs_kf)
        _lib.check(_lib.lib().ovs_local_ba_prepare(self._h, C.byref(cam), int(setup_is_mono), self.K, pp, pf, self.L, pq, self.M,
                                                   pk, pl, po, px, pi))

    @classmethod
    def from_device(cls, cam, setup_is_mono, K, L, M, d_poses, d_fixed, d_points, d_obs_kf, d_obs_lm, d_obs_xy, d_obs_x_right, d_inv_sigma_sq, device=0, handle=None):
        """The graph is already resident in device memory (device pointers as ints; d_obs_x_right may be None)."""
        self = handle if handle is not None else cls.__new__(cls)
        if handle is None:
            _optimizer_handle.__init__(self, device)
        self.K, self.L, self.M = int(K), int(L), int(M)
        vp = lambda x: None if x is None else C.c_void_p(int(x))
        _lib.check(_lib.lib().ovs_local_ba_prepare_device(self._h, C.byref(cam), int(setup_is_mono), self.K, vp(d_poses), vp(d_fixed), self.L, vp(d_points),
                                                          self.M, vp(d_obs_kf), vp(d_obs_lm), vp(d_obs_xy), vp(d_obs_x_right), vp(d_inv_sigma_sq)))
        return self

    def run(self, num_first_iter=5, num_second_iter=10):
        st = BaStats()
        _lib.check(_lib.lib().ovs_local_ba_run(self._h, int(num_first_iter), int(num_second_iter), None, C.byref(st)))
        return _stats(st)

    def fetch(self):
        poses = np.zeros((self.K, 12)); points = np.zeros((self.L, 3)); out = np.zeros(self.M, np.uint8)
        _lib.check(_lib.lib().ovs_local_ba_fetch(self._h, poses.ctypes.data_as(C.c_void_p), points.ctypes.data_as(C.c_void_p),
                                                 out.ctypes.data_as(C.c_void_p)))
        return poses, points, out.astype(bool)


def smoke_check(O):
    """Used by __graft_entry__.smoke(): one small pose optimisation and local BA against the oracle."""
    from . import synth
    p = synth.pose_problem(400, model="perspective", seed=5, stereo=True)
    po = pose_optimizer()
    n, pose, flags, _ = po.optimize(camera(**p["cam"]), False, p["pts_w"], p["obs_xy"], p["obs_xr"], p["inv_sigma_sq"], p["poses"][0])
    on, opose, oflags, _ = O.pose_optimize(O.camera(**p["cam"]), False, p["pts_w"], p["obs_xy"], p["obs_xr"], p["inv_sigma_sq"], p["poses"][0])
    assert n == on and np.array_equal(flags, oflags) and np.allclose(pose, opose, rtol=0, atol=1e-7), "pose optimiser differs from the oracle"
    po.close()
    q = synth.ba_problem(6, 2, 300, model="equirectangular", seed=6)
    ba = local_bundle_adjuster()
    poses, points, outl, _ = ba.optimize(camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                         q["obs_xy"], None, q["inv_sigma_sq"])
    oposes, opoints, ooutl, _ = O.local_ba(O.camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                           q["obs_xy"], None, q["inv_sigma_sq"])
    c = synth.reprojection_chi2(q["cam"], poses, points, q["obs_kf"], q["obs_lm"], q["obs_xy"], None, q["inv_sigma_sq"], ~outl)
    oc = synth.reprojection_chi2(q["cam"], oposes, opoints, q["obs_kf"], q["obs_lm"], q["obs_xy"], None, q["inv_sigma_sq"], ~ooutl)
    assert abs(c - oc) <= 1e-4 * oc, "local BA final reprojection error differs from the oracle (%g vs %g)" % (c, oc)
    ba.close()
