"""Host-side mirror of openvslam::solve::sim3_solver, solve::pnp_solver, solve::essential_solver, solve::homography_solver and
solve::fundamental_solver (src/openvslam/solve/*_solver.h; names as in SURVEY.md 8a) over the C ABI of libovs_b200.so: loop
detection's Sim3 RANSAC, relocalisation's PnP RANSAC, the tracker's essential-matrix RANSAC and perspective map initialisation's
homography and fundamental-matrix RANSAC, each solved on the GPU for a whole batch of problems in one call.  The reference
constructs one solver per problem; here each problem is a `problem` of flat arrays (see include/ovs_b200.h,
ovs_*_solve_ransac_host, for the field-by-field mapping)."""
import ctypes as C

import numpy as np

from . import _lib
from .match import _matcher_handle
from .optimize import Camera, _optimizer_handle, _p


class sim3_solver(_optimizer_handle):
    """openvslam::solve::sim3_solver(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2, fix_scale, min_num_inliers = 20), batched.

    find_via_ransac(problems, max_num_iter=200, seeds=None): problems is a list of dicts with
      cam_1, cam_2            optimize.Camera of keyframe 1 / keyframe 2,
      pose_1w, pose_2w        cam_pose_cw of each keyframe as {R row-major (9), t (3)},
      pos_w_1, pos_w_2        (n, 3) world positions of the matched landmarks (lm_1 of keyframe 1, lm_2 matched to it),
      sigma_sq_1, sigma_sq_2  (n,) level_sigma_sq_ of each landmark's keypoint octave in its keyframe;
    seeds: one sampler seed per problem (default: the problem's index).  A problem gives the same result alone or in a batch.
    Returns one dict per problem: valid (solution_is_valid()), sim3_12 {R (9), t (3), s}, num_inliers, best_iter (-1: no
    hypothesis had an inlier), inliers (n,) bool."""

    def __init__(self, fix_scale, min_num_inliers=20, device=0):
        super().__init__(device)
        self.fix_scale_ = bool(fix_scale)
        self.min_num_inliers_ = int(min_num_inliers)

    def find_via_ransac(self, problems, max_num_iter=200, seeds=None):
        B = len(problems)
        counts = []
        for p in problems:
            n = len(np.asarray(p["sigma_sq_1"]).reshape(-1))
            if not (np.asarray(p["pos_w_1"]).size == np.asarray(p["pos_w_2"]).size == 3 * n and np.asarray(p["sigma_sq_2"]).size == n):
                raise ValueError("sim3_solver: pos_w_1 / pos_w_2 need (n, 3) and sigma_sq_1 / sigma_sq_2 n entries")
            counts.append(n)
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum(counts)
        N = int(off[-1])
        seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.asarray(seeds, np.uint64).reshape(-1)
        if len(seeds) != B:
            raise ValueError("sim3_solver: one seed per problem")
        cams_1 = (Camera * max(B, 1))(*[p["cam_1"] for p in problems])
        cams_2 = (Camera * max(B, 1))(*[p["cam_2"] for p in problems])

        def cat(key, width, dt):
            if N == 0:
                return np.zeros((1, width) if width > 1 else 1, dt)
            return np.concatenate([np.asarray(p[key], dt).reshape(-1, width) if width > 1 else np.asarray(p[key], dt).reshape(-1)
                                   for p in problems])
        pose1, pp1 = _p(np.concatenate([np.asarray(p["pose_1w"], np.float64).reshape(12) for p in problems]) if B else np.zeros(12), np.float64)
        pose2, pp2 = _p(np.concatenate([np.asarray(p["pose_2w"], np.float64).reshape(12) for p in problems]) if B else np.zeros(12), np.float64)
        w1, pw1 = _p(cat("pos_w_1", 3, np.float64), np.float64); s1, ps1 = _p(cat("sigma_sq_1", 1, np.float32), np.float32)
        w2, pw2 = _p(cat("pos_w_2", 3, np.float64), np.float64); s2, ps2 = _p(cat("sigma_sq_2", 1, np.float32), np.float32)
        off_, po = _p(off, np.int32); seeds_, pseed = _p(seeds if B else np.zeros(1, np.uint64), np.uint64)
        S = np.zeros((max(B, 1), 13)); valid = np.zeros(max(B, 1), np.uint8)
        ninl = np.zeros(max(B, 1), np.int32); best = np.zeros(max(B, 1), np.int32); flags = np.zeros(max(N, 1), np.uint8)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().ovs_sim3_solve_ransac_host(self._h, B, po, cams_1, pp1, cams_2, pp2, pw1, ps1, pw2, ps2, int(self.fix_scale_),
                                                         self.min_num_inliers_, int(max_num_iter), pseed, vp(S), vp(valid), vp(ninl), vp(best),
                                                         vp(flags)))
        return [dict(valid=bool(valid[b]), sim3_12=S[b].copy(), num_inliers=int(ninl[b]), best_iter=int(best[b]),
                     inliers=flags[off[b]:off[b + 1]].astype(bool)) for b in range(B)]


class pnp_solver(_optimizer_handle):
    """openvslam::solve::pnp_solver(valid_bearings, valid_keypts, valid_points, scale_factors, min_num_inliers = 10), batched.

    find_via_ransac(problems, max_num_iter=30, recompute=True, seeds=None): problems is a list of dicts with
      bearings      (n, 3) unit bearings of the frame keypoints (frm.bearings_),
      pos_w         (n, 3) world positions of the matched landmarks,
      scale_factor  (n,) scale_factors_[octave] of each keypoint, in (0, 90];
    seeds: one sampler seed per problem (default: the problem's index).  A problem gives the same result alone or in a batch.
    Returns one dict per problem: valid (solution_is_valid()), pose_cw {R row-major (9), t (3)} (get_best_cam_pose()),
    num_inliers, best_iter (-1: no hypothesis had an inlier), inliers (n,) bool (get_inlier_flags())."""

    def __init__(self, min_num_inliers=10, device=0):
        super().__init__(device)
        self.min_num_inliers_ = int(min_num_inliers)

    def find_via_ransac(self, problems, max_num_iter=30, recompute=True, seeds=None):
        B = len(problems)
        counts = []
        for p in problems:
            n = len(np.asarray(p["scale_factor"]).reshape(-1))
            if not (np.asarray(p["bearings"]).size == np.asarray(p["pos_w"]).size == 3 * n):
                raise ValueError("pnp_solver: bearings / pos_w need (n, 3) and scale_factor n entries")
            counts.append(n)
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum(counts)
        N = int(off[-1])
        seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.asarray(seeds, np.uint64).reshape(-1)
        if len(seeds) != B:
            raise ValueError("pnp_solver: one seed per problem")

        def cat(key, width, dt):
            if N == 0:
                return np.zeros((1, width) if width > 1 else 1, dt)
            return np.concatenate([np.asarray(p[key], dt).reshape(-1, width) if width > 1 else np.asarray(p[key], dt).reshape(-1)
                                   for p in problems])
        b, pb = _p(cat("bearings", 3, np.float64), np.float64); w, pw = _p(cat("pos_w", 3, np.float64), np.float64)
        s, ps = _p(cat("scale_factor", 1, np.float32), np.float32)
        off_, po = _p(off, np.int32); seeds_, pseed = _p(seeds if B else np.zeros(1, np.uint64), np.uint64)
        pose = np.zeros((max(B, 1), 12)); valid = np.zeros(max(B, 1), np.uint8)
        ninl = np.zeros(max(B, 1), np.int32); best = np.zeros(max(B, 1), np.int32); flags = np.zeros(max(N, 1), np.uint8)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().ovs_pnp_solve_ransac_host(self._h, B, po, pb, pw, ps, self.min_num_inliers_, int(max_num_iter),
                                                        int(bool(recompute)), pseed, vp(pose), vp(valid), vp(ninl), vp(best), vp(flags)))
        return [dict(valid=bool(valid[b]), pose_cw=pose[b].copy(), num_inliers=int(ninl[b]), best_iter=int(best[b]),
                     inliers=flags[off[b]:off[b + 1]].astype(bool)) for b in range(B)]


class essential_solver(_matcher_handle):
    """openvslam::solve::essential_solver(bearings_1, bearings_2, matches_12), batched, on a matcher handle (its own buffers: the
    handle's brute-force matchers are unaffected).

    find_via_ransac(problems, max_num_iter, recompute=True, seeds=None): problems is a list of dicts with
      bearings_1  (n, 3) unit bearings of camera 1 gathered per match (bearings_1_[matches_12_[i].first]),
      bearings_2  (n, 3) the same for camera 2 (bearings_2_[matches_12_[i].second]);
    seeds: one sampler seed per problem (default: the problem's index).  A problem gives the same result alone or in a batch.
    Returns one dict per problem: valid (solution_is_valid()), E_21 (3, 3) (get_best_E_21(); zero when no hypothesis scored),
    num_inliers, best_iter (-1: none), best_score, inliers (n,) bool (get_inlier_matches())."""

    def find_via_ransac(self, problems, max_num_iter, recompute=True, seeds=None):
        B = len(problems)
        counts = []
        for p in problems:
            n = np.asarray(p["bearings_1"]).size // 3
            if not (np.asarray(p["bearings_1"]).size == np.asarray(p["bearings_2"]).size == 3 * n):
                raise ValueError("essential_solver: bearings_1 / bearings_2 need (n, 3) each")
            counts.append(n)
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum(counts)
        N = int(off[-1])
        seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.asarray(seeds, np.uint64).reshape(-1)
        if len(seeds) != B:
            raise ValueError("essential_solver: one seed per problem")

        def cat(key):
            if N == 0:
                return np.zeros((1, 3))
            return np.concatenate([np.asarray(p[key], np.float64).reshape(-1, 3) for p in problems])
        b1, pb1 = _p(cat("bearings_1"), np.float64); b2, pb2 = _p(cat("bearings_2"), np.float64)
        off_, po = _p(off, np.int32); seeds_, pseed = _p(seeds if B else np.zeros(1, np.uint64), np.uint64)
        E = np.zeros((max(B, 1), 9)); valid = np.zeros(max(B, 1), np.uint8); score = np.zeros(max(B, 1))
        ninl = np.zeros(max(B, 1), np.int32); best = np.zeros(max(B, 1), np.int32); flags = np.zeros(max(N, 1), np.uint8)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().ovs_essential_solve_ransac_host(self._h, B, po, pb1, pb2, int(max_num_iter), int(bool(recompute)), pseed,
                                                              vp(E), vp(valid), vp(ninl), vp(best), vp(score), vp(flags)))
        return [dict(valid=bool(valid[b]), E_21=E[b].reshape(3, 3).copy(), num_inliers=int(ninl[b]), best_iter=int(best[b]),
                     best_score=float(score[b]), inliers=flags[off[b]:off[b + 1]].astype(bool)) for b in range(B)]


# cv::KeyPoint / ovs_keypoint (28 bytes): the two-view solvers read pt only
_KEYPOINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"),
                      ("class_id", "<i4")])


class _two_view_solver(_matcher_handle):
    _entry = None
    _key = None

    def __init__(self, sigma=1.0, device=0):
        super().__init__(device)
        self.sigma_ = float(sigma)

    def find_via_ransac(self, problems, max_num_iter, recompute=True, seeds=None):
        name = type(self).__name__
        B = len(problems)
        kp1, kp2, mt = [], [], []
        for p in problems:
            k1 = np.asarray(p["keypts_1"], np.float32); k2 = np.asarray(p["keypts_2"], np.float32)
            m = np.asarray(p["matches_12"]).reshape(-1, 2) if np.asarray(p["matches_12"]).size else np.zeros((0, 2), np.int32)
            if k1.size % 2 or k2.size % 2:
                raise ValueError(name + ": keypts_1 / keypts_2 need (n, 2) each")
            kp1.append(k1.reshape(-1, 2)); kp2.append(k2.reshape(-1, 2)); mt.append(m.astype(np.int32))

        def offsets(arrs):
            off = np.zeros(B + 1, np.int32)
            off[1:] = np.cumsum([len(a) for a in arrs])
            return off
        koff1, koff2, moff = offsets(kp1), offsets(kp2), offsets(mt)
        N = int(moff[-1])
        seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.asarray(seeds, np.uint64).reshape(-1)
        if len(seeds) != B:
            raise ValueError(name + ": one seed per problem")

        def keypoints(arrs):
            xy = np.concatenate(arrs) if B and sum(len(a) for a in arrs) else np.zeros((0, 2), np.float32)
            out = np.zeros(max(len(xy), 1), _KEYPOINT)
            out["x"][:len(xy)] = xy[:, 0]; out["y"][:len(xy)] = xy[:, 1]
            return out
        k1, k2 = keypoints(kp1), keypoints(kp2)
        m, pm = _p(np.concatenate(mt) if N else np.zeros((1, 2), np.int32), np.int32)
        o1, po1 = _p(koff1, np.int32); o2, po2 = _p(koff2, np.int32); om, pom = _p(moff, np.int32)
        seeds_, pseed = _p(seeds if B else np.zeros(1, np.uint64), np.uint64)
        M = np.zeros((max(B, 1), 9)); valid = np.zeros(max(B, 1), np.uint8); score = np.zeros(max(B, 1))
        ninl = np.zeros(max(B, 1), np.int32); best = np.zeros(max(B, 1), np.int32); flags = np.zeros(max(N, 1), np.uint8)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(getattr(_lib.lib(), self._entry)(self._h, B, po1, vp(k1), po2, vp(k2), pom, pm, C.c_float(self.sigma_), int(max_num_iter),
                                                    int(bool(recompute)), pseed, vp(M), vp(valid), vp(ninl), vp(best), vp(score), vp(flags)))
        return [{"valid": bool(valid[b]), self._key: M[b].reshape(3, 3).copy(), "num_inliers": int(ninl[b]), "best_iter": int(best[b]),
                 "best_score": float(score[b]), "inliers": flags[moff[b]:moff[b + 1]].astype(bool)} for b in range(B)]


class homography_solver(_two_view_solver):
    """openvslam::solve::homography_solver(undist_keypts_1, undist_keypts_2, matches_12, sigma), batched, on a matcher handle (its
    own buffers: the handle's matchers and essential solver are unaffected).  Perspective map initialisation passes sigma = 1.0.

    find_via_ransac(problems, max_num_iter, recompute=True, seeds=None): problems is a list of dicts with
      keypts_1    (n1, 2) undistorted keypoints of view 1 (all of them: the normalisation runs over every keypoint),
      keypts_2    (n2, 2) the same of view 2,
      matches_12  (m, 2) pairs (idx_1, idx_2) into them;
    seeds: one sampler seed per problem (default: the problem's index).  A problem gives the same result alone or in a batch.
    Returns one dict per problem: valid (solution_is_valid()), H_21 (3, 3) (get_best_H_21(), p2 ~ H_21 p1; zero when no hypothesis
    scored), num_inliers, best_iter (-1: none), best_score (get_best_score()), inliers (m,) bool (get_inlier_matches())."""
    _entry = "ovs_homography_solve_ransac_host"
    _key = "H_21"


class fundamental_solver(_two_view_solver):
    """openvslam::solve::fundamental_solver(undist_keypts_1, undist_keypts_2, matches_12, sigma), batched; the same interface as
    homography_solver, with F_21 (3, 3) (get_best_F_21(), p2^T F_21 p1 = 0, rank 2) in place of H_21."""
    _entry = "ovs_fundamental_solve_ransac_host"
    _key = "F_21"
