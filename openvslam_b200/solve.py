"""Host-side mirror of openvslam::solve::sim3_solver, solve::pnp_solver, solve::essential_solver, solve::homography_solver and
solve::fundamental_solver (src/openvslam/solve/*_solver.h; names as in SURVEY.md 8a) over the C ABI of libovs_b200.so: loop
detection's Sim3 RANSAC, relocalisation's PnP RANSAC, the tracker's essential-matrix RANSAC and perspective map initialisation's
homography and fundamental-matrix RANSAC, each solved on the GPU for a whole batch of problems in one call.  The reference
constructs one solver per problem; here each problem is a `problem` of flat arrays (see include/ovs_b200.h,
ovs_*_solve_ransac_host, for the field-by-field mapping)."""
import ctypes as C
import itertools
import types

import numpy as np

from . import _lib
from .match import _matcher_handle
from .optimize import Camera, _optimizer_handle


def _offsets(counts):
    """(B + 1,) int32 offsets of B problems with these item counts"""
    return np.fromiter(itertools.accumulate(counts, initial=0), np.int32, len(counts) + 1)


def _batch(name, B, seeds, items, width):
    """What a batched solver passes to the C ABI for B problems.

    items: {kind: (B per-problem arrays, row shape, dtype)}.  Each kind gives off[kind], its (B + 1,) int32 offsets, and
    cat[kind], the arrays as rows of that shape concatenated in problem order (one zero row when there is none, so that there
    is a pointer to pass).  seeds: one per problem (default: the problem's index).  The outputs, zeroed, for at least one
    problem: model (B, width), valid, num_inliers, best_iter and best_score per problem, flags per item of the first kind."""
    off, cat = {}, {}
    for kind, (arrays, row, dt) in items.items():
        rows = [np.asarray(a, dt).reshape((-1,) + row) for a in arrays]
        off[kind] = _offsets([len(r) for r in rows])
        cat[kind] = np.concatenate(rows) if off[kind][-1] else np.zeros((1,) + row, dt)
    seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.ascontiguousarray(seeds, np.uint64).reshape(-1)
    if len(seeds) != B:
        raise ValueError(name + ": one seed per problem")
    N, Bo = int(off[next(iter(items))][-1]), max(B, 1)
    return types.SimpleNamespace(off=off, cat=cat, seeds=seeds if B else np.zeros(1, np.uint64), model=np.zeros((Bo, width)),
                                 valid=np.zeros(Bo, np.uint8), num_inliers=np.zeros(Bo, np.int32), best_iter=np.zeros(Bo, np.int32),
                                 best_score=np.zeros(Bo), flags=np.zeros(max(N, 1), np.uint8))


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


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
        for p in problems:
            n = len(np.asarray(p["sigma_sq_1"]).reshape(-1))
            if not (np.asarray(p["pos_w_1"]).size == np.asarray(p["pos_w_2"]).size == 3 * n and np.asarray(p["sigma_sq_2"]).size == n):
                raise ValueError("sim3_solver: pos_w_1 / pos_w_2 need (n, 3) and sigma_sq_1 / sigma_sq_2 n entries")
        col = lambda key: [p[key] for p in problems]
        t = _batch("sim3_solver", B, seeds, {"pos_w_1": (col("pos_w_1"), (3,), np.float64), "sigma_sq_1": (col("sigma_sq_1"), (), np.float32),
                                             "pos_w_2": (col("pos_w_2"), (3,), np.float64), "sigma_sq_2": (col("sigma_sq_2"), (), np.float32)}, 13)
        cams_1 = (Camera * max(B, 1))(*col("cam_1"))
        cams_2 = (Camera * max(B, 1))(*col("cam_2"))
        pose1, pose2 = (np.concatenate([np.asarray(p[k], np.float64).reshape(12) for p in problems]) if B else np.zeros(12)
                        for k in ("pose_1w", "pose_2w"))
        c, off = t.cat, t.off["pos_w_1"]
        _lib.check(_lib.lib().ovs_sim3_solve_ransac_host(self._h, B, _vp(off), cams_1, _vp(pose1), cams_2, _vp(pose2),
                                                         _vp(c["pos_w_1"]), _vp(c["sigma_sq_1"]), _vp(c["pos_w_2"]), _vp(c["sigma_sq_2"]),
                                                         int(self.fix_scale_), self.min_num_inliers_, int(max_num_iter), _vp(t.seeds),
                                                         _vp(t.model), _vp(t.valid), _vp(t.num_inliers), _vp(t.best_iter), _vp(t.flags)))
        return [dict(valid=bool(t.valid[b]), sim3_12=t.model[b].copy(), num_inliers=int(t.num_inliers[b]), best_iter=int(t.best_iter[b]),
                     inliers=t.flags[off[b]:off[b + 1]].astype(bool)) for b in range(B)]


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
        for p in problems:
            n = len(np.asarray(p["scale_factor"]).reshape(-1))
            if not (np.asarray(p["bearings"]).size == np.asarray(p["pos_w"]).size == 3 * n):
                raise ValueError("pnp_solver: bearings / pos_w need (n, 3) and scale_factor n entries")
        col = lambda key: [p[key] for p in problems]
        t = _batch("pnp_solver", B, seeds, {"bearings": (col("bearings"), (3,), np.float64), "pos_w": (col("pos_w"), (3,), np.float64),
                                            "scale_factor": (col("scale_factor"), (), np.float32)}, 12)
        c, off = t.cat, t.off["bearings"]
        _lib.check(_lib.lib().ovs_pnp_solve_ransac_host(self._h, B, _vp(off), _vp(c["bearings"]), _vp(c["pos_w"]), _vp(c["scale_factor"]),
                                                        self.min_num_inliers_, int(max_num_iter), int(bool(recompute)), _vp(t.seeds),
                                                        _vp(t.model), _vp(t.valid), _vp(t.num_inliers), _vp(t.best_iter), _vp(t.flags)))
        return [dict(valid=bool(t.valid[b]), pose_cw=t.model[b].copy(), num_inliers=int(t.num_inliers[b]), best_iter=int(t.best_iter[b]),
                     inliers=t.flags[off[b]:off[b + 1]].astype(bool)) for b in range(B)]


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
        for p in problems:
            n = np.asarray(p["bearings_1"]).size // 3
            if not (np.asarray(p["bearings_1"]).size == np.asarray(p["bearings_2"]).size == 3 * n):
                raise ValueError("essential_solver: bearings_1 / bearings_2 need (n, 3) each")
        t = _batch("essential_solver", B, seeds, {k: ([p[k] for p in problems], (3,), np.float64) for k in ("bearings_1", "bearings_2")}, 9)
        off = t.off["bearings_1"]
        _lib.check(_lib.lib().ovs_essential_solve_ransac_host(self._h, B, _vp(off), _vp(t.cat["bearings_1"]), _vp(t.cat["bearings_2"]),
                                                              int(max_num_iter), int(bool(recompute)), _vp(t.seeds), _vp(t.model), _vp(t.valid),
                                                              _vp(t.num_inliers), _vp(t.best_iter), _vp(t.best_score), _vp(t.flags)))
        return [dict(valid=bool(t.valid[b]), E_21=t.model[b].reshape(3, 3).copy(), num_inliers=int(t.num_inliers[b]),
                     best_iter=int(t.best_iter[b]), best_score=float(t.best_score[b]), inliers=t.flags[off[b]:off[b + 1]].astype(bool))
                for b in range(B)]


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
        for p in problems:
            if np.size(p["keypts_1"]) % 2 or np.size(p["keypts_2"]) % 2:
                raise ValueError(name + ": keypts_1 / keypts_2 need (n, 2) each")
        t = _batch(name, B, seeds, {"matches_12": ([p["matches_12"] for p in problems], (2,), np.int32)}, 9)

        def keypoints(key):
            # the records are filled from each view's x, y, so the float copy of all keypoints is never formed
            arrs = [np.asarray(p[key], np.float32).reshape(-1, 2) for p in problems]
            off = _offsets([len(a) for a in arrs])
            out = np.zeros(max(int(off[-1]), 1), _KEYPOINT)
            for a, o in zip(arrs, off):
                out["x"][o:o + len(a)] = a[:, 0]; out["y"][o:o + len(a)] = a[:, 1]
            return off, out
        (o1, k1), (o2, k2), moff = keypoints("keypts_1"), keypoints("keypts_2"), t.off["matches_12"]
        _lib.check(getattr(_lib.lib(), self._entry)(self._h, B, _vp(o1), _vp(k1), _vp(o2), _vp(k2), _vp(moff),
                                                    _vp(t.cat["matches_12"]), C.c_float(self.sigma_), int(max_num_iter), int(bool(recompute)),
                                                    _vp(t.seeds), _vp(t.model), _vp(t.valid), _vp(t.num_inliers), _vp(t.best_iter),
                                                    _vp(t.best_score), _vp(t.flags)))
        return [{"valid": bool(t.valid[b]), self._key: t.model[b].reshape(3, 3).copy(), "num_inliers": int(t.num_inliers[b]),
                 "best_iter": int(t.best_iter[b]), "best_score": float(t.best_score[b]), "inliers": t.flags[moff[b]:moff[b + 1]].astype(bool)}
                for b in range(B)]


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
