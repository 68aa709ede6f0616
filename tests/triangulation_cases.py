"""Named, constructed cases for the two-view triangulator (tests/triangulation_reference.py, its CPU and GPU tests).

Each case holds noise-free points whose bearings are taken from the exact points; one input is then stepped over single
floats (single doubles for rays_parallax_deg_thr and for a camera centre) so that exactly one gate flips between
neighbouring pairs, and each knife-edge case has pairs on both sides of its gate.  Where a two-camera point stands between
the pair and its gate, the stepped values are chosen so that no decision lies within the point's error bound (the
construction moves the point and searches again until that holds).

A Case: name, group, expect (the triangulation_reference.gate_counts keys the case must reach: both outcomes of the gate it
steps), knife_edge, and problems: [(keyfrm_1, keyfrm_2, pairs (m, 2) int32, rays_parallax_deg_thr)]."""
import math

import numpy as np

import triangulation_problems as TP
import triangulation_reference as R
from openvslam_b200 import module, optimize

F32 = np.float32
FX, FY, CX, CY = TP.FX, TP.FY, TP.CX, TP.CY
TRUE_BASELINE = 0.5
TINY = np.nextafter(F32(0.0), F32(1.0))            # the smallest positive float (subnormal)


class Case:
    def __init__(self, name, group, problems, expect=(), knife_edge=True):
        self.name, self.group, self.problems, self.knife_edge = name, group, problems, knife_edge
        self.expect = [(expect, True), (expect, False)] if isinstance(expect, str) else list(expect)

    def __repr__(self):
        return self.name


def tables(levels, scale_factor=1.2):
    sf = np.cumprod(np.concatenate([[F32(1.0)], np.full(levels - 1, F32(scale_factor))]).astype(F32)).astype(F32)
    return sf, (sf * sf).astype(F32)


def rot_y(deg):
    a = math.radians(deg)
    return np.array([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]])


R_Y90 = np.array([[0.0, 0.0, -1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])    # optical axis along world +x, exact
R_Y180 = np.diag([-1.0, 1.0, -1.0])                                        # optical axis along world -z, exact


def perspective(fb=FX * TRUE_BASELINE):
    return optimize.camera("perspective", FX, FY, CX, CY, focal_x_baseline=fb, cols=TP.COLS, rows=TP.ROWS)


def equirectangular():
    return optimize.camera("equirectangular", cols=TP.EQ_COLS, rows=TP.EQ_ROWS)


class View:
    """One keyframe being filled keypoint by keypoint."""

    def __init__(self, R_cw, centre, camera=None, levels=8, sf=None, sig=None, scale_factor=1.2, true_baseline=TRUE_BASELINE):
        self.R = np.asarray(R_cw, np.float64)
        self.pose = np.concatenate([self.R.reshape(9), -self.R @ np.asarray(centre, np.float64)])
        self.camera = camera if camera is not None else perspective()
        t_sf, t_sig = tables(levels)
        self.sf = t_sf if sf is None else np.asarray(sf, F32)
        self.sig = t_sig if sig is None else np.asarray(sig, F32)
        self.scale_factor, self.true_baseline = scale_factor, true_baseline
        self.kp = []

    def observe(self, X):
        """exact bearing, (u, v) in double, camera-frame z"""
        Xc = self.R @ np.asarray(X, np.float64) + self.pose[9:]
        b = Xc / np.linalg.norm(Xc)
        if self.camera.model == R.EQUIRECTANGULAR:
            u = self.camera.cols * (0.5 + math.atan2(b[0], b[2]) / (2 * math.pi))
            v = self.camera.rows * (0.5 + math.asin(b[1]) / math.pi)
        else:
            u, v = FX * Xc[0] / Xc[2] + CX, FY * Xc[1] / Xc[2] + CY
        return b, u, v, Xc[2]

    def add(self, bearing, x, y, octave=0, x_right=-1.0, depth=-1.0):
        self.kp.append((np.asarray(bearing, np.float64), F32(x), F32(y), int(octave), F32(x_right), F32(depth)))
        return len(self.kp) - 1

    def add_point(self, X, octave=0, stereo=False, depth=None):
        """an exact observation of X (keypoint = the float of the projection); stereo: x_right = (float)(u - fb / z)"""
        b, u, v, z = self.observe(X)
        if stereo:
            d = z if depth is None else depth
            return self.add(b, u, v, octave, F32(u - self.camera.focal_x_baseline / z), d)
        return self.add(b, u, v, octave)

    def keyframe(self):
        n = len(self.kp)
        col = lambda k: [p[k] for p in self.kp]
        return module.keyframe(self.pose, self.camera, self.scale_factor, self.sf, self.sig, np.array(col(1), F32), np.array(col(2), F32),
                               np.array(col(3), np.int32), np.array(col(0)).reshape(n, 3), angle=np.zeros(n, F32),
                               stereo_x_right=np.array(col(4), F32), depths=np.array(col(5), F32), true_baseline=self.true_baseline)


def _problem(v1, v2, deg=1.0):
    n = len(v1.kp)
    assert n == len(v2.kp)
    return v1.keyframe(), v2.keyframe(), np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32), deg


def _floats_around(x, below, above):
    """the `below` floats under float(x) and the `above` ones from it on"""
    f = F32(x)
    out = [f]
    for _ in range(below):
        out.insert(0, np.nextafter(out[0], F32(-np.inf)))
    for _ in range(above - 1):
        out.append(np.nextafter(out[-1], F32(np.inf)))
    return out


def _crossing(values, outcome):
    """index k with outcome(values[k]) != outcome(values[k + 1]) (the first), or None"""
    o = [outcome(v) for v in values]
    for k in range(len(o) - 1):
        if o[k] != o[k + 1]:
            return k
    return None


def _clear(problem):
    """the reference leaves no decision of this problem to the point's bound"""
    kf1, kf2, pairs, deg = problem
    return not R.triangulate(kf1, kf2, pairs, deg).skip


# ------------------------------------------------------------------------------------------------ parallax


def _deg_crossing(c, strict_above):
    """the largest double deg with cos_threshold(deg) > c (strict_above) or >= c, found by bisection on the bits"""
    ok = (lambda d: R.cos_threshold(d) > c) if strict_above else (lambda d: R.cos_threshold(d) >= c)
    lo = np.float64(math.degrees(math.acos(c)) * 0.999)
    hi = np.float64(math.degrees(math.acos(c)) * 1.001)
    assert ok(lo) and not ok(hi)
    a, b = lo.view(np.int64), hi.view(np.int64)
    while b - a > 1:
        m = (a + b) // 2
        if ok(np.int64(m).view(np.float64)):
            a = m
        else:
            b = m
    return float(np.int64(a).view(np.float64)), float(np.int64(b).view(np.float64))


def parallax():
    out = []
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(rot_y(1.0), [0.3, 0.01, 0.02])
    X = np.array([0.2, 0.1, 10.0])
    v1.add_point(X); v2.add_point(X)
    kf1, kf2, pairs, _ = _problem(v1, v2)
    c = R.cos_rays(kf1, 0, kf2, 0)
    probs = []
    for strict in (True, False):       # cos_thr just above / at or below cos_rays, at consecutive doubles of the threshold
        a, b = _deg_crossing(c, strict)
        probs += [(kf1, kf2, pairs, a), (kf1, kf2, pairs, b)]
    at = [p for p in probs if R.cos_threshold(p[3]) == c]
    out.append(Case("parallax: cos_thr steps across cos_rays (%d thresholds at cos_rays)" % len(at), "parallax", probs, "parallax"))
    # rays at 90 degrees (cos_rays == 0 exactly) and beyond: never two cameras; a hair under 90 degrees: two cameras
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(R_Y90, [-5.0, 0, 5.0])
    X = np.array([0.0, 0.0, 5.0])
    v1.add_point(X); v2.add_point(X)
    v1.add_point(X); v2.add(*_bearing_of(v2, [5.0, 0.0, -0.5]), CX, CY)               # opposite side of 90 degrees
    v1.add_point(X); v2.add(*_bearing_of(v2, [5.0, 0.0, 1e-9]), CX, CY)               # just under 90 degrees
    out.append(Case("parallax: cos_rays == 0, < 0 and just above 0", "parallax", [_problem(v1, v2)], "parallax"))
    return out


def _bearing_of(view, d_world):
    """the bearing (in view's frame) of the world direction d_world"""
    b = view.R @ np.asarray(d_world, np.float64)
    return (b / np.linalg.norm(b),)


# ------------------------------------------------------------------------------------------------ stereo parallax


def _depth_crossing(cos_r, h):
    """floats d around the crossing of (d^2 - h^2) / (d^2 + h^2) with cos_r"""
    d0 = h / math.tan(math.acos(cos_r) / 2.0)
    vals = _floats_around(d0, 40, 40)
    cs = lambda d: (float(d) ** 2 - h * h) / (float(d) ** 2 + h * h)
    k = _crossing(vals, lambda d: cos_r < cs(d))
    assert k is not None
    return vals[k - 1:k + 3]


def stereo_parallax():
    out = []
    h = TRUE_BASELINE / 2.0
    X = np.array([0.25, 0.05, 12.0])
    # stereo in view 1, in view 2, in both (the other view's depth far): the stepped depth's cs crosses cos_rays
    for which in ("1", "2", "both"):
        v1, v2 = View(np.eye(3), [0, 0, 0]), View(np.eye(3), [0.5, 0.0, 0.0])
        b1, u1, y1, z1 = v1.observe(X); b2, u2, y2, z2 = v2.observe(X)
        for d in _depth_crossing(_cos_rays_at(v1, v2, X), h):
            xr1, xr2 = F32(u1 - v1.camera.focal_x_baseline / z1), F32(u2 - v2.camera.focal_x_baseline / z2)
            if which == "1":
                v1.add(b1, u1, y1, 0, xr1, d); v2.add(b2, u2, y2)
            elif which == "2":
                v1.add(b1, u1, y1); v2.add(b2, u2, y2, 0, xr2, d)
            else:
                v1.add(b1, u1, y1, 0, xr1, d); v2.add(b2, u2, y2, 0, xr2, F32(1000.0))
        out.append(Case("stereo parallax: depth of view %s across cos_rays" % which, "stereo_parallax", [_problem(v1, v2)], "stereo parallax"))
    # both stereo, equal depth and baseline: cs1 == cs2, so when the two-camera test fails no branch is taken
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(np.eye(3), [0.5, 0.0, 0.0])
    b1, u1, y1, z1 = v1.observe(X); b2, u2, y2, z2 = v2.observe(X)
    for d in _depth_crossing(_cos_rays_at(v1, v2, X), h):
        v1.add(b1, u1, y1, 0, F32(u1 - v1.camera.focal_x_baseline / z1), d)
        v2.add(b2, u2, y2, 0, F32(u2 - v2.camera.focal_x_baseline / z2), d)
    out.append(Case("stereo parallax: equal depths, cs1 == cs2 (two cameras or no branch)", "stereo_parallax", [_problem(v1, v2)],
                    [("stereo parallax", True), ("branch", "none")]))
    # x_right in {-smallest float, -0.0f, 0.0f, +smallest float}: monocular (two cameras) against stereo (stereo 1).  The
    # point sits where u - fb / z is 0, so x_right = 0 is the right-image x of a true stereo observation.
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(np.eye(3), [0.1, 0.0, 0.0])
    X = np.array([(FX * TRUE_BASELINE / 2.0 - CX) / FX * 2.0, 0.1, 2.0])
    b1, u1, y1, z1 = v1.observe(X)
    for xr in (-TINY, F32(-0.0), F32(0.0), TINY):
        v1.add(b1, u1, y1, 0, xr, F32(z1)); v2.add_point(X)
    out.append(Case("stereo parallax: x_right -tiny, -0, +0, +tiny", "stereo_parallax", [_problem(v1, v2)],
                    [("branch", "two cameras"), ("branch", "stereo 1")]))
    # a stereo keypoint of depth 0 (and -0, and negative) takes its branch and is rejected (zero vector at camera 1's centre);
    # one of the smallest positive depth is back-projected
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(np.eye(3), [0.1, 0.0, 0.0])
    for d in (F32(0.0), F32(-0.0), F32(-1.0), TINY):
        v1.add(b1, u1, y1, 0, F32(u1 - v1.camera.focal_x_baseline / z1), d); v2.add_point(X)
    out.append(Case("stereo parallax: depth 0, -0, -1 and the smallest float", "stereo_parallax", [_problem(v1, v2)], "cheirality 1"))
    return out


def _cos_rays_at(v1, v2, X):
    """cos_rays of the exact observations of X from the poses of v1 and v2"""
    a, b = View(v1.R, [0, 0, 0]), View(v2.R, [0, 0, 0])
    a.pose, b.pose = v1.pose, v2.pose
    a.add_point(X); b.add_point(X)
    kf1, kf2, _, _ = _problem(a, b)
    return R.cos_rays(kf1, 0, kf2, 0)


# ------------------------------------------------------------------------------------------------ reprojection


def _reprojection_problem(levels, octave, view, stereo, model, shift):
    """one two-camera pair per stepped value of view `view`'s keypoint x (mono) or x_right (stereo) across the chi-square
    bound of its octave"""
    cam = equirectangular() if model == "equirectangular" else perspective()
    sf, sig = tables(levels)
    mk = lambda R_, c: View(R_, c, cam, levels, sf, sig)
    X = np.array([0.3 + shift, -0.2 + 0.5 * shift, 8.0]) if model != "equirectangular" else np.array([2.0 + shift, 1.0, 5.0])
    v = [mk(np.eye(3), [0, 0, 0]), mk(rot_y(2.0), [1.0, 0.02, 0.05])]
    obs = [w.observe(X) for w in v]
    bnd = float((R.CHI_SQ_3D if stereo else R.CHI_SQ_2D) * sig[octave])
    s = view - 1
    b, u, y, z = obs[s]
    if stereo:
        xr0 = u - cam.focal_x_baseline / z
        cands = _floats_around(xr0 - math.sqrt(bnd), 3, 3)
    else:
        cands = _floats_around(u + math.sqrt(max(bnd - (y - float(F32(y))) ** 2, 0.0)), 3, 3)
    for val in cands:
        for k, w in enumerate(v):
            bk, uk, yk, zk = obs[k]
            xrk = F32(uk - cam.focal_x_baseline / zk) if stereo else F32(-1.0)
            dk = F32(zk) if stereo else F32(-1.0)
            if k == s:
                w.add(bk, uk if stereo else val, yk, octave, val if stereo else xrk, dk)
            else:
                w.add(bk, uk, yk, octave, xrk, dk)
    kf1, kf2, pairs, deg = _problem(*v)
    res = R.triangulate(kf1, kf2, pairs, deg)
    k = _crossing(list(range(len(cands))), lambda j: bool(res.reason[j] == R.REPROJ_1 + s))
    assert k is not None and k >= 1 and k + 2 < len(cands), (levels, octave, view, stereo, model, res.reason)
    sel = pairs[k - 1:k + 3]
    prob = (kf1, kf2, sel, deg)
    return prob if _clear(prob) else None


def reprojection():
    out = []
    for model in ("perspective", "equirectangular"):
        for stereo in ((False, True) if model == "perspective" else (False,)):
            for view in (1, 2):
                probs = []
                for levels in (range(1, 9) if model == "perspective" else (8,)):
                    for octave in range(levels):
                        for shift in np.arange(0.0, 0.05, 0.001):
                            p = _reprojection_problem(levels, octave, view, stereo, model, shift)
                            if p is not None:
                                break
                        assert p is not None
                        probs.append(p)
                kind = "stereo" if stereo else "mono"
                out.append(Case("reprojection: %s %s view %d, every octave of 1- to 8-level tables" % (model, kind, view), "reprojection",
                                probs, "reprojection %d %s" % (view, kind)))
    out.append(Case("reprojection: squared error exactly at the bound (mono and stereo, stereo-1 branch)", "reprojection",
                    [_exact_bound_problem(False), _exact_bound_problem(True)],
                    [(g, ok) for g in ("reprojection 2 mono", "reprojection 2 stereo") for ok in (True, False)]))
    return out


def _square_bound(chi):
    """(a, sigma^2): a float a of 10 fractional bits and a float sigma^2 with (float)(chi * sigma^2) == a * a exactly"""
    for k in range(int(math.sqrt(float(chi)) * 1024), 4096):
        a = k / 1024.0
        s0 = F32(a * a / float(chi))
        for s in _floats_around(s0, 3, 4):
            if float(F32(chi * s)) == a * a:
                return a, s
    raise AssertionError("no exact square bound")


def _exact_bound_problem(stereo):
    """The stereo-1 point (0, 0, 10) from a keypoint at the principal point; camera 2 one metre behind camera 1 on its axis
    reprojects it onto its principal point exactly.  Keyframe 2's keypoint x (mono) or x_right (stereo) is offset by a, so
    its squared error is a^2 == the float bound exactly, and by the floats on either side.  At the bound the pair passes
    (the gate rejects when bound < error)."""
    chi = R.CHI_SQ_3D if stereo else R.CHI_SQ_2D
    a, sig = _square_bound(chi)
    levels = 3
    sf, tab = tables(levels)
    tab = tab.copy(); tab[2] = sig
    v1 = View(np.eye(3), [0, 0, 0], levels=levels, sf=sf, sig=tab)
    v2 = View(np.eye(3), [0, 0, -1.0], levels=levels, sf=sf, sig=tab)
    d = 10.0
    for step in (-1, 0, 1):
        v1.add([0.0, 0.0, 1.0], CX, CY, 2, F32(CX - v1.camera.focal_x_baseline / d), F32(d))
        xr2 = F32(CX - v2.camera.focal_x_baseline / (d + 1.0))
        if stereo:
            off = F32(xr2 - F32(a))
            off = {-1: np.nextafter(off, F32(np.inf)), 0: off, 1: np.nextafter(off, F32(-np.inf))}[step]
            v2.add([0.0, 0.0, 1.0], CX, CY, 2, off, F32(d + 1.0))
        else:
            x = F32(CX + a)
            x = {-1: np.nextafter(x, F32(-np.inf)), 0: x, 1: np.nextafter(x, F32(np.inf))}[step]
            v2.add([0.0, 0.0, 1.0], x, CY, 2)
    return _problem(v1, v2)


# ------------------------------------------------------------------------------------------------ scale


def _scale_views(sf2=None, sig2=None, scale_factor=1.2, shift=0.0):
    levels = 1 if sf2 is None else len(sf2)
    ones = np.ones(max(levels, 1), F32)
    v1 = View(np.eye(3), [0, 0, 0], levels=1, sf=[1.0], sig=[1.0], scale_factor=scale_factor)
    v2 = View(rot_y(-3.0), [1.0, 0.0, 0.0], levels=levels, sf=ones if sf2 is None else sf2, sig=ones if sig2 is None else sig2)
    X = np.array([0.2 + shift, 0.1, 6.0])
    return v1, v2, X


def _ratio_dists(shift):
    v1, v2, X = _scale_views(shift=shift)
    v1.add_point(X); v2.add_point(X)
    kf1, kf2, pairs, _ = _problem(v1, v2)
    p = R.triangulate(kf1, kf2, pairs).pairs[0]
    d1 = np.linalg.norm(p.pos - 0.0); d2 = np.linalg.norm(p.pos - np.array([1.0, 0.0, 0.0]))
    return d2 / d1


def scale():
    out = []
    # keyframe 2's scale_factors entry stepped: ratio_octave = 1 / sf2 crosses ratio_dists * f (low) and ratio_dists / f (high)
    for side in ("low", "high"):
        for shift in np.arange(0.0, 0.05, 0.001):
            rd = _ratio_dists(shift)
            f = float(F32(F32(1.5) * F32(1.2)))
            target = 1.0 / (rd * f) if side == "low" else f / rd
            vals = _floats_around(target, 3, 3)
            v1, v2, X = _scale_views(sf2=vals, shift=shift)
            for o in range(len(vals)):
                v1.add_point(X); v2.add_point(X, octave=o)
            kf1, kf2, pairs, deg = _problem(v1, v2)
            res = R.triangulate(kf1, kf2, pairs, deg)
            k = _crossing(list(range(len(vals))), lambda j: bool(res.reason[j] == R.SCALE))
            if k is None or k < 1 or k + 2 >= len(vals):
                continue
            prob = (kf1, kf2, pairs[k - 1:k + 3], deg)
            if _clear(prob):
                break
        else:
            raise AssertionError("no clear crossing of the %s scale bound" % side)
        out.append(Case("scale: keyframe-2 scale_factors entry across the %s bound" % side, "scale", [prob], "scale " + side))
    # keyframe 1's scale_factor stepped: f = 1.5f * scale_factor crosses ratio_octave / ratio_dists (low) and
    # ratio_dists / ratio_octave (high), one problem per value; ratio_octave = 1 / 0.6 or 0.6
    for side, sf2 in (("low", F32(0.6)), ("high", F32(1.0 / 0.6))):
        for shift in np.arange(0.0, 0.05, 0.001):
            rd = _ratio_dists(shift)
            ro = float(F32(F32(1.0) / sf2))
            target = (ro / rd if side == "low" else rd / ro) / 1.5
            probs = []
            for s in _floats_around(target, 3, 3):
                v1, v2, X = _scale_views(sf2=[sf2], sig2=[1.0], scale_factor=float(s), shift=shift)
                v1.add_point(X); v2.add_point(X)
                probs.append(_problem(v1, v2))
            reasons = [R.triangulate(*p).reason[0] for p in probs]
            k = _crossing(list(range(len(probs))), lambda j: bool(reasons[j] == R.SCALE))
            if k is None or k < 1 or k + 2 >= len(probs):
                continue
            probs = probs[k - 1:k + 3]
            if all(_clear(p) for p in probs):
                break
        else:
            raise AssertionError("no clear crossing of the %s scale bound" % side)
        out.append(Case("scale: keyframe 1's scale_factor across the %s bound" % side, "scale", probs, "scale " + side))
    return out


# ------------------------------------------------------------------------------------------------ cheirality


def cheirality():
    out = []
    X = np.array([0.5, 0.2, -20.0])
    # two cameras, the point behind camera 1 (camera 2 looks along -z) and behind camera 2
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(R_Y180, [1.0, 0.0, 0.0])
    v1.add(*_bearing_of(v1, X), CX, CY); v2.add_point(X)
    w1, w2 = View(R_Y180, [0, 0, 0]), View(np.eye(3), [1.0, 0.0, 0.0])
    w1.add_point(X); w2.add(*_bearing_of(w2, X - np.array([1.0, 0.0, 0.0])), CX, CY)
    out.append(Case("cheirality: two cameras, behind camera 1 / behind camera 2", "cheirality", [_problem(v1, v2), _problem(w1, w2)],
                    [("cheirality 1", False), ("cheirality 2", False)], knife_edge=False))
    # stereo 1: behind camera 2 (camera 2 beyond the point), and behind camera 1 through a negative depth (the zero vector)
    d = 3.0
    Xs = np.array([0.1, 0.05, d])
    v1, v2 = View(np.eye(3), [0, 0, 0]), View(np.eye(3), [0.1, 0.0, 2 * d])
    v1.add_point(Xs, stereo=True); v2.add(*_bearing_of(v2, Xs - np.array([0.1, 0.0, 2 * d])), CX, CY)
    b1, u1, y1, z1 = v1.observe(Xs)
    v1.add(b1, u1, y1, 0, F32(100.0), F32(-1.0)); v2.add(b1, CX, CY)
    # stereo 2: behind camera 1, and behind camera 2 through a negative depth (camera 1 behind the origin)
    w1, w2 = View(np.eye(3), [0.1, 0.0, 2 * d]), View(np.eye(3), [0, 0, 0])
    w2.add_point(Xs, stereo=True); w1.add(*_bearing_of(w1, Xs - np.array([0.1, 0.0, 2 * d])), CX, CY)
    u1_, v1_ = View(np.eye(3), [0.0, 0.0, -5.0]), View(np.eye(3), [0, 0, 0])
    bb, uu, yy, zz = v1_.observe(Xs)
    u1_.add(bb, CX, CY); v1_.add(bb, uu, yy, 0, F32(100.0), F32(-1.0))
    out.append(Case("cheirality: stereo 1 and stereo 2, behind either camera", "cheirality",
                    [_problem(v1, v2), _problem(w1, w2), _problem(u1_, v1_)],
                    [("cheirality 1", False), ("cheirality 2", False), ("branch", "stereo 1"), ("branch", "stereo 2")], knife_edge=False))
    out.append(Case("cheirality: camera-1 z of 2^-150 (float 0) and the next double", "cheirality", _float_z_problems(), "cheirality 1"))
    return out


def _float_z_problems():
    """The stereo-2 point (0, 0, zeta) on camera 1's optical axis: camera 1 at the origin, camera 2 at (-D, 0, zeta) looking
    along +x, its keypoint at the principal point with depth D (the smallest float).  zeta = 2^-150 rounds to float 0, so
    (float)z > 0 rejects the point at camera 1; at the next double it rounds to 2^-149 and the pair makes a landmark: the
    point reprojects onto the principal point of both views (camera 2 has focal_x_baseline 0, so its right-image x is cx),
    and d2 / d1 = 2 is inside the scale bounds (octave 1 against octave 0).  Without the float cast both pairs would be
    valid, so this edge shows in `valid` alone.  (Off the optical axis, a camera-frame z this small puts the reprojection
    far outside the image and the reprojection gate rejects the pair whatever the cast does.)"""
    probs = []
    for zeta in (2.0 ** -150, float(np.nextafter(2.0 ** -150, 1.0))):
        v1 = View(np.eye(3), [0, 0, 0])
        v2 = View(R_Y90, [0, 0, 0], camera=perspective(fb=0.0))
        v2.pose = np.concatenate([R_Y90.reshape(9), [zeta, 0.0, float(TINY)]])    # -R c for c = (-D, 0, zeta), exact
        v1.add([0.0, 0.0, 1.0], CX, CY, octave=1)
        v2.add([0.0, 0.0, 1.0], CX, CY, 0, F32(CX), TINY)
        probs.append(_problem(v1, v2))
    return probs


# ------------------------------------------------------------------------------------------------ far stereo


def far_stereo(seed=5, n=600):
    """Both keypoints stereo (rig baseline 0.3 m), keyframes 0.5 m apart, depths 50 - 500 m: the two-camera branch at
    0.06 - 0.6 degrees of parallax; keypoints with 0.5 px noise (bearings from the noisy keypoints) so that the gates'
    margins spread."""
    rng = np.random.default_rng(seed)
    rig = 0.3
    cam = perspective(fb=FX * rig)
    v1 = View(np.eye(3), [0, 0, 0], cam, true_baseline=rig)
    v2 = View(rot_y(0.2), [0.5, 0.0, 0.0], cam, true_baseline=rig)
    sf, _ = tables(8)
    depth = np.exp(rng.uniform(math.log(50.0), math.log(500.0), n))
    u = rng.uniform(40, TP.COLS - 40, n); w = rng.uniform(40, TP.ROWS - 40, n)
    Xs = np.stack([(u - CX) / FX * depth, (w - CY) / FY * depth, depth], 1)
    for X in Xs:
        o = int(rng.integers(0, 3))
        for view in (v1, v2):
            b, uu, yy, z = view.observe(X)
            x, y = uu + rng.normal(0, 0.5) * sf[o], yy + rng.normal(0, 0.5) * sf[o]
            bb = np.array([(F32(x) - CX) / FX, (F32(y) - CY) / FY, 1.0]); bb /= np.linalg.norm(bb)
            view.add(bb, x, y, o, F32(uu - cam.focal_x_baseline / z + rng.normal(0, 0.3)), F32(z * (1 + rng.normal(0, 0.002))))
    return Case("far stereo: depths 50 - 500 m, two cameras at 0.06 - 0.6 degrees", "far_stereo", [_problem(v1, v2)], (), knife_edge=False)


# ------------------------------------------------------------------------------------------------ sizes


def sizes():
    """pair counts around the kernel's 128-thread block: single problems of 127, 128, 129 pairs, one batch of 128 k +- 1,
    and one batch of problems with 0, 1, 127 and 129 pairs"""
    single = [Case("sizes: M = %d" % m, "sizes", [TP.pair_problem(900 + m, m, "perspective", 0.5, 0.05) + (1.0,)], (), False)
              for m in (127, 128, 129)]
    batch = [TP.pair_problem(950 + k, 128 * (k // 2 + 2) + (1 if k % 2 else -1), "perspective", 0.5, 0.4) + (1.0,) for k in range(6)]
    mixed = [TP.pair_problem(970 + m, m, "perspective", 0.5, 0.4) + (1.0,) for m in (0, 1, 127, 129)]
    return single + [Case("sizes: one batch of 128 k +- 1", "sizes", batch, (), False),
                     Case("sizes: one batch of 0, 1, 127 and 129 pairs", "sizes", mixed, (), False)]


def knife_edge_cases():
    return parallax() + stereo_parallax() + reprojection() + scale() + cheirality()


def planar_neighbourhood(seed, n1, B):
    """every point on the plane of the camera centres and one descriptor per few hundred keypoints, in two nodes: every
    candidate of a query passes the epipolar test, so the 8-entry lists run out and the replay has to re-query"""
    rng = np.random.default_rng(seed)
    scene = TP.make_scene(rng, int(n1 * 1.3))
    scene["X"][:, 1] = 0.0
    base = rng.integers(0, 256, (3, 32), dtype=np.uint8)

    def kf(c):
        k, _ = TP.make_keyframe(rng, scene, c, np.eye(3), 0.0, 2, outlier_frac=0.0, noise_px=0.2)
        k.descriptors[:] = base[rng.integers(0, 3, k.num_keypts)]
        return k
    kf1 = TP._trim(kf(np.zeros(3)), n1)
    nbs = [kf(np.array([0.3 * (b + 1) * (-1) ** b, 0.0, 0.05 * b])) for b in range(B)]
    Es, eps = zip(*[TP.e12_epipole(kf1, n) for n in nbs])
    return kf1, nbs, np.array(Es), np.array(eps)


def uneven_neighbourhood(seed, n1=1500):
    """keyframe 1 and 5 neighbours whose unlisted (no landmark, in a node) keypoint counts differ greatly -- all, none,
    a few dozen, about half, a few hundred -- so that every neighbour's candidates start at a different offset"""
    kf1, nbs, E, ep = TP.neighbourhood(seed, n1, 5, stereo_frac=0.3)
    out = []
    for b, n in enumerate(nbs):
        has = n.has_landmark.copy()
        if b == 0:
            has[:] = 0
        elif b == 1:
            has[:] = 1
        elif b == 2:
            n = TP._trim(n, 40)
            has = np.zeros(n.num_keypts, np.uint8)
        elif b == 3:
            has = (np.arange(n.num_keypts) % 2).astype(np.uint8)
        else:
            n = TP._trim(n, 300)
            has = n.has_landmark.copy()
        out.append(module.keyframe(n.pose_cw, n.camera, n.scale_factor, n.scale_factors, n.level_sigma_sq, n.keypts["x"], n.keypts["y"],
                                   n.keypts["octave"], n.bearings, angle=n.keypts["angle"], stereo_x_right=n.stereo_x_right,
                                   depths=n.depths, true_baseline=n.true_baseline, descriptors=n.descriptors, has_landmark=has,
                                   bow_node=n.bow_node))
    return kf1, out, E, ep
