"""Scenes and hand-made keypoints for match::stereo::compute that reach every branch of the matcher
(tests/stereo_reference.py names them): rows, octave, x and Hamming gates at their knife edges, the SAD windows at the
borders of every pyramid level, the sub-pixel branches, the median test, the launch geometry's size boundaries and
non-finite coordinates.

A case is a dict: scene (the name of an image pair, see scene()), kl / dl and kr / dr (keypoints with fields x, y,
octave and 32-byte descriptors), fxb and baseline, and `expect`, the reasons the case exists to reach.  The matcher runs
on the pyramids of the scene's images; the keypoints are made here (the ABI takes any keypoint arrays), apart from the
sub-pixel scenes, which use the extractor's own.  All images are 1241 x 376 (KITTI): every pyramid level's device row
pitch (the width rounded up to 128 bytes) differs from its width."""
import functools

import numpy as np

from openvslam_b200 import synth

f32 = np.float32
KP = np.dtype([("x", "<f4"), ("y", "<f4"), ("octave", "<i4")])
COLS, ROWS, LEVELS = 1241, 376, 8
FXB, BASELINE = 386.1448, 0.5372           # bench config 3's camera: max_disp = 718.8
SHIFT = 3                                  # disparity of the "shift" scene
PLANE_D0, PLANE_A = 20.0, 0.02             # disparity plane of the "plane" scene: d(x_left) = d0 + a x_left


def scale_factors():
    s = [f32(1.0)]
    for _ in range(1, LEVELS):
        s.append(f32(s[-1] * f32(1.2)))
    return np.array(s, f32)


def level_sizes():
    from oracle import oracle as O
    return O.level_sizes(COLS, ROWS, 1.2, LEVELS)


def _symmetric_patch(rng, h, w):
    half = rng.integers(30, 220, (h, w // 2 + 1))
    return np.concatenate([half[:, :0:-1], half], 1)[:, :w].astype(np.uint8)   # p[:, c + k] == p[:, c - k], c = w // 2


def _stripes(h, w):
    return np.where(np.arange(w)[None, :] % 2 == 0, 60, 180).repeat(h, 0).astype(np.uint8)


SYM_AT = (300, 100)        # (x, y) centre of the mirror-symmetric patch, present in both images of "shift"
STRIPES_AT = (700, 100)    # centre of the period-2 stripes, present in both images of "shift"


@functools.lru_cache(maxsize=None)
def scene(name):
    """-> (left, right) u8 images.
    plane:    right resampled (bilinear, float64) from the left with disparity d0 + a x_left, plus integer noise in [-2, 2];
    shift:    right = left shifted by SHIFT px plus noise in [-2, 2], with a mirror-symmetric patch and period-2 stripes
              pasted at the same place in both (zero disparity there);
    exact:    right = left shifted by SHIFT px, no noise (the median cases perturb single pixels of it);
    same:     right = left."""
    if name == "plane":
        left = synth.frame(COLS, ROWS, seed=31)
        xr = np.arange(COLS, dtype=np.float64)
        xl = (xr + PLANE_D0) / (1.0 - PLANE_A)          # x_left - d(x_left) = x_right
        i0 = np.clip(np.floor(xl).astype(np.int64), 0, COLS - 2)
        t = np.clip(xl - i0, 0.0, 1.0)
        L = left.astype(np.float64)
        right = L[:, i0] * (1 - t) + L[:, i0 + 1] * t
        right = np.clip(np.rint(right) + np.random.default_rng(5).integers(-2, 3, right.shape), 0, 255).astype(np.uint8)
        return left, right
    left = synth.frame(COLS, ROWS, seed={"shift": 32, "exact": 33, "same": 34}[name])
    if name == "same":
        return left, left.copy()
    right = np.roll(left, -SHIFT, axis=1)
    if name == "shift":
        right = np.clip(right.astype(np.int16) + np.random.default_rng(6).integers(-2, 3, right.shape), 0, 255).astype(np.uint8)
        sym = _symmetric_patch(np.random.default_rng(7), 31, 31)
        st = _stripes(31, 41)
        for img in (left, right):
            x, y = SYM_AT; img[y - 15:y + 16, x - 15:x + 16] = sym
            x, y = STRIPES_AT; img[y - 15:y + 16, x - 20:x + 21] = st
    return left, np.ascontiguousarray(right)


def at_level(target, level, sf=None):
    """A float32 level-0 coordinate whose rint(float32(c * inv_s[level])) is `target`, as close to target * s as possible."""
    sf = scale_factors() if sf is None else sf
    inv = f32(f32(1.0) / sf[level])
    c0 = f32(target * float(sf[level]))
    for k in range(200):
        for c in (f32(c0 + f32(0.01) * k), f32(c0 - f32(0.01) * k)):
            if np.rint(f32(c * inv)) == target:
                return f32(c)
    raise AssertionError((target, level))


def band_edge_y(row, r, upper):
    """A right y on the knife edge of the row band [floor(y - r), ceil(y + r)]: float32(y - r) == row + 1 (upper) or
    float32(y + r) == row - 1 (not upper), so that the band just misses `row`."""
    target = f32(row + 1) if upper else f32(row - 1)
    y = f32(target + r) if upper else f32(target - r)
    for _ in range(64):
        v = f32(y - r) if upper else f32(y + r)
        if v == target:
            return y
        y = np.nextafter(y, -np.inf if v > target else np.inf, dtype=f32)
    raise AssertionError((row, r, upper))


class _Builder:
    """Left probes, each with its own random descriptor, and right keypoints whose descriptors are a probe's XOR-ed with
    exactly k bits (random descriptors are ~128 bits from any other, so probes do not see each other's right keypoints)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.L, self.Ld, self.R, self.Rd = [], [], [], []

    def left(self, x, y, octave):
        self.L.append((x, y, octave)); self.Ld.append(self.rng.integers(0, 256, 32, dtype=np.uint8))
        return len(self.L) - 1

    def flipped(self, probe, k):
        d = self.Ld[probe].copy()
        bits = self.rng.choice(256, k, replace=False)
        for b in bits:
            d[b >> 3] ^= np.uint8(1 << (b & 7))
        return d

    def right(self, probe, x, y, octave, k=10):
        self.R.append((x, y, octave)); self.Rd.append(self.flipped(probe, k))
        return len(self.R) - 1

    def filler(self, n):
        """n right keypoints with random descriptors, spread over the image."""
        x = self.rng.uniform(20, COLS - 20, n).astype(f32); y = self.rng.uniform(20, ROWS - 20, n).astype(f32)
        o = self.rng.integers(0, LEVELS, n); d = self.rng.integers(0, 256, (n, 32), dtype=np.uint8)
        self.R.extend(zip(x, y, o)); self.Rd.extend(d)

    def case(self, name, scene_name, expect, fxb=FXB, baseline=BASELINE):
        return dict(name=name, scene=scene_name, kl=_kp(self.L), dl=_desc(self.Ld), kr=_kp(self.R), dr=_desc(self.Rd),
                    fxb=fxb, baseline=baseline, expect=set(expect))


def _kp(rows):
    a = np.zeros(len(rows), KP)
    if rows:
        x, y, o = zip(*rows)
        a["x"], a["y"], a["octave"] = x, y, o
    return a


def _desc(rows):
    return np.array(rows, np.uint8).reshape(-1, 32)


def _extracted(img, nkp=2000):
    from oracle import oracle as O
    k, d, _ = O.extract(img, O.params(nkp))
    a = np.zeros(len(k), KP)
    a["x"], a["y"], a["octave"] = k["x"], k["y"], k["octave"]
    return a, d


# ------------------------------------------------------------------------------------------------------------------ cases
def plane_case():
    left, right = scene("plane")
    kl, dl = _extracted(left); kr, dr = _extracted(right)
    return dict(name="plane", scene="plane", kl=kl, dl=dl, kr=kr, dr=dr, fxb=FXB, baseline=BASELINE, expect={"matched"})


def bench_case():
    import bench
    cfg = bench.CONFIGS[3]
    wl = bench.make_workload(cfg, 0, 6)
    left, right = wl["frames"][0], wl["frames_right"][0]
    kl, dl = _extracted(left, cfg["NKP"]); kr, dr = _extracted(right, cfg["NKP"])
    fxb = wl["pose"]["cam"]["focal_x_baseline"]
    return dict(name="bench_config3", scene=("bench", left, right), kl=kl, dl=dl, kr=kr, dr=dr, fxb=fxb,
                baseline=fxb / wl["pose"]["cam"]["fx"], expect={"matched", "median_rejected"})


def gates_case():
    """Rows, octaves, Hamming distances and the row band at every octave, on the shifted pair (true match SHIFT px left)."""
    sf = scale_factors()
    b = _Builder(1)
    x0 = f32(600.25)
    for y in (-1.0, -0.5, ROWS - 1, ROWS, ROWS - 0.5):                 # int(y): -1 out, 0 in, rows0 - 1 in, rows0 out
        p = b.left(x0, f32(y), 0); b.right(p, x0 - SHIFT, f32(max(y, 0.0)), 0)
    for o in (1, 2, 4, 5):                                              # octave gate |o_r - o_l| <= 1 around o_l = 3
        p = b.left(x0, f32(180.5), 3); b.right(p, x0 - SHIFT, f32(180.5), o)
    for k in (74, 75):                                                  # Hamming threshold: < 75
        p = b.left(x0, f32(150.5), 0); b.right(p, x0 - SHIFT, f32(150.5), 0, k=k)
    row = 188
    for o in range(LEVELS):                                             # the row band [floor(y - 2 s), ceil(y + 2 s)]
        r = f32(f32(2.0) * sf[o])
        x = f32(420.0 + 90.0 * o)
        for upper in (True, False):
            y = band_edge_y(row, r, upper)
            p = b.left(x, f32(row + 0.5), o); b.right(p, x - SHIFT, y, o)                        # just misses the row
            p = b.left(x, f32(row + 0.5), o)
            b.right(p, x - SHIFT, np.nextafter(y, -np.inf if upper else np.inf, dtype=f32), o)   # one ulp inside
    # ties go to the lower right index: the first candidate is the true match, the second (same distance) 5 px off
    p = b.left(x0, f32(120.5), 0); b.right(p, x0 - SHIFT, f32(120.5), 0, k=20); b.right(p, x0 - SHIFT - 5, f32(120.5), 0, k=20)
    return b.case("gates", "shift", {"row_outside", "no_candidate_below_threshold", "matched"})


def xgate_case():
    """The x window [x_left - max_disp, x_left] at both ends and one float32 ulp outside, max_disp = 13 / 4 = 3.25."""
    b = _Builder(2)
    for x in (400.25, 777.75, 901.0):
        lo, hi = f32(f32(x) - f32(3.25)), f32(x)
        for xr in (lo, np.nextafter(lo, -np.inf, dtype=f32), hi, np.nextafter(hi, np.inf, dtype=f32)):
            p = b.left(f32(x), f32(200.5), 0); b.right(p, xr, f32(200.5), 0)
    p = b.left(f32(-0.0), f32(200.5), 0); b.right(p, f32(0.0), f32(200.5), 0)           # max_x_right = -0: not negative
    p = b.left(f32(-1e-6), f32(200.5), 0); b.right(p, f32(-1e-6), f32(200.5), 0)        # max_x_right < 0
    return b.case("xgate", "shift", {"no_candidate_below_threshold", "matched", "max_x_right_negative", "right_window_outside"},
                  fxb=13.0, baseline=4.0)


def max_disp_case():
    """max_disp = 3 on a disparity-3 pair: refined disparities fall on both sides of it."""
    b = _Builder(3)
    rng = np.random.default_rng(30)
    for _ in range(60):
        x = f32(rng.integers(40, COLS - 40)); y = f32(rng.integers(20, ROWS - 20) + 0.5)
        p = b.left(x, y, 0); b.right(p, x - SHIFT, y, 0)
    return b.case("max_disp", "shift", {"disparity_out_of_range", "matched"}, fxb=12.0, baseline=4.0)


def borders_case():
    """The SAD windows at the borders of every level: sxl, syl at 4 / 5 and W - 6 / W - 5 (H likewise), the right windows
    at ini_x = 0 / -1 and end_x = W - 1 / W, and half-integer level-0 coordinates (round half to even)."""
    sf = scale_factors()
    sizes = level_sizes()
    b = _Builder(4)
    for lvl in range(LEVELS):
        W, H = sizes[lvl]
        xc, yc = at_level(W // 2, lvl), at_level(H // 2, lvl)
        for t in (4, 5, H - 6, H - 5):                        # syl
            y = at_level(t, lvl); p = b.left(xc, y, lvl); b.right(p, xc - SHIFT, y, lvl)
        for t in (4, 5, W - 6, W - 5):                        # sxl; the right keypoint 7 level px left of it
            x = at_level(t, lvl); p = b.left(x, yc, lvl); b.right(p, at_level(t - 7, lvl), yc, lvl)
        for t in (9, 10, W - 12, W - 11):                     # sxr: ini_x = -1 / 0, end_x = W - 1 / W
            xr = at_level(t, lvl); p = b.left(f32(xr + SHIFT), yc, lvl); b.right(p, xr, yc, lvl)
    W, H = sizes[0]
    for y in (4.5, 5.5, H - 6.5, H - 5.5, H - 6.0 + 0.5):     # rint: 4, 6, 370, 370, 370 (half to even)
        p = b.left(f32(600.0), f32(y), 0); b.right(p, f32(600.0 - SHIFT), f32(y), 0)
    for x in (600.5, 601.5, W - 6.5, W - 5.5):
        p = b.left(f32(x), f32(200.0), 0); b.right(p, f32(x - SHIFT - 4), f32(200.0), 0)
    for xr in (8.5, 9.5, 10.5, W - 12.5, W - 11.5):
        p = b.left(f32(xr + SHIFT), f32(200.0), 0); b.right(p, f32(xr), f32(200.0), 0)
    return b.case("borders", "shift", {"left_window_outside", "right_window_outside", "matched"})


def subpixel_case():
    """A right keypoint 5 level px off the true match (best offset at the edge), the mirror-symmetric patch at zero
    disparity (c1 == c3, delta = 0, disparity 0 clamped to 0.01) and the period-2 stripes (equal minima: the first wins)."""
    b = _Builder(5)
    for lvl in (0, 2, 5):
        x, y = f32(500.0), f32(250.5)
        p = b.left(x, y, lvl); b.right(p, at_level(int(np.rint(f32((x - SHIFT) / scale_factors()[lvl]))) - 5, lvl), y, lvl)
        p = b.left(x, y, lvl); b.right(p, at_level(int(np.rint(f32((x - SHIFT) / scale_factors()[lvl]))) + 5, lvl), y, lvl)
    x, y = SYM_AT
    p = b.left(f32(x), f32(y), 0); b.right(p, f32(x), f32(y), 0)
    x, y = STRIPES_AT
    p = b.left(f32(x), f32(y), 0); b.right(p, f32(x), f32(y), 0)
    rng = np.random.default_rng(50)                          # ordinary matches, so the median SAD is not 0
    for _ in range(30):
        x = f32(rng.integers(40, COLS - 40) + 0.25); y = f32(rng.integers(20, ROWS - 20) + 0.5)
        if abs(x - SYM_AT[0]) < 40 or abs(x - STRIPES_AT[0]) < 40:
            continue
        p = b.left(x, y, 0); b.right(p, x - SHIFT, y, 0)
    return b.case("subpixel", "shift", {"best_offset_at_edge", "clamped_zero_disparity", "matched"})


def median_case(sads, seed):
    """Matches on the noise-free shifted pair whose best SADs are exactly `sads`: one right pixel of each window (not the
    centre) is changed by the SAD wanted.  The images are perturbed per case (scene ("exact", perturbations))."""
    left, right = scene("exact")
    right = right.copy()
    b = _Builder(seed)
    for k, s in enumerate(sads):
        x, y = 60 + 40 * k, 60 + 60 * (k % 4)
        p = b.left(f32(x), f32(y + 0.5), 0); b.right(p, f32(x - SHIFT), f32(y + 0.5), 0)
        px, py = x - SHIFT + 2, y + 3
        v = int(right[py, px])
        right[py, px] = v + s if v + s <= 255 else v - s
    return dict(name="median_%d" % len(sads), scene=("median_%d" % seed, left, right), kl=_kp(b.L), dl=_desc(b.Ld), kr=_kp(b.R),
                dr=_desc(b.Rd), fxb=FXB, baseline=BASELINE, expect={"matched", "median_rejected"}, sads=sorted(sads))


def same_case():
    """An identical pair: every SAD at the match is 0, so is the median, and the median test rejects every match."""
    left, _ = scene("same")
    kl, dl = _extracted(left, 500)
    return dict(name="identical_pair", scene="same", kl=kl, dl=dl, kr=kl.copy(), dr=dl.copy(), fxb=FXB, baseline=BASELINE,
                expect={"median_rejected"})


def seam_case(n_left, n_right, winners=()):
    """n_left probes on the shifted pair against n_right right keypoints: fillers, and each probe's true match placed at the
    end of the right list (or at the indices `winners`), with an equally distant decoy 5 px off at the index after it."""
    b = _Builder(1000 + n_left * 7 + n_right)
    rng = np.random.default_rng(n_left + 3 * n_right)
    probes = [b.left(f32(rng.integers(40, COLS - 40) + 0.5), f32(rng.integers(20, ROWS - 20) + 0.5), 0) for _ in range(n_left)]
    slots = {}
    if winners:
        for p, w in zip(probes, winners):
            slots[w] = (p, True); slots[w + 1] = (p, False)
    else:
        for k, p in enumerate(probes[-n_right:] if n_right else []):
            slots[n_right - min(n_left, n_right) + k] = (p, True)
    b.filler(n_right)
    for i, (p, true) in slots.items():
        x, y, _ = b.L[p]
        b.R[i] = (f32(x - SHIFT - (0 if true else 5)), y, 0); b.Rd[i] = b.flipped(p, 20)
    return b.case("sizes_%d_%d%s" % (n_left, n_right, "_seams" if winners else ""), "shift", set())


def nonfinite_case():
    """Non-finite and out-of-image coordinates on either side; every such left keypoint comes back -1, and a right keypoint
    with such a coordinate is no candidate (the true match behind it, at a higher index, wins)."""
    b = _Builder(7)
    bad = (np.nan, np.inf, -np.inf, 1e10, -1e10, 2.0 ** 32 + 512, -(2.0 ** 32) + 512)
    for v in bad:
        p = b.left(f32(v), f32(200.5), 0); b.right(p, f32(v), f32(200.5), 0)
        p = b.left(f32(600.5), f32(v), 0); b.right(p, f32(600.5 - SHIFT), f32(v), 0)
        p = b.left(f32(v), f32(v), 3); b.right(p, f32(v), f32(v), 3)
    for v in bad:
        p = b.left(f32(650.25), f32(0.5), 0); b.right(p, f32(650.25 - SHIFT), f32(v), 0, k=5)     # y = NaN: no row 0
        p = b.left(f32(650.25), f32(210.5), 0)
        b.right(p, f32(v), f32(210.5), 0, k=5); b.right(p, f32(650.25 - SHIFT), f32(210.5), 0, k=20)
        p = b.left(f32(650.25), f32(230.5), 0)
        b.right(p, f32(650.25 - SHIFT), f32(v), 0, k=5); b.right(p, f32(650.25 - SHIFT), f32(230.5), 0, k=20)
    return b.case("non_finite", "shift", {"not_finite", "row_outside", "matched"}, fxb=2.0 ** 40, baseline=1.0)


SIZES_LEFT = (0, 1, 3, 4, 5, 127, 128, 129)
SIZES_RIGHT = (0, 1, 255, 256, 257, 511, 512, 513)


def size_cases():
    out = [seam_case(nl, nr) for nl in SIZES_LEFT for nr in SIZES_RIGHT]
    out.append(seam_case(4, 520, winners=(255, 511)))                  # equal distances at 255 / 256 and 511 / 512
    out.append(seam_case(2, 65534, winners=(65532,)))                  # the largest right set: the decoy at 65533
    c = seam_case(1, 65534); c["name"] = "sizes_1_65534_last"          # the winner at index 65533
    out.append(c)
    return out


def all_cases():
    return ([plane_case(), bench_case(), gates_case(), xgate_case(), max_disp_case(), borders_case(), subpixel_case(),
             median_case([30, 30, 40, 40, 40, 80, 80], 8), median_case([10, 20, 20, 20, 40, 41], 9),
             median_case([25, 25, 25, 50, 25, 12, 50, 49, 60], 10), same_case(), nonfinite_case()]
            + size_cases())


def images(case):
    s = case["scene"]
    return scene(s) if isinstance(s, str) else (s[1], s[2])


def scene_key(case):
    s = case["scene"]
    return s if isinstance(s, str) else s[0]
