"""Seeded stereo rigs and map edge cases for the stereo rectification tests (oracle against cv2, library against the oracle).
Rotations and distortions are random; a rig's rectified camera matrix K_rect is slightly different from both cameras' K so
that part of each map falls outside the image."""
import numpy as np

# (model, cols, rows, seed) of tests/golden/rectify_golden.npz
GOLDEN_CASES = [("perspective", 1, 1, 11), ("perspective", 37, 23, 12), ("perspective", 61, 40, 13), ("fisheye", 1, 1, 21),
                ("fisheye", 37, 23, 22), ("fisheye", 61, 40, 23)]
SIZES = [(1, 1), (7, 5), (333, 97), (752, 480), (1241, 376), (1920, 1080)]   # widths 1, 7, 333, 1241: not multiples of 4


def rodrigues(v):
    v = np.asarray(v, np.float64)
    th = np.linalg.norm(v)
    if th == 0:
        return np.eye(3)
    k = v / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def rig(model, cols, rows, seed, rot=0.05):
    """-> dict(K_l, D_l, R_l, K_r, D_r, R_r, K_rect) of a random stereo rig for cols x rows images."""
    rng = np.random.default_rng(seed)
    f = max(cols, rows, 8) * rng.uniform(0.6, 0.9)

    def K():
        return np.array([[f * rng.uniform(0.97, 1.03), 0, cols / 2 + rng.normal(0, 2)],
                         [0, f * rng.uniform(0.97, 1.03), rows / 2 + rng.normal(0, 2)], [0, 0, 1]])

    def D():
        if model == "perspective":
            return np.array([rng.normal(0, 0.15), rng.normal(0, 0.05), rng.normal(0, 2e-3), rng.normal(0, 2e-3), rng.normal(0, 0.01)])
        return rng.normal(0, 0.03, 4)

    out = dict(K_l=K(), D_l=D(), R_l=rodrigues(rng.normal(0, rot, 3)), K_r=K(), D_r=D(), R_r=rodrigues(rng.normal(0, rot, 3)))
    out["K_rect"] = np.array([[f, 0, cols / 2], [0, f, rows / 2], [0, 0, 1]])
    return out


def identity_rig(model, cols, rows):
    """D = 0, R = I, K_rect = K: for the perspective model every map entry is its own pixel, so remap gives the input back."""
    K = np.array([[500.0, 0, (cols - 1) / 2], [0, 500.0, (rows - 1) / 2], [0, 0, 1]])
    D = np.zeros(5 if model == "perspective" else 4)
    return dict(K_l=K, D_l=D, R_l=np.eye(3), K_r=K.copy(), D_r=D.copy(), R_r=np.eye(3), K_rect=K.copy())


def edge_maps(cols, rows, seed):
    """Maps of cols x rows holding every value class remap has to saturate or round: in range, partly and fully outside,
    the half-1/64 ties (rounded to even), values whose product with 32 leaves int, +-FLT_MAX, +-inf and NaN."""
    rng = np.random.default_rng(seed)
    n = cols * rows
    fmax = np.finfo(np.float32).max
    special = np.array([np.nan, np.inf, -np.inf, fmax, -fmax, 1e9, -1e9, 6.7e7, -6.7e7, 1e6, -1e6, 40000.0, -40000.0, 32767.0,
                        -32768.0, -1.0, -0.5, -1.0 / 64, cols - 1, cols - 0.5, cols, cols + 1.0 / 64, rows - 1, rows], np.float32)
    ties = (rng.integers(-2, max(cols, rows) + 2, n) + (2 * rng.integers(0, 32, n) + 1) / 64.0).astype(np.float32)
    inside_x = rng.uniform(-1.5, cols + 0.5, n).astype(np.float32)
    inside_y = rng.uniform(-1.5, rows + 0.5, n).astype(np.float32)
    pick = rng.integers(0, 4, n)
    mx = np.where(pick == 0, ties, np.where(pick == 1, special[rng.integers(0, len(special), n)], inside_x)).astype(np.float32)
    pick = rng.integers(0, 4, n)
    ties_y = (rng.integers(-2, rows + 2, n) + (2 * rng.integers(0, 32, n) + 1) / 64.0).astype(np.float32)
    my = np.where(pick == 0, ties_y, np.where(pick == 1, special[rng.integers(0, len(special), n)], inside_y)).astype(np.float32)
    return mx.reshape(rows, cols), my.reshape(rows, cols)


def image(cols, rows, channels, seed):
    rng = np.random.default_rng(seed)
    shape = (rows, cols) if channels == 1 else (rows, cols, channels)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def ulp_distance(a, b):
    """Per-entry distance in float32 ulps (0 where the bits are equal, NaN == NaN)."""
    ai = a.view(np.int32).astype(np.int64); bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai); bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.where(a.view(np.uint32) == b.view(np.uint32), 0, np.abs(ai - bi))
