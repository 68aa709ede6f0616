"""util::stereo_rectifier on the device against the rectification oracle (oracle/rectify_oracle.c, itself pinned against cv2):
the maps, ovs_stereo_rectify_host, ovs_extract_host_rectified (keypoints, descriptors, pyramid level 0, launches, host waits,
threads) and the stereo chain rectify -> extract -> match::stereo; and the argument checks of the C ABI."""
import ctypes as C
import threading

import numpy as np
import pytest

import rectify_cases as RC
from openvslam_b200 import _lib, synth

pytestmark = pytest.mark.gpu


def _waits():
    f = _lib.lib().ovs_host_wait_count
    f.restype = C.c_uint64
    return int(f())


@pytest.fixture(scope="module")
def RO(oracle):
    from oracle import rectify
    return rectify


def _rectifier(model, cols, rows, r):
    from openvslam_b200 import util
    return util.stereo_rectifier(cols, rows, r["K_rect"], r["K_l"], r["D_l"], r["R_l"], r["K_r"], r["D_r"], r["R_r"], model=model)


def _oracle_maps(RO, model, cols, rows, r, side):
    s = "lr"[side]
    return RO.init_rectify_map(model, cols, rows, r["K_" + s], r["D_" + s], r["R_" + s], r["K_rect"])


def _check_maps(RO, rect, model, cols, rows, r):
    for side in (0, 1):
        gx, gy = rect.maps(side)
        ox, oy = _oracle_maps(RO, model, cols, rows, r, side)
        d = np.maximum(RC.ulp_distance(gx, ox), RC.ulp_distance(gy, oy))
        if model == "perspective":
            assert d.max() == 0, "%d perspective map entries differ" % int((d > 0).sum())
        else:
            assert d.max() <= 1 and (d == 0).mean() > 0.999, (int((d > 0).sum()), int(d.max()))


CASES = [(m, c, r, 0.1) for m in ("perspective", "fisheye") for (c, r) in RC.SIZES] + \
        [("perspective", 160, 120, 1.2), ("fisheye", 160, 120, 1.2)]   # strong rotations: huge, infinite map entries


@pytest.mark.parametrize("model,cols,rows,rot", CASES)
def test_maps_and_rectify_host(RO, model, cols, rows, rot):
    r = RC.rig(model, cols, rows, seed=cols * 7 + rows, rot=rot)
    rect = _rectifier(model, cols, rows, r)
    _check_maps(RO, rect, model, cols, rows, r)
    for ch in (1, 3, 4):
        il, ir = RC.image(cols, rows, ch, 1 + ch), RC.image(cols, rows, ch, 11 + ch)
        ol, orr = rect.rectify(il, ir)
        for side, (img, out) in enumerate(((il, ol), (ir, orr))):
            assert np.array_equal(out, RO.remap(img, *rect.maps(side))), (side, ch)
            if model == "perspective":
                assert np.array_equal(out, RO.remap(img, *_oracle_maps(RO, model, cols, rows, r, side))), (side, ch)
    rect.close()


@pytest.mark.parametrize("cols,rows", [(7, 5), (752, 480)])
def test_identity_rectification(cols, rows):
    r = RC.identity_rig("perspective", cols, rows)
    rect = _rectifier("perspective", cols, rows, r)
    for ch in (1, 3, 4):
        il, ir = RC.image(cols, rows, ch, ch), RC.image(cols, rows, ch, 5 + ch)
        ol, orr = rect.rectify(il, ir)
        assert np.array_equal(ol, il) and np.array_equal(orr, ir)
    rect.close()


def _colour(gray, order, channels):
    """A colour image whose gray conversion carries the structure of `gray`."""
    rng = np.random.default_rng(int(gray[0, 0]) + channels)
    c = np.stack([gray, np.clip(gray.astype(np.int16) + rng.integers(-20, 21, gray.shape), 0, 255).astype(np.uint8),
                  255 - gray], axis=2)
    if channels == 4:
        c = np.concatenate([c, rng.integers(0, 256, gray.shape + (1,), dtype=np.uint8)], axis=2)
    return np.ascontiguousarray(c)


def _extractor(n=1000):
    from openvslam_b200 import feature
    return feature.orb_extractor(feature.orb_params(max_num_keypts=n))


def _same(a, b):
    (ka, da), (kb, db) = a, b
    assert len(ka) == len(kb) and len(ka) > 0
    assert np.array_equal(ka.view(np.uint8), kb.view(np.uint8)) and np.array_equal(da, db)


@pytest.mark.parametrize("model", ["perspective", "fisheye"])
@pytest.mark.parametrize("channels,order", [(1, "BGR"), (3, "BGR"), (3, "RGB"), (4, "BGR")])
@pytest.mark.parametrize("masked", [False, True])
def test_extract_host_rectified(RO, model, channels, order, masked):
    cols, rows = 752, 480
    r = RC.rig(model, cols, rows, seed=5, rot=0.02)
    rect = _rectifier(model, cols, rows, r)
    gray = synth.frame(cols, rows, seed=8)
    raw = gray if channels == 1 else _colour(gray, order, channels)
    mask = None
    if masked:
        mask = np.ones((rows, cols), np.uint8); mask[:, :200] = 0
    ext, ref = _extractor(), _extractor()
    for side in (0, 1):
        fixed = RO.remap(raw, *rect.maps(side))      # what a user feeds ovs_extract_host / _color today: the remapped image
        want = ref.extract(fixed, mask, color_order=order)
        got = ext.extract(raw, mask, color_order=order, rectifier=rect, side=side)   # the first call also sizes the handle
        _same(got, want)
        assert np.array_equal(ext.image_pyramid(0), ref.image_pyramid(0))
        l0 = _lib.launch_count(); w0 = _waits()
        _same(ext.extract(raw, mask, color_order=order, rectifier=rect, side=side), got)   # repeatable
        launches, waits = _lib.launch_count() - l0, _waits() - w0
        l0 = _lib.launch_count(); w0 = _waits()
        ref.extract(fixed, mask, color_order=order)
        ref_launches, ref_waits = _lib.launch_count() - l0, _waits() - w0
        # colour: the fused remap replaces the colour conversion; gray: the remap is the one launch more than a plain upload
        assert launches == ref_launches + (1 if channels == 1 else 0)
        assert waits == ref_waits == 1
    # a plain extract on the same handle is unchanged afterwards
    _same(ext.extract(gray), ref.extract(gray))
    ext.close(); ref.close(); rect.close()


def test_two_threads_share_one_rectifier(RO):
    cols, rows = 752, 480
    r = RC.rig("perspective", cols, rows, seed=6, rot=0.02)
    rect = _rectifier("perspective", cols, rows, r)
    imgs = [_colour(synth.frame(cols, rows, seed=20 + s), "BGR", 3) for s in (0, 1)]
    exts = [_extractor(), _extractor()]
    want = [exts[s].extract(imgs[s], rectifier=rect, side=s) for s in (0, 1)]
    got = [[None] * 10, [None] * 10]

    def run(s):
        for k in range(10):
            got[s][k] = exts[s].extract(imgs[s], rectifier=rect, side=s)
    th = [threading.Thread(target=run, args=(s,)) for s in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for s in (0, 1):
        for g in got[s]:
            _same(g, want[s])
    for e in exts:
        e.close()
    rect.close()


def test_stereo_chain_equals_oracle(RO, oracle):
    from openvslam_b200 import match
    cols, rows = 752, 480
    r = RC.rig("perspective", cols, rows, seed=9, rot=0.01)
    rect = _rectifier("perspective", cols, rows, r)
    left = synth.frame(cols, rows, seed=31)
    right = np.ascontiguousarray(np.roll(left, -12, axis=1))
    el, er = _extractor(), _extractor()
    kl, dl = el.extract(left, rectifier=rect, side=0)
    kr, dr = er.extract(right, rectifier=rect, side=1)
    xr, dp, nm = match.stereo().compute(el, er, kl, dl, kr, dr, 386.1448, 0.5372)
    P = oracle.params(1000)
    ol, orr = RO.rectify("perspective", r["K_l"], r["D_l"], r["R_l"], r["K_r"], r["D_r"], r["R_r"], r["K_rect"], left, right)
    okl, odl, _ = oracle.extract(ol, P); okr, odr, _ = oracle.extract(orr, P)
    for f in ("x", "y", "angle", "response", "octave"):
        assert np.array_equal(kl[f], okl[f]) and np.array_equal(kr[f], okr[f]), f
    assert np.array_equal(dl, odl) and np.array_equal(dr, odr)
    oxr, odp, onm = oracle.stereo_compute(oracle.build_pyramid(ol, P), oracle.build_pyramid(orr, P), oracle.scale_factors(1.2, 8),
                                          kl, dl, kr, dr, 386.1448, 0.5372)
    assert nm == onm and nm > 100
    assert np.array_equal(xr.view(np.uint32), oxr.view(np.uint32)) and np.array_equal(dp.view(np.uint32), odp.view(np.uint32))
    el.close(); er.close(); rect.close()


def test_invalid_arguments_launch_nothing():
    L = _lib.lib()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    K = np.array([[300.0, 0, 40], [0, 300.0, 30], [0, 0, 1]]); D = np.zeros(5); R = np.eye(3)
    h = C.c_void_p()
    l0 = _lib.launch_count()
    create = lambda model=0, cols=80, rows=60, Kr=K, D_l=D: L.ovs_stereo_rectifier_create(
        0, model, cols, rows, vp(K), vp(D_l) if D_l is not None else None, vp(R), vp(K), vp(D), vp(R), vp(Kr), C.byref(h))
    assert create(model=1) == -1 and create(model=3) == -1               # equirectangular, radial division
    assert create(D_l=None) == -1 and create(cols=0) == -1 and create(rows=40000) == -1
    assert create(Kr=np.zeros((3, 3))) == -1                               # singular K_rect R
    assert _lib.launch_count() == l0
    from openvslam_b200 import util
    rect = util.stereo_rectifier(80, 60, K, K, D, R, K, D, R)
    ext = _extractor(200)
    img = np.zeros((60, 80), np.uint8); big = np.zeros((61, 80), np.uint8)
    kps = np.zeros(ext._cap, np.dtype((np.void, 28))); desc = np.zeros((ext._cap, 32), np.uint8); n = C.c_int()
    out = np.zeros_like(img)

    def extract(rectifier=rect._h, side=0, image=img, channels=1, order=0, w=80, hgt=60, pitch=80, num=C.byref(n)):
        return L.ovs_extract_host_rectified(ext._h, rectifier, side, vp(image) if image is not None else None, w, hgt, C.c_size_t(pitch),
                                            channels, order, None, C.c_size_t(0), vp(kps), vp(desc), ext._cap, num)
    l0 = _lib.launch_count(); w0 = _waits()
    assert extract(side=2) == -1 and extract(side=-1) == -1
    assert extract(channels=2) == -1 and extract(channels=5) == -1
    assert extract(image=big, hgt=61) == -1 and extract(w=79, pitch=80) == -1
    assert extract(rectifier=None) == -1 and extract(image=None) == -1 and extract(num=None) == -1
    assert extract(order=7, channels=3, pitch=240) == -1
    assert L.ovs_stereo_rectify_host(rect._h, vp(img), vp(img), 80, 60, C.c_size_t(80), 2, vp(out), vp(out), C.c_size_t(80)) == -1
    assert L.ovs_stereo_rectify_host(rect._h, vp(big), vp(big), 80, 61, C.c_size_t(80), 1, vp(out), vp(out), C.c_size_t(80)) == -1
    assert L.ovs_stereo_rectify_host(rect._h, None, vp(img), 80, 60, C.c_size_t(80), 1, vp(out), vp(out), C.c_size_t(80)) == -1
    mx = np.zeros((60, 80), np.float32)
    assert L.ovs_stereo_rectifier_maps(rect._h, 2, vp(mx), vp(mx)) == -1
    assert _lib.launch_count() == l0 and _waits() == w0
    # a rectifier on another device than the extractor: only checkable with two devices
    ext.close(); rect.close()
