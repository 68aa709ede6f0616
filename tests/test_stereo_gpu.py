"""match::stereo::compute on the device (k_stereo_match + k_stereo_subpixel, csrc/match_window.cu) against the oracle and
the numpy restatement of tests/stereo_reference.py, bit for bit, on every scene of tests/stereo_cases.py: the knife
edges of the gates, the window borders of every pyramid level, the sub-pixel branches, the median test, the shared-memory
tile and CTA boundaries, and non-finite coordinates.  The pyramids the kernel reads are the extractors' own, read back and
checked equal to the oracle's, so all three see the same pixels."""
import numpy as np
import pytest

import stereo_cases as SC
import stereo_reference as SR

pytestmark = pytest.mark.gpu

CASES = SC.all_cases()


@pytest.fixture(scope="module")
def scenes(oracle):
    """scene key -> (left extractor, right extractor, left pyramid, right pyramid) after extracting the scene's pair."""
    from openvslam_b200 import feature
    P = oracle.params(2000)
    out = {}
    for c in CASES:
        k = SC.scene_key(c)
        if k in out:
            continue
        left, right = SC.images(c)
        el = feature.orb_extractor(feature.orb_params(max_num_keypts=2000))
        er = feature.orb_extractor(feature.orb_params(max_num_keypts=2000))
        el.extract(left); er.extract(right)
        lp, rp = oracle.build_pyramid(left, P), oracle.build_pyramid(right, P)
        for lvl in range(SC.LEVELS):
            assert np.array_equal(el.image_pyramid(lvl), lp[lvl]) and np.array_equal(er.image_pyramid(lvl), rp[lvl]), (k, lvl)
        out[k] = (el, er, lp, rp)
    yield out
    for el, er, _, _ in out.values():
        el.close(); er.close()


@pytest.fixture(scope="module")
def st():
    from openvslam_b200 import match
    s = match.stereo()
    yield s
    s.close()


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_kernel_equals_oracle_and_reference(oracle, scenes, st, name):
    from openvslam_b200 import _lib
    c = next(c for c in CASES if c["name"] == name)
    el, er, lp, rp = scenes[SC.scene_key(c)]
    args = (c["kl"], c["dl"], c["kr"], c["dr"], c["fxb"], c["baseline"])
    before = _lib.launch_count()
    xr, dp, n = st.compute(el, er, *args)
    assert _lib.launch_count() - before == (2 if len(c["kl"]) and len(c["kr"]) else 0)
    oxr, odp, on = oracle.stereo_compute(lp, rp, SC.scale_factors(), *args)
    r = SR.compute(lp, rp, SC.scale_factors(), *args)
    assert n == on == r["num_matched"]
    for want in (oxr, r["x_right"]):
        assert np.array_equal(_bits(xr), _bits(want))
    for want in (odp, r["depth"]):
        assert np.array_equal(_bits(dp), _bits(want))
    xr2, dp2, n2 = st.compute(el, er, *args)                            # a repeat call is bit-identical
    assert n2 == n and np.array_equal(_bits(xr2), _bits(xr)) and np.array_equal(_bits(dp2), _bits(dp))


def _refused(code, fn):
    from openvslam_b200 import _lib
    before = _lib.launch_count()
    with pytest.raises(_lib.OvsError) as e:
        fn()
    assert e.value.code == code and _lib.launch_count() == before


def test_refused_before_any_launch(scenes, st):
    from openvslam_b200 import feature
    OVS_ERR_INVALID_ARG, OVS_ERR_UNSUPPORTED = -1, -6
    c = next(c for c in CASES if c["name"] == "gates")
    el, er, _, _ = scenes["shift"]
    kl, dl, kr, dr = c["kl"], c["dl"], c["kr"], c["dr"]
    for bad in (-1, SC.LEVELS):
        k = kl.copy(); k["octave"][len(k) // 2] = bad
        _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(el, er, k, dl, kr, dr, SC.FXB, SC.BASELINE))
        k = kr.copy(); k["octave"][len(k) // 2] = bad
        _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(el, er, kl, dl, k, dr, SC.FXB, SC.BASELINE))
    for bl in (0.0, -0.5, float("nan")):
        _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(el, er, kl, dl, kr, dr, SC.FXB, bl))
    # the largest supported right set is 65534 (sizes_*_65534 cases); one more is refused
    big = next(c for c in CASES if c["name"] == "sizes_1_65534_last")
    kr1 = np.concatenate([big["kr"], big["kr"][:1]]); dr1 = np.concatenate([big["dr"], big["dr"][:1]])
    _refused(OVS_ERR_UNSUPPORTED, lambda: st.compute(el, er, big["kl"], big["dl"], kr1, dr1, SC.FXB, SC.BASELINE))
    fresh = feature.orb_extractor(feature.orb_params(max_num_keypts=2000))
    _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(fresh, er, kl, dl, kr, dr, SC.FXB, SC.BASELINE))   # never extracted
    _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(el, fresh, kl, dl, kr, dr, SC.FXB, SC.BASELINE))
    left, _ = SC.scene("shift")
    fresh.extract(np.ascontiguousarray(left[:, :1200]))                                              # another image size
    _refused(OVS_ERR_INVALID_ARG, lambda: st.compute(el, fresh, kl, dl, kr, dr, SC.FXB, SC.BASELINE))
    fresh.close()
