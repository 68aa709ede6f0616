"""GPU parity of the ORB extractor against the CPU oracle at its size-driven limits: the global-memory sorts of the tree
distribution (large budgets; which branch each case reaches is pinned on the CPU with the numpy tree model), dense-corner images
whose candidate lists fill the per-level buffers, and the 4096 px candidate coordinate range.  Every extraction is compared on all
cv::KeyPoint fields, on the descriptors and on each level's candidate list."""
import numpy as np
import pytest

import extractor_limit_cases as lc
from test_extractor_gpu import _assert_same

pytestmark = pytest.mark.gpu


def _extractor(n, **kw):
    from openvslam_b200 import feature
    return feature.orb_extractor(feature.orb_params(max_num_keypts=n, **kw))


def _assert_same_with_candidates(oracle, img, ext, n, **okw):
    kps, desc, dbg = _assert_same(oracle, img, ext, n, **okw)
    P = oracle.params(n, **okw)
    sf = oracle.scale_factors(P.scale_factor, P.num_levels)
    cands = []
    for l, level in enumerate(oracle.build_pyramid(img, P)):
        c = oracle.level_candidates(P, level, float(sf[l]))
        assert len(c) == dbg["num_candidates"][l]
        got = ext.debug_candidates(l)
        assert np.array_equal(got, np.stack([c["x"], c["y"], c["score"]], 1).reshape(-1, 3)), l
        cands.append(got)
    return kps, desc, dbg, cands


@pytest.mark.parametrize("case", list(lc.TREE_CASES))
def test_tree_sort_branches(oracle, case):
    make, n, levels, _, _ = lc.TREE_CASES[case]
    img = make()
    ext = _extractor(n, num_levels=levels)
    kps = _assert_same_with_candidates(oracle, img, ext, n, num_levels=levels)[0]
    assert len(kps) >= n
    ext.close()


@pytest.mark.parametrize("w,h,n", lc.DENSE_SIZES)
@pytest.mark.parametrize("image", list(lc.DENSE_IMAGES))
def test_dense_corner_images(oracle, image, w, h, n):
    make, kw = lc.DENSE_IMAGES[image]
    img = make(w, h)
    ext = _extractor(n, **kw)
    kps, _, dbg, _ = _assert_same_with_candidates(oracle, img, ext, n, **kw)
    assert len(kps) > 0.85 * n
    if image.startswith("lattice"):
        # more level-0 candidates than an area estimate of w * h / 8 (+ 1024) slots would hold
        assert dbg["num_candidates"][0] > w * h // 8 + 1024
    ext.close()


@pytest.mark.parametrize("w,h", [(4133, 120), (120, 4133)])
def test_coordinate_limit(oracle, w, h):
    """Candidates pack x and y relative to the 19 px border in 12 bits each: 4133 px (4095 px inside the borders) is the largest
    extent accepted, 4134 px is refused with OVS_ERR_UNSUPPORTED and leaves the handle usable.  At this aspect ratio the tree's
    first pass alone returns more keypoints than the handle was sized for at creation: the handle grows and the call is retried."""
    from openvslam_b200 import _lib
    img = lc.noise(w, h, 7)
    ext = _extractor(300)
    cap0 = ext._cap
    # refused on a fresh handle, then on a handle configured for the valid image
    for bw, bh in ((4134, 120), (120, 4134)) if w > h else ((120, 4134), (4134, 120)):
        with pytest.raises(_lib.OvsError) as e:
            ext.extract(lc.noise(bw, bh, 8))
        assert e.value.code == -6, (bw, bh)
        kps, _, _, cands = _assert_same_with_candidates(oracle, img, ext, 300)
        assert len(kps) > cap0
        # level-0 candidates reach the last column / row the detection cells examine (3 px inside the last cell's ROI)
        long_axis = 0 if w > h else 1
        assert cands[0][:, long_axis].max() == max(w, h) - 2 * 19 - 4
    ext.close()


@pytest.mark.parametrize("make,n,levels", [(lambda: lc.noise(1920, 960, 1), 40000, 1), (lambda: lc.lattice(1920, 960), 4000, 8)],
                         ids=["noise1920-n40000", "lattice1920-n4000"])
def test_extract_device_matches_host(make, n, levels):
    """ovs_extract_device (image already in HBM, outputs left in HBM) gives the bits of the host entry point."""
    import torch
    from openvslam_b200 import feature
    img = make()
    h, w = img.shape
    ext = _extractor(n, num_levels=levels)
    kps, desc = ext.extract(img)
    dev = torch.device("cuda", 0)
    d_img = torch.from_numpy(img).to(dev)
    cap = ext._cap
    d_kps = torch.zeros((cap, feature.KEYPOINT_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((cap, 32), dtype=torch.uint8, device=dev)
    num = ext.extract_device(d_img.data_ptr(), w, h, w, d_kps.data_ptr(), d_desc.data_ptr(), cap)
    assert num == len(kps)
    assert d_kps[:num].cpu().numpy().tobytes() == kps.tobytes()
    assert np.array_equal(d_desc[:num].cpu().numpy(), desc)
    ext.close()
