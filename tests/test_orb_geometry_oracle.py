"""CPU checks of the ORB oracle (oracle/image_ops.py) away from the two image sizes the parity tests use: pyramid levels too small for a
cell (the product's rule: no cells, no keypoints, no quota moved), geometries without an initial octree node (refused), and the pyramid,
blur border and resize arithmetic down to 1-px levels, where the CUDA kernels' formulas are pinned to cv2."""
import math

import cv2
import numpy as np
import pytest

from oracle import image_ops as io
from tests.test_image_oracle import _resize_fixed_point
from vdo_slam_b200.synth import make_frame


def _noise(seed, w, h):
    rng = np.random.default_rng(seed)
    a = cv2.GaussianBlur(rng.normal(0, 1, (h, w)).astype(np.float32), (0, 0), 1.5)
    lo, hi = np.percentile(a, (1, 99))
    return np.clip((a - lo) / (hi - lo) * 255, 0, 255).round().astype(np.uint8)


def _level_sizes(w, h, prm):
    """cvRound(w * invScale) in float, as ComputePyramid sizes its levels (src/ORBextractor.cc:1117)"""
    return [(w, h)] + [(io.cvround(float(np.float32(w) * prm.inv_scale[l])), io.cvround(float(np.float32(h) * prm.inv_scale[l])))
                       for l in range(1, prm.nlevels)]


def _per_level_unchanged(levels, prm):
    """the oracle's per-level path before levels without cells had a rule: candidates and octree on every level"""
    out = []
    for lv, img in enumerate(levels):
        h, w = img.shape
        _, (minX, maxX, minY, maxY) = io.level_cells(w, h)
        cand = io.fast_candidates(img, prm)
        out.append((len(cand), io.distribute_octtree(cand, minX, maxX, minY, maxY, prm.per_level[lv])))
    return out


@pytest.mark.parametrize("w,h", [(1242, 375), (640, 480)])
def test_no_cell_rule_leaves_levels_with_cells_unchanged(w, h):
    """at the sizes the parity tests use every level has cells, and orb_extract is the per-level path it always was"""
    g = make_frame(4, width=w, height=h)["gray"]
    prm = io.OrbParams()
    r = io.orb_extract(g, prm, with_angle=False)
    assert all(io.level_cells(im.shape[1], im.shape[0])[0] for im in r["levels"])
    ref = _per_level_unchanged(r["levels"], prm)
    assert r["n_candidates"] == [n for n, _ in ref]
    for lv, (_, kept) in enumerate(ref):
        m = r["octave"] == lv
        assert np.array_equal(r["response"][m], np.asarray([k[2] for k in kept], np.float32)), lv
        assert np.array_equal(r["level_x"][m], np.asarray([k[0] + np.float32(16) for k in kept], np.float32)), lv


@pytest.mark.parametrize("w,h,n_with_cells", [(64, 64, 1), (200, 64, 1), (2048, 96, 3), (4096, 64, 1), (375, 220, 7)])
def test_levels_without_cells_keep_nothing_and_move_no_quota(w, h, n_with_cells):
    prm = io.OrbParams()
    g = _noise(w + h, w, h)
    r = io.orb_extract(g, prm, with_angle=False)
    cells = [io.level_cells(im.shape[1], im.shape[0])[0] for im in r["levels"]]
    assert [bool(c) for c in cells] == [l < n_with_cells for l in range(prm.nlevels)]          # the regime this case is for
    assert all(n == 0 for n in r["n_candidates"][n_with_cells:]) and not (r["octave"] >= n_with_cells).any()
    # a level with cells gives what the octree of its candidates at its own quota gives: the quota of the empty levels goes nowhere
    for lv in range(n_with_cells):
        img = r["levels"][lv]
        _, (minX, maxX, minY, maxY) = io.level_cells(img.shape[1], img.shape[0])
        cand = io.fast_candidates(img, prm)
        kept = io.distribute_octtree(cand, minX, maxX, minY, maxY, prm.per_level[lv])
        assert r["n_candidates"][lv] == len(cand) > 0
        assert np.array_equal(r["response"][r["octave"] == lv], np.asarray([k[2] for k in kept], np.float32)), lv


def test_level_cells_boundary_is_62_px():
    assert io.level_cells(61, 200)[0] == [] and io.level_cells(200, 61)[0] == []
    assert len(io.level_cells(62, 62)[0]) == 1 and len(io.level_cells(91, 62)[0]) == 1 and len(io.level_cells(92, 62)[0]) == 2


def test_geometries_without_an_initial_node_are_refused():
    with pytest.raises(ValueError, match="nIni = 0"):
        io.orb_extract(_noise(1, 375, 1242), io.OrbParams())
    with pytest.raises(ValueError, match="nIni = 0"):          # level 0 has a node; level 4 (106 x 181) has cells and none
        io.orb_extract(_noise(2, 220, 375), io.OrbParams())
    with pytest.raises(ValueError, match="nIni = 0"):          # refused whatever the keys, like the device refuses the geometry
        io.distribute_octtree([], 16, 116, 16, 318, 100)
    assert io.distribute_octtree([], 16, 116, 16, 216, 100) == []                     # 100 / 200 = 0.5 rounds away from zero: one node


@pytest.mark.parametrize("w,h,scale,nlevels", [(64, 64, 2.0, 7), (65, 97, 1.5, 12), (97, 65, 1.7, 9), (4096, 64, 2.0, 7), (375, 220, 1.3, 12)])
def test_pyramid_is_the_cv2_resize_chain_down_to_1px(w, h, scale, nlevels):
    """compute_pyramid sizes its levels like the reference and is the chain of cv2.resize calls; the fixed-point formula k_resize_u8
    implements equals every link of the chain, and the fixed-point blur k_blur7_batch implements equals cv2.GaussianBlur on every level"""
    prm = io.OrbParams(500, scale, nlevels)
    sizes = _level_sizes(w, h, prm)
    assert min(min(s) for s in sizes) >= 1
    g = _noise(7, w, h)
    lv = io.compute_pyramid(g, prm)
    assert [im.shape[::-1] for im in lv] == sizes
    prev = g
    for l in range(1, nlevels):
        want = cv2.resize(prev, sizes[l], interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(lv[l], want), l
        assert np.array_equal(_resize_fixed_point(prev, *sizes[l]), want), l
        prev = want
    for l, im in enumerate(lv):
        assert np.array_equal(io.blur_level(im), io.blur_level_fixed_point(im)), l
    if (w, h, scale) == (64, 64, 2.0):
        assert [s[0] for s in sizes] == [64, 32, 16, 8, 4, 2, 1]


def _reflect101_kernel(p, n):
    """the border rule of blur7_px in frame_kernels.cu, restated"""
    if n == 1:
        return 0
    while not 0 <= p < n:
        p = -p if p < 0 else 2 * n - 2 - p
    return p


def test_blur_border_rule_is_cv2_reflect101_on_tiny_levels():
    """a 7-tap kernel on a 1 .. 3 px level reaches past the far border: the index reflects more than once"""
    for n in range(1, 9):
        row = np.arange(n, dtype=np.uint8)[None, :]
        padded = cv2.copyMakeBorder(row, 0, 0, 3, 3, cv2.BORDER_REFLECT_101)[0]
        assert padded.tolist() == [_reflect101_kernel(p, n) for p in range(-3, n + 3)], n


def test_zero_size_level_is_what_the_reference_cannot_resize():
    prm = io.OrbParams(500, 2.0, 8)
    assert _level_sizes(64, 64, prm)[-1] == (0, 0)
    with pytest.raises(cv2.error):
        io.compute_pyramid(_noise(3, 64, 64), prm)


def test_exact_half_ratios_round_away_from_zero():
    """nIni = round((w - 32) / (h - 32)) with C round(): .5 goes up, as roundf on the device and std::round on the host"""
    for (w, h), nini in (((132, 232), 1), ((332, 232), 2), ((282, 132), 3)):
        _, (minX, maxX, minY, maxY) = io.level_cells(w, h)
        r = np.float32(maxX - minX) / np.float32(maxY - minY)
        assert r * 2 == math.floor(r * 2) and r != math.floor(r)                            # exactly k + 1/2
        assert int(math.floor(float(r) + 0.5)) == nini
