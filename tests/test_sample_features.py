"""Sampled background features (UseSampleFeature: 1) on the CPU: the cv::RNG restatement against OpenCV's own generator, its
jump-ahead form against serial stepping, and the shape of Frame::SampleKeyPoints' output."""
import numpy as np
import pytest

from tests.sample_reference import RNG_A, RNG_M, SAMPLE_DIV, SAMPLE_N, CvRNG, rng_jump, sample_keypoints


@pytest.mark.parametrize("seed", [0, 1, 977, 1_600_000_000, 2 ** 31 - 1])
@pytest.mark.parametrize("low,width", [(0, 24), (62, 62), (18 * 7, 18)])
def test_generator_equals_cv2(seed, low, width):
    """cv2.randu on int32 draws one uniform(low, low + width) per element from theRNG(); widths that are not powers of two take the
    modulo path RNG::uniform(int, int) always takes"""
    cv2 = pytest.importorskip("cv2")
    cv2.setRNGSeed(seed)
    a = np.zeros((1, 400), np.int32)
    cv2.randu(a, low, low + width)
    r = CvRNG(seed)
    assert a[0].tolist() == [r.uniform(low, low + width) for _ in range(400)]


@pytest.mark.parametrize("seed", [0, 5, 2 ** 32 - 1])
def test_jump_equals_serial_steps(seed):
    r = CvRNG(seed)
    s0 = r.state
    for k in range(1, 7201):
        r.next()
        if k % 97 == 0 or k in (1, 2, 798, 7200):
            assert rng_jump(s0, k) == r.state, k
    assert r.state < RNG_M and RNG_M == RNG_A * 2 ** 32 - 1


@pytest.mark.parametrize("rows,cols,seed", [(480, 640, 0), (375, 1242, 2 ** 32 - 1), (20, 20, 3)])
def test_sampler_shape_and_order(rows, cols, seed):
    kx, ky = sample_keypoints(rows, cols, seed)
    assert len(kx) == SAMPLE_N and len(ky) == SAMPLE_N
    assert (kx > 0).all() and (ky > 0).all() and (kx < cols).all() and (ky < rows).all()
    assert np.array_equal(kx, np.floor(kx)) and np.array_equal(ky, np.floor(ky))
    cell = (kx.astype(int) // (cols // SAMPLE_DIV)) * SAMPLE_DIV + ky.astype(int) // (rows // SAMPLE_DIV)
    assert (np.diff(cell) >= 0).all()                                     # cell by cell, i*20 + j ascending
    # every round accepts the 361 cells with i, j >= 1, so those cells hold 7 to 9 keys each
    inner = np.bincount(cell, minlength=SAMPLE_DIV ** 2).reshape(SAMPLE_DIV, SAMPLE_DIV)[1:, 1:]
    assert inner.min() >= 7 and inner.max() <= 9

