"""GPU parity of the image-side kernels against the oracle (numpy restatement + cv2 as the OpenCV pin).
Integer / index outputs (keypoint coordinates, order, octaves, responses, sampled pixels, labels) must match exactly."""
import numpy as np
import pytest

from oracle import image_ops as io
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_frame, KITTI_K

pytestmark = pytest.mark.gpu
BF, FACTOR = 387.5744, 256.0


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def test_pyramid_and_fast_score_maps_match_cv2(ctx):
    from tests.test_image_oracle import _fast_score
    f = make_frame(0)
    F = capi.Frame(ctx, 1242, 375)
    F.upload(gray=f["gray"])
    F.orb_extract()
    levels = io.compute_pyramid(f["gray"], io.OrbParams())
    for lv in range(8):
        img, sc = F.debug_level(lv)
        assert img.shape == levels[lv].shape and np.array_equal(img, levels[lv]), f"pyramid level {lv}"     # cv2.resize chain, bit exact
        assert np.array_equal(sc.astype(np.int32), np.minimum(_fast_score(levels[lv]), 255)), f"score level {lv}"


@pytest.mark.parametrize("seed,shape", [(0, (375, 1242)), (5, (375, 1242)), (2, (480, 640))])
def test_orb_extract_matches_oracle_exactly(ctx, seed, shape):
    f = make_frame(seed, width=shape[1], height=shape[0])
    F = capi.Frame(ctx, shape[1], shape[0])
    F.upload(gray=f["gray"])
    g = F.orb_extract()
    o = io.orb_extract(f["gray"], io.OrbParams())
    assert g["n_candidates"] == o["n_candidates"]                  # FAST + NMS + threshold fallback, every level
    assert len(g["x"]) == len(o["x"])
    assert np.array_equal(g["octave"], o["octave"]) and np.array_equal(g["x"], o["x"]) and np.array_equal(g["y"], o["y"])
    assert np.array_equal(g["response"], o["response"]) and np.array_equal(g["size"], o["size"])
    np.testing.assert_allclose(g["angle"], o["angle"], atol=1e-3)  # cv::fastAtan2 polynomial, degrees


def test_orb_extract_after_a_scale_factor_change(ctx):
    """a second extraction on one frame that changes only the scale factor extracts at the new scale"""
    f = make_frame(0)
    F = capi.Frame(ctx, 1242, 375)
    F.upload(gray=f["gray"])
    F.orb_extract(scale=1.3)
    g = F.orb_extract(scale=1.2)
    o = io.orb_extract(f["gray"], io.OrbParams(scale=1.2))
    assert g["n_candidates"] == o["n_candidates"] and len(g["x"]) == len(o["x"])
    for k in ("x", "y", "octave", "response", "size"):
        assert np.array_equal(g[k], o[k]), k
    np.testing.assert_allclose(g["angle"], o["angle"], atol=1e-3)


def test_orb_on_flat_image_is_empty(ctx):
    F = capi.Frame(ctx, 640, 480)
    F.upload(gray=np.full((480, 640), 128, np.uint8))
    assert len(F.orb_extract()["x"]) == 0


def test_depth_static_filter_and_object_sampling(ctx):
    f = make_frame(7)
    H, W = f["gray"].shape
    F = capi.Frame(ctx, W, H)
    F.upload(gray=f["gray"], depth=f["depth_raw"], flow=f["flow"], mask=f["mask"])
    d = F.depth_prep(BF, FACTOR)
    do = io.depth_prep(f["depth_raw"], BF, FACTOR)
    assert np.array_equal(d, do)                                   # includes +inf where the raw disparity is 0
    kp = F.orb_extract()
    idx, cx, cy, fu, fv, dep = F.filter_static(kp["x"], kp["y"], 40.0)
    oidx, ocx, ocy, ofu, ofv, odep = io.filter_static(kp["x"], kp["y"], f["mask"], do, f["flow"], 40.0)
    assert np.array_equal(idx, oidx) and np.array_equal(cx, ocx) and np.array_equal(cy, ocy) and np.array_equal(dep, odep)
    s = F.sample_objects(25.0)
    so = io.sample_objects(f["mask"], do, f["flow"], 25.0)
    for k in ("x", "y", "label", "cx", "cy", "fx", "fy", "depth"):
        assert np.array_equal(s[k], so[k]), k


def test_sampling_edge_cases(ctx):
    H, W = 96, 128
    F = capi.Frame(ctx, W, H)
    z = np.zeros((H, W), np.float32)
    F.upload(gray=np.zeros((H, W), np.uint8), depth=z, flow=np.zeros((H, W, 2), np.float32), mask=np.zeros((H, W), np.int32))
    assert len(F.sample_objects(25.0)["x"]) == 0                   # nothing labelled
    m = np.ones((H, W), np.int32); d = np.full((H, W), 10.0, np.float32); fl = np.full((H, W, 2), 0.5, np.float32)
    F.upload(depth=d, flow=fl, mask=m)
    s = F.sample_objects(25.0); so = io.sample_objects(m, d, fl, 25.0)
    assert len(s["x"]) == len(so["x"]) == (H // 4) * (W // 4) and np.array_equal(s["x"], so["x"])


def test_scene_flow_matches_oracle(ctx):
    rng = np.random.default_rng(0)
    n = 5000
    up, vp = rng.uniform(0, 1241, n).astype(np.float32), rng.uniform(0, 374, n).astype(np.float32)
    uc, vc = (up + rng.normal(0, 3, n)).astype(np.float32), (vp + rng.normal(0, 1, n)).astype(np.float32)
    zp, zc = rng.uniform(4, 25, n).astype(np.float32), rng.uniform(4, 25, n).astype(np.float32)
    lp, lc = rng.integers(-1, 4, n).astype(np.int32), rng.integers(-1, 4, n).astype(np.int32)
    def pose(a, t):
        T = np.eye(4, dtype=np.float32); c, s = np.cos(a), np.sin(a)
        T[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], np.float32); T[:3, 3] = t
        return T
    Tp, Tc = pose(0.02, [0.1, 0.0, -1.0]), pose(0.035, [0.15, 0.01, -2.0])
    f3, Xp, valid = capi.scene_flow(ctx, up, vp, zp, Tp, uc, vc, zc, Tc, KITTI_K, lp, lc)
    of, ov = io.scene_flow(up, vp, zp, Tp, uc, vc, zc, Tc, KITTI_K, lp, lc)
    assert np.array_equal(valid, ov)
    np.testing.assert_allclose(f3, of, rtol=0, atol=2e-5)           # float32 world coordinates of ~25 m: 1 ulp = 2e-6
    np.testing.assert_allclose(Xp, io.unproject_world(up, vp, zp, KITTI_K, Tp), rtol=0, atol=4e-6)


def test_blur_and_descriptors_match_oracle(ctx):
    """A6: k_blur7_batch bit-exact against cv2.GaussianBlur on every pyramid level; rotated-BRIEF descriptors identical to the oracle's."""
    from vdo_slam_b200.synth import make_frame
    fr = make_frame(5)
    H, W = fr["gray"].shape
    F = capi.Frame(ctx, W, H)
    F.upload(gray=fr["gray"])
    kp = F.orb_extract()
    D = F.orb_describe(len(kp["x"]))
    res = io.orb_extract(fr["gray"], io.OrbParams())
    assert np.array_equal(kp["x"], res["x"]) and np.array_equal(kp["octave"], res["octave"])
    for lv, img in enumerate(res["levels"]):
        assert np.array_equal(F.debug_blur(lv, img.shape), io.blur_level(img)), lv
    Do = io.orb_describe(res)
    # the device angle may differ from cv2's fastAtan2 in the last float bit (<= 1e-3 deg, see the angle test): a descriptor bit can then flip
    # only where a rotated sample lands within rounding of a pixel boundary -- allow a handful of bits in total, none systematic
    nbits = int(np.unpackbits(D ^ Do).sum())
    assert D.shape == Do.shape and nbits <= max(4, D.size * 8 // 50000), nbits
