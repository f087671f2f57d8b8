"""synth.make_view_pair: the second view is the first one warped through the geometry, so a pixel of B shows what its source in A shows."""
import numpy as np

from vdo_slam_b200 import synth


def test_view_pair_pixel_maps_back_to_its_source():
    v = synth.make_view_pair(t=3, seed=1, dt=1, yaw_extra=0.01, shift=(0.2, 0.0, 0.0))
    K = v["K"].astype(np.float64)
    H, W = v["gray_b"].shape
    rng = np.random.default_rng(0)
    vb, ub = rng.integers(0, H, 400), rng.integers(0, W, 400)
    src = v["src_b"][vb, ub]
    seen = np.isfinite(src[:, 0])
    assert seen.mean() > 0.8
    # B's pixel -> 3-D point through B's depth -> A's camera through the true poses: lands on the source the warp used
    z = v["depth_b"][vb, ub].astype(np.float64)
    Xb = np.stack([(ub - K[2]) * z / K[0], (vb - K[3]) * z / K[1], z, np.ones_like(z)], 1)
    Xa = (v["Tcw_a"] @ v["Twc_b"] @ Xb.T).T
    ua, va = K[0] * Xa[:, 0] / Xa[:, 2] + K[2], K[1] * Xa[:, 1] / Xa[:, 2] + K[3]
    assert np.abs(ua[seen] - src[seen, 0]).max() < 1e-3 and np.abs(va[seen] - src[seen, 1]).max() < 1e-3
    # ... where A's depth agrees with the point's depth in A (the scene is static and both depths are the same corridor), and B's
    # gray value is A's image there
    ia, ja = np.round(va[seen]).astype(int), np.round(ua[seen]).astype(int)
    inner = (ia > 0) & (ia < H - 1) & (ja > 0) & (ja < W - 1)
    rel = np.abs(v["depth_a"][ia, ja][inner] - Xa[seen, 2][inner]) / Xa[seen, 2][inner]
    assert np.median(rel) < 0.02
    gb = v["gray_b"][vb, ub][seen].astype(np.float64)
    ga = synth._bilinear(v["gray_a"], ua[seen], va[seen])
    assert np.abs(gb - ga).max() <= 0.5 + 1e-6
    # T_ba maps A's camera frame to B's
    assert np.allclose(v["T_ba"], v["Tcw_b"] @ v["Twc_a"])


def test_view_pair_first_view_is_the_sequence_frame():
    v = synth.make_view_pair(t=2, seed=0)
    f = synth.make_sequence_frame(2, seed=0, n_obj=0)
    assert np.array_equal(v["gray_a"], f["gray"]) and np.array_equal(v["Twc_a"], f["Twc"])
