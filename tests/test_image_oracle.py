"""CPU checks of the image-side oracle (oracle/image_ops.py): the formulas the CUDA kernels implement for the OpenCV-owned
arithmetic are verified bit-exact against the cv2 in this image (the pin), and the oracle's own pieces are sanity-checked."""
import math

import cv2
import numpy as np

from oracle import image_ops as io
from vdo_slam_b200.synth import make_frame


def _resize_fixed_point(src, dw, dh):
    sh, sw = src.shape

    def coeffs(dn, sn):
        scale = sn / dn
        idx, a = np.zeros(dn, np.int64), np.zeros((dn, 2), np.int32)
        for d in range(dn):
            f = np.float32((d + 0.5) * scale - 0.5)
            s = int(math.floor(float(f))); f = np.float32(f - np.float32(s))
            if s < 0: s, f = 0, np.float32(0)
            if s >= sn - 1: s, f = sn - 1, np.float32(0)
            idx[d] = s
            a[d] = (int(np.rint(np.float32(1.0 - f) * np.float32(2048))), int(np.rint(f * np.float32(2048))))
        return idx, a

    xi, xa = coeffs(dw, sw); yi, ya = coeffs(dh, sh)
    S = src.astype(np.int32)
    H = S[:, xi] * xa[:, 0] + S[:, np.minimum(xi + 1, sw - 1)] * xa[:, 1]
    out = (((ya[:, 0:1] * (H[yi] >> 4)) >> 16) + ((ya[:, 1:2] * (H[np.minimum(yi + 1, sh - 1)] >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def test_resize_formula_is_bit_exact_vs_cv2():
    rng = np.random.default_rng(0)
    for (h, w) in [(375, 1242), (313, 1035), (97, 131)]:
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        dw, dh = int(np.rint(w / 1.2)), int(np.rint(h / 1.2))
        assert np.array_equal(cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR), _resize_fixed_point(img, dw, dh))


_OFF = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]


def _fast_score(img):
    h, w = img.shape; I = img.astype(np.int32)
    c = I[3:h - 3, 3:w - 3]
    d = np.stack([c - I[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for (dx, dy) in _OFF], 0)
    best = np.full(c.shape, -10 ** 6)
    for k in range(16):
        idx = [(k + j) % 16 for j in range(9)]
        best = np.maximum(best, np.maximum(d[idx].min(0), (-d[idx]).min(0)))
    sc = np.zeros((h, w), np.int32)
    sc[3:h - 3, 3:w - 3] = np.maximum(best - 1, 0)
    return sc


def test_fast_score_and_nms_formula_matches_cv2():
    rng = np.random.default_rng(1)
    img = cv2.GaussianBlur(rng.integers(0, 256, (160, 220), dtype=np.uint8), (5, 5), 1.2)
    sc = _fast_score(img)
    for thr in (20, 7):
        kps = cv2.FastFeatureDetector_create(thr, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16).detect(img)
        s = np.where(sc >= thr, sc, 0); p = np.pad(s, 1)
        nb = np.stack([p[1 + dy:p.shape[0] - 1 + dy, 1 + dx:p.shape[1] - 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy) != (0, 0)], 0).max(0)
        ys, xs = np.nonzero((sc >= thr) & (s > nb))
        assert [(int(k.pt[0]), int(k.pt[1])) for k in kps] == list(zip(xs.tolist(), ys.tolist()))      # same set, same order
        assert [int(k.response) for k in kps] == sc[ys, xs].tolist()                                      # same responses


def test_orb_oracle_quota_and_order():
    f = make_frame(0)
    prm = io.OrbParams()
    assert prm.per_level == [543, 452, 377, 314, 262, 218, 182, 152]          # SURVEY.md section 8
    r = io.orb_extract(f["gray"], prm, with_angle=False)
    assert 2000 < len(r["x"]) < 2700
    assert (np.diff(r["octave"]) >= 0).all()                                 # level-major output
    assert r["x"].min() >= 16 and r["x"].max() < 1242 - 16


def test_sampling_oracle_properties():
    f = make_frame(3)
    d = io.depth_prep(f["depth_raw"], 387.5744, 256.0)
    assert (d[f["depth_raw"] < 0] == 0).all() and np.isfinite(d[f["depth_raw"] > 0]).all()
    s = io.sample_objects(f["mask"], d, f["flow"], 25.0)
    assert len(s["x"]) > 100 and (s["label"] > 0).all() and (s["x"] % 4 == 0).all() and (s["y"] % 4 == 0).all()
    key = s["y"].astype(np.int64) * 10000 + s["x"]
    assert (np.diff(key) > 0).all()                                           # raster order


# ---- A6: 7x7 blur + rotated-BRIEF descriptors (src/ORBextractor.cc:1083-1084, 97-136) ----
def test_blur_restatement_is_cv2_gaussianblur_bit_for_bit():
    rng = np.random.default_rng(3)
    for shape in ((64, 80), (37, 129), (375, 1242)):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(io.blur_level(img), io.blur_level_fixed_point(img))      # the fixed-point arithmetic k_blur7_batch implements


def test_descriptors_match_cv2_orb_up_to_blur_rounding():
    """cv2.ORB carries the same sampling pattern, the same rotation arithmetic and the same blur call; its internal blur (on a view of its
    bordered pyramid) differs from a stand-alone cv2.GaussianBlur by +-1 in a few pixels, so descriptor bits may differ only where the two
    samples of a pair are within 2 of each other (each off by at most 1) -- every other bit must be identical."""
    import cv2
    from vdo_slam_b200.synth import make_frame
    g = make_frame(0)["gray"]
    res = io.orb_extract(g, io.OrbParams())
    D = io.orb_describe(res)
    m = np.nonzero(res["octave"] == 0)[0]
    orb = cv2.ORB_create(nfeatures=5000, scaleFactor=1.2, nlevels=1, edgeThreshold=19, patchSize=31)
    kps = [cv2.KeyPoint(float(res["x"][i]), float(res["y"][i]), 31.0, float(res["angle"][i]), float(res["response"][i]), 0) for i in m]
    kps2, des = orb.compute(g, kps)
    where = {(k.pt[0], k.pt[1]): i for i, k in enumerate(kps2)}
    pat, bl, f32 = io.orb_pattern(), io.blur_level(g), np.float32
    n_cmp = n_same = 0
    for j, i in enumerate(m):
        c = des[where[(kps[j].pt[0], kps[j].pt[1])]]
        n_cmp += 1
        if np.array_equal(c, D[i]):
            n_same += 1
            continue
        ang = f32(f32(res["angle"][i]) * f32(np.pi / f32(180.0)))
        a, b = f32(np.cos(np.float64(ang))), f32(np.sin(np.float64(ang)))
        cy, cx = io.cvround(float(res["y"][i])), io.cvround(float(res["x"][i]))
        for bit in np.nonzero(np.unpackbits((c ^ D[i])[:, None], axis=1, bitorder="little").reshape(-1))[0]:
            p = pat[2 * bit:2 * bit + 2].astype(f32)
            iy = np.rint(p[:, 0] * b + p[:, 1] * a).astype(int); ix = np.rint(p[:, 0] * a - p[:, 1] * b).astype(int)
            t = bl[cy + iy, cx + ix].astype(int)
            assert abs(int(t[0]) - int(t[1])) <= 2, (i, bit, t)      # each sample off by at most 1
    assert n_cmp > 300 and n_same > n_cmp // 2
