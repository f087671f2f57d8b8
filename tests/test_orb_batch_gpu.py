"""Batched ORB extraction from device images (OrbExtractor / vdo_orb_extract_batch_dev) and the device octree behind it.

Pinned to the oracle (oracle/image_ops.py, cv2 as the OpenCV pin) at every ORB setting below -- keypoints, responses, sizes and candidate
counts exactly, angles and descriptors to the oracle's float rounding -- and, for the octree alone, bit for bit to
image_ops.distribute_octtree on adversarial candidate sets.  Frame.orb_extract / orb_describe and the tracker run on the same extractor.
Also: batch independence, input layouts, capture in a CUDA graph, and the argument refusals."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import image_ops as io
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import bgr_to_gray_opencv34, colour_from_gray, make_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
FIELDS = ("x", "y", "octave", "response", "angle", "size")


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


_frames = {}


def _gray(seed, w=1242, h=375):
    if (seed, w, h) not in _frames:
        _frames[(seed, w, h)] = make_frame(seed, width=w, height=h)["gray"]
    return _frames[(seed, w, h)]


def _oracle(gray, s):
    """the oracle's single-frame path: ORBextractor::operator() and the descriptors of its keypoints"""
    r = io.orb_extract(gray, io.OrbParams(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"]))
    r["descriptors"] = io.orb_describe(r)
    return r


def _row(res, i):
    """frame i of a batch result as host arrays cut to its count"""
    n = int(res["count"][i])
    d = {k: res[k][i, :n].cpu().numpy() for k in FIELDS}
    if "descriptors" in res:
        d["descriptors"] = res["descriptors"][i, :n].cpu().numpy()
    d["n_candidates"] = res["n_candidates"][i].cpu().tolist()
    d["status"] = int(res["status"][i])
    return d


def _assert_same(a, b, what):
    assert a["n_candidates"] == b["n_candidates"], what
    assert len(a["x"]) == len(b["x"]), what
    for k in FIELDS + ("descriptors",):
        if k in a and k in b:
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{what}: {k}"


SETTINGS = [
    dict(n_features=1000, scale_factor=1.2, n_levels=8, ini_th_fast=20, min_th_fast=7),
    dict(n_features=2500, scale_factor=1.2, n_levels=8, ini_th_fast=20, min_th_fast=7),
    dict(n_features=3000, scale_factor=1.2, n_levels=8, ini_th_fast=20, min_th_fast=7),
    dict(n_features=3000, scale_factor=1.3, n_levels=4, ini_th_fast=20, min_th_fast=7),
    dict(n_features=1000, scale_factor=1.3, n_levels=4, ini_th_fast=12, min_th_fast=5),
]


# ------------------------------------------------------------------------------------------------ 1. against the oracle's single-frame path
@pytest.mark.parametrize("w,h", [(1242, 375), (640, 480)])
@pytest.mark.parametrize("si", range(len(SETTINGS)))
def test_batch_matches_single_frame_path(ctx, w, h, si):
    s = SETTINGS[si]
    seeds = (0, 3, 11)
    ex = capi.OrbExtractor(ctx, w, h, len(seeds), **s)
    grays = [_gray(seed, w, h) for seed in seeds]
    res = ex.extract(torch.from_numpy(np.stack(grays)).to(DEV))
    torch.cuda.synchronize()
    for i, g in enumerate(grays):
        got, ref = _row(res, i), _oracle(g, s)
        what = f"seed {seeds[i]} {w}x{h} {s}"
        assert got["status"] == 0 and 0 < len(got["x"]) <= ex.capacity, what
        assert got["n_candidates"] == ref["n_candidates"] and len(got["x"]) == len(ref["x"]), what
        for k in ("x", "y", "octave", "response", "size"):
            assert np.array_equal(got[k], ref[k]), f"{what}: {k}"
        np.testing.assert_allclose(got["angle"], ref["angle"], atol=1e-3, err_msg=what)
        # as in test_image_gpu.py: an angle one float bit off the oracle's can flip a descriptor bit whose rotated sample lands within
        # rounding of a pixel boundary -- a handful of bits in total, none systematic
        nbits = int(np.unpackbits(got["descriptors"] ^ ref["descriptors"]).sum())
        assert got["descriptors"].shape == ref["descriptors"].shape and nbits <= max(4, got["descriptors"].size * 8 // 50000), f"{what}: {nbits} bits"


def test_capacity_is_the_octree_bound(ctx):
    """capacity = sum over levels of max(N_l + 2, 4 nIni_l), from the reference's level geometry"""
    for (w, h), s in (((1242, 375), SETTINGS[2]), ((640, 480), SETTINGS[3])):
        ex = capi.OrbExtractor(ctx, w, h, 2, **s)
        prm = io.OrbParams(s["n_features"], s["scale_factor"], s["n_levels"], s["ini_th_fast"], s["min_th_fast"])
        cap = 0
        for lv in range(s["n_levels"]):
            lw = w if lv == 0 else io.cvround(float(np.float32(w) * prm.inv_scale[lv]))
            lh = h if lv == 0 else io.cvround(float(np.float32(h) * prm.inv_scale[lv]))
            _, (minX, maxX, minY, maxY) = io.level_cells(lw, lh)
            nini = int(math.floor(float(np.float32(maxX - minX) / np.float32(maxY - minY)) + 0.5))
            cap += max(prm.per_level[lv] + 2, 4 * nini)
        info = ex.info()
        assert info["capacity"] == ex.capacity == cap and info["n_levels"] == s["n_levels"] and info["max_batch"] == 2 and info["device_bytes"] > 0


# ------------------------------------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize("seed,shape", [(0, (375, 1242)), (2, (480, 640))])
def test_batch_matches_oracle(ctx, seed, shape):
    g = _gray(seed, shape[1], shape[0])
    ex = capi.OrbExtractor(ctx, shape[1], shape[0], 1)
    got = _row(ex.extract([torch.from_numpy(g).to(DEV)], describe=False), 0)
    o = io.orb_extract(g, io.OrbParams())
    assert got["n_candidates"] == o["n_candidates"] and len(got["x"]) == len(o["x"])
    for k in ("x", "y", "octave", "response", "size"):
        assert np.array_equal(got[k], o[k]), k
    np.testing.assert_allclose(got["angle"], o["angle"], atol=1e-3)


# ------------------------------------------------------------------------------------------------ 3. the device octree alone
def _octree_cases():
    rng = np.random.default_rng(7)
    cases = []
    # many equally sized nodes: a lattice of pairs, so every expandable node holds 2 keys and the sorted phase breaks ties by creation order
    xs, ys = np.meshgrid(np.arange(4, 600, 24), np.arange(4, 340, 24))
    lat = np.stack([xs.ravel(), ys.ravel()], 1).astype(np.float32)
    pairs = np.concatenate([lat, lat + np.float32(1)])
    for N in (40, 150, 333, 500):
        cases.append((f"lattice_pairs_N{N}", np.column_stack([pairs, rng.integers(7, 12, len(pairs))]), (16, 623, 16, 359), N))
    # duplicate coordinates: overlapping cells report the same pixel twice, and a cluster of one pixel never splits
    base = rng.uniform(0, 590, (800, 2)).astype(np.float32); base[:, 1] %= 330
    dup = np.concatenate([base, base[:300], np.tile(np.float32([[100, 100]]), (50, 1))])
    for N in (60, 400, 2000):
        cases.append((f"duplicates_N{N}", np.column_stack([np.floor(dup), rng.integers(7, 40, len(dup))]), (16, 623, 16, 359), N))
    # keys on split lines: integer coordinates on every power-of-two boundary of the subdivision
    line = np.array([[x, y] for x in range(0, 600, 8) for y in (0, 1, 84, 85, 168, 169, 170, 171)], np.float32)
    for N in (25, 200, 700):
        cases.append((f"split_lines_N{N}", np.column_stack([line, rng.integers(7, 9, len(line))]), (16, 623, 16, 359), N))
    # N = 1, N >= the number of candidates, a single key, no keys
    small = np.column_stack([rng.uniform(0, 600, 37), rng.uniform(0, 340, 37), rng.integers(7, 60, 37)])
    cases += [("N1", small, (16, 623, 16, 359), 1), ("N_ge_n", small, (16, 623, 16, 359), 37), ("N_gt_n", small, (16, 623, 16, 359), 500),
              ("single", small[:1], (16, 623, 16, 359), 20), ("single_N1", small[:1], (16, 623, 16, 359), 1), ("empty", small[:0], (16, 623, 16, 359), 20)]
    # nIni = 1 .. 5 (the aspect ratio of the border box), random keys and equal responses
    for nini in range(1, 6):
        H = 200
        W = nini * H + 37
        k = np.column_stack([rng.uniform(0, W - 0.5, 900), rng.uniform(0, H, 900), rng.integers(7, 15, 900)])   # x < W after rounding to f32
        for N in (3, 120, 450):
            cases.append((f"nini{nini}_N{N}", k, (16, 16 + W, 16, 16 + H), N))
    # several thousand candidates (a KITTI level 0 quota and more)
    big = np.column_stack([rng.uniform(0, 1209.5, 6000), rng.uniform(0, 343, 6000), rng.integers(7, 80, 6000)])
    for N in (651, 1500, 5990):
        cases.append((f"big_N{N}", big, (16, 1226, 16, 359), N))
    return cases


OCT_CASES = _octree_cases()


@pytest.mark.parametrize("case", OCT_CASES, ids=[c[0] for c in OCT_CASES])
def test_device_octree_matches_oracle(ctx, case):
    name, keys, (minX, maxX, minY, maxY), N = case
    keys = np.asarray(keys, np.float32).reshape(-1, 3)
    got, status = capi.orb_debug_octree(ctx, keys, minX, maxX, minY, maxY, N)
    ref = io.distribute_octtree([tuple(np.float32(v) for v in k) for k in keys], minX, maxX, minY, maxY, N)
    ref = np.asarray(ref, np.float32).reshape(-1, 3)
    assert status == 0
    assert got.shape == ref.shape and np.array_equal(got, ref), name
    nini = int(math.floor(float(np.float32(maxX - minX) / np.float32(maxY - minY)) + 0.5))
    assert len(got) <= max(N + 2, 4 * nini)


# ------------------------------------------------------------------------------------------------ 4. batch independence
def test_batch_independence(ctx):
    seeds = (1, 4, 5, 6, 8, 9, 12, 13)
    s = SETTINGS[2]
    ex = capi.OrbExtractor(ctx, 1242, 375, 8, **s)
    frames = [torch.from_numpy(_gray(seed)).to(DEV) for seed in seeds]
    alone = [_row(ex.extract([f]), 0) for f in frames]
    rng = np.random.default_rng(3)
    for B in (1, 3, 8):
        for trial in range(2):
            pick = rng.permutation(len(seeds))[:B] if trial else np.arange(B)
            res = ex.extract([frames[j] for j in pick])
            for i, j in enumerate(pick):
                _assert_same(_row(res, i), alone[j], f"B={B} slot {i} = seed {seeds[j]}")


# ------------------------------------------------------------------------------------------------ 5. input layouts
def test_input_layouts_match_the_resident_gray(ctx):
    w, h = 1242, 375
    bgr = colour_from_gray(_gray(2), seed=4)
    ex = capi.OrbExtractor(ctx, w, h, 8)
    F = capi.Frame(ctx, w, h)
    t = torch.from_numpy(bgr).to(DEV)                      # (H,W,3) BGR
    rgb_t = t.flip(2).contiguous()                         # (H,W,3) RGB
    big = torch.zeros((h + 6, w + 10, 3), dtype=torch.uint8, device=DEV)
    crop = big[2:2 + h, 5:5 + w]
    crop.copy_(t)
    wide = torch.zeros((h, 2 * w), dtype=torch.uint8, device=DEV)
    strided = wide[:, ::2]                                 # a gray view with stride_x = 2
    strided.copy_(torch.from_numpy(bgr_to_gray_opencv34(bgr)).to(DEV))
    views = [("bgr_hwc", t, False), ("rgb_hwc", rgb_t, True), ("bgr_chw", t.permute(2, 0, 1).contiguous(), False), ("rgb_chw_view", rgb_t.permute(2, 0, 1), True),
             ("bgr_hwc_crop", crop, False), ("bgra_hwc", torch.cat([t, torch.full((h, w, 1), 77, dtype=torch.uint8, device=DEV)], 2), False),
             ("gray_strided", strided, True)]
    res = {}
    for name, v, rgb in views:
        F.upload_tensors(image=v, rgb=rgb)
        F.orb_extract()
        gray = torch.from_numpy(F.debug_level(0)[0]).to(DEV)
        ref = _row(ex.extract(gray[None]), 0)
        got = _row(ex.extract([v], rgb=rgb), 0)
        _assert_same(got, ref, name)
        res[name] = got
    # all layouts in one call (rgb applies to every frame of a call: the BGR ones)
    bgr_views = [v for name, v, rgb in views if not rgb]
    names = [name for name, v, rgb in views if not rgb]
    out = ex.extract(bgr_views, rgb=False)
    for i, name in enumerate(names):
        _assert_same(_row(out, i), res[name], f"mixed batch {name}")


# ------------------------------------------------------------------------------------------------ 6. capture in a CUDA graph
def test_cuda_graph_capture_and_replay(ctx):
    w, h, B = 1242, 375, 3
    ex = capi.OrbExtractor(ctx, w, h, B, n_features=3000)
    static_in = torch.from_numpy(np.stack([_gray(s) for s in (0, 1, 2)])).to(DEV)
    out = ex.empty_outputs(B)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm-up outside the capture
        ex.extract(static_in, out=out)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                              # fails if the call synchronises or allocates
        ex.extract(static_in, out=out)
    for seeds in ((3, 4, 5), (6, 7, 8)):
        static_in.copy_(torch.from_numpy(np.stack([_gray(s) for s in seeds])).to(DEV))
        g.replay()
        torch.cuda.synchronize()
        replay = {k: v.clone() for k, v in out.items()}
        eager = ex.extract(torch.from_numpy(np.stack([_gray(s) for s in seeds])).to(DEV))
        torch.cuda.synchronize()
        for i in range(B):
            r = _row(replay, i)
            assert r["status"] == 0 and len(r["x"]) > 0
            _assert_same(r, _row(eager, i), f"replay seed {seeds[i]}")


# ------------------------------------------------------------------------------------------------ 7. refusals
def test_python_refusals(ctx):
    w, h = 640, 480
    ex = capi.OrbExtractor(ctx, w, h, 2)
    g = torch.from_numpy(_gray(0, w, h)).to(DEV)
    bad = [
        ("dtype", [g.float()]),
        ("device", [g.cpu()]),
        ("size", [g[:-1]]),
        ("channels", [torch.zeros((h, w, 2), dtype=torch.uint8, device=DEV)]),
        ("too many frames", [g, g, g]),
        ("no frames", []),
        ("not a tensor", [np.zeros((h, w), np.uint8)]),
        ("2-D tensor", g),
    ]
    for what, images in bad:
        with pytest.raises(ValueError):
            ex.extract(images)
    out = ex.empty_outputs(2)
    out["x"] = out["x"][:, :-1]
    with pytest.raises(ValueError):
        ex.extract([g], out=out)
    with pytest.raises(capi.VdoError):
        capi.OrbExtractor(ctx, w, h, 65)                   # max_batch over 64
    with pytest.raises(capi.VdoError):
        capi.OrbExtractor(ctx, 375, 1242, 1)               # nIni = 0: more than twice as tall as wide


def test_c_abi_refusals_do_no_device_work(ctx):
    w, h = 640, 480
    ex = capi.OrbExtractor(ctx, w, h, 2)
    L = ctx.L
    g = torch.from_numpy(_gray(0, w, h)).to(DEV)
    out = ex.empty_outputs(2)
    for t in out.values():
        t.fill_(-7 if t.dtype != torch.uint8 else 7)
    torch.cuda.synchronize()
    snap = {k: v.clone() for k, v in out.items()}
    keys = ("x", "y", "octave", "response", "angle", "size", "descriptors", "count", "n_candidates", "status")

    def outs(**over):
        p = {k: out[k].data_ptr() for k in keys}
        p.update(over)
        return capi.OrbBatchOut(*[p[k] for k in keys])

    def plane(**over):
        p = capi._dev_plane(ctx, "image", g, w, h)
        for k, v in over.items():
            setattr(p, k, v)
        return p

    host = np.zeros((h, w), np.uint8)
    cases = [
        ("n > max_batch", 3, [plane()] * 3, outs()),
        ("n = 0", 0, [plane()], outs()),
        ("dtype", 1, [plane(dtype=capi.VDO_DT_F32)], outs()),
        ("channels", 1, [plane(channels=2)], outs()),
        ("host image", 1, [plane(data_dev=host.ctypes.data)], outs()),
        ("NULL image", 1, [plane(data_dev=None)], outs()),
        ("misaligned output", 1, [plane()], outs(x=out["x"].data_ptr() + 1)),
        ("host output", 1, [plane()], outs(count=np.zeros(4, np.int32).ctypes.data)),
        ("NULL output", 1, [plane()], outs(status=None)),
    ]
    stream = int(torch.cuda.current_stream().cuda_stream)
    for what, n, planes, o in cases:
        arr = (capi.DevPlane * max(len(planes), 1))(*planes)
        rc = L.vdo_orb_extract_batch_dev(ex.h_, C.c_int(n), arr, C.byref(o), C.c_uint64(stream))
        assert rc == ERR_ARG, what
        assert L.vdo_last_error(ctx.h).decode().startswith("vdo_orb_extract_batch_dev"), what
    torch.cuda.synchronize()
    for k in keys:
        assert torch.equal(out[k], snap[k]), f"{k} was written by a refused call"
    # the same arguments, corrected, are accepted
    arr = (capi.DevPlane * 1)(plane())
    assert L.vdo_orb_extract_batch_dev(ex.h_, C.c_int(1), arr, C.byref(outs()), C.c_uint64(stream)) == 0
    torch.cuda.synchronize()
    assert int(out["count"][0]) > 0 and int(out["status"][0]) == 0
