"""Device-resident frame input (vdo_frame_upload_dev / vdo_tracker_track_dev through Frame.upload_tensors / Tracker.track_tensors).

The colour conversion is pinned to cv2.cvtColor, the strided ingest to the host upload, and the whole tracker on device planes to the
tracker on host buffers, bit for bit.  test_tracker_gpu.py pins the host-input tracker to the oracle pipeline, so identity with it
carries that parity over."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import bgr_to_gray_opencv34, colour_from_gray, make_frame, make_sequence_frame

pytestmark = pytest.mark.gpu
BF, FACTOR = 387.5744, 256.0
DEV = torch.device("cuda", 0)
ERR_ARG = -2

GET_NAMES = ("Tcw", "mVelocity", "mvKeys", "mvStatKeys", "mvStatKeysTmp", "mvStatDepth", "mvStatDepthTmp", "mvCorres", "mvFlowNext", "mvStat3DPointTmp",
             "nStaInlierID", "mvObjKeys", "mvObjDepth", "mvObjCorres", "mvObjFlowNext", "mvObj3DPoint", "vSemObjLabel", "vObjLabel", "nDynInlierID",
             "vFlow_3d", "nModLabel", "nSemPosition", "TemperalMatch_subset", "bObjStat", "vObjCentre3D", "vObjMod", "max_id", "f_id", "local_ba")
MAP_NAMES = ("vmCameraPose", "vmCameraPose_RF", "vmRigidMotion", "vmRigidMotion_RF", "vmRigidCentre", "n_per_frame", "vp3DPointSta", "vp3DPointDyn",
             "vnRMLabel", "n_frames")


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.fixture(scope="module")
def sequence():
    """config-3-shaped sequence (1242x375, seed 0), 11 frames"""
    return [make_sequence_frame(t, seed=0) for t in range(11)]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _crop(t, pad=(3, 5)):
    """the same values as a view into a larger tensor (row stride larger than the width, non-zero offset) over the first two dims"""
    shape = list(t.shape)
    big = torch.zeros([shape[0] + 2 * pad[0], shape[1] + 2 * pad[1]] + shape[2:], dtype=t.dtype, device=t.device)
    v = big[pad[0]:pad[0] + shape[0], pad[1]:pad[1] + shape[1]]
    v.copy_(t)
    return v


def _crop_chw(t):
    """a planar (C,H,W) tensor as a view into a larger one"""
    c, h, w = t.shape
    big = torch.zeros((c, h + 4, w + 6), dtype=t.dtype, device=t.device)
    v = big[:, 2:2 + h, 3:3 + w]
    v.copy_(t)
    return v


def _image_layouts(hwc):
    """HWC, CHW (contiguous and as a permuted view), and crops of both"""
    t = _dev(hwc)
    chw = t.permute(2, 0, 1).contiguous()
    return {"hwc": t, "chw": chw, "chw_view": t.permute(2, 0, 1), "hwc_crop": _crop(t), "chw_crop": _crop_chw(chw)}


def _resident_gray(F):
    F.orb_extract()
    return F.debug_level(0)[0]                     # level 0 of the pyramid is the resident gray image


# ------------------------------------------------------------------------------------------------ 1. colour conversion
@pytest.mark.parametrize("w,h", [(1242, 375), (641, 257)])
@pytest.mark.parametrize("fmt", ["GRAY", "RGB", "BGR", "RGBA", "BGRA"])
def test_colour_conversion_matches_opencv(ctx, w, h, fmt):
    """Bit for bit the fixed point of the OpenCV the reference builds (3.4, the same formula as the System shim); cv2 4.x's 15-bit
    coefficients may differ by one grey level on under 1 % of the pixels (tests/test_converter.py pins that drift)."""
    rng = np.random.default_rng(w * 10 + len(fmt))
    F = capi.Frame(ctx, w, h)
    if fmt == "GRAY":
        ref = cv = rng.integers(0, 256, (h, w), dtype=np.uint8)
        t = _dev(ref)
        views, rgb = {"hw": t, "hw_crop": _crop(t)}, True
    else:
        img = rng.integers(0, 256, (h, w, len(fmt)), dtype=np.uint8)
        rgb = fmt.startswith("RGB")
        ref = bgr_to_gray_opencv34(img, rgb=rgb)
        cv = cv2.cvtColor(img, getattr(cv2, f"COLOR_{fmt}2GRAY"))
        views = _image_layouts(img)
    for name, v in views.items():
        F.upload(gray=np.zeros((h, w), np.uint8))                  # nothing of the previous layout may survive
        F.upload_tensors(image=v, rgb=rgb)
        got = _resident_gray(F)
        assert np.array_equal(got, ref), f"{fmt} {name}: {int((got != ref).sum())} pixels differ from the OpenCV 3.4 conversion"
        diff = np.abs(got.astype(np.int16) - cv)
        assert diff.max() <= 1 and (diff != 0).mean() < 0.01, f"{fmt} {name}: against cv2.cvtColor"


# ------------------------------------------------------------------------------------------------ 2. strided ingest
def _frame_outputs(F):
    d = F.depth_prep(BF, FACTOR)
    kp = F.orb_extract()
    st = F.filter_static(kp["x"], kp["y"], 40.0)
    so = F.sample_objects(25.0)
    return d, st, so


def _assert_outputs_equal(a, b, what):
    assert np.array_equal(a[0], b[0]), f"{what}: depth_prep"
    for x, y in zip(a[1], b[1]):
        assert np.array_equal(x, y), f"{what}: filter_static"
    for k in a[2]:
        assert np.array_equal(a[2][k], b[2][k]), f"{what}: sample_objects {k}"


def test_device_ingest_equals_host_upload(ctx):
    f = make_frame(7)
    H, W = f["gray"].shape
    Fh = capi.Frame(ctx, W, H)
    Fh.upload(gray=f["gray"], depth=f["depth_raw"], flow=f["flow"], mask=f["mask"])
    ref = _frame_outputs(Fh)
    assert len(ref[1][0]) > 100 and len(ref[2]["x"]) > 100         # both selections are populated
    g, d, fl, m = _dev(f["gray"]), _dev(f["depth_raw"]), _dev(f["flow"]), _dev(f["mask"])
    fl_2hw = fl.permute(2, 0, 1).contiguous()
    m64 = m.to(torch.int64)
    wide = torch.zeros((H, 2 * W), dtype=torch.int32, device=DEV)
    m_step2 = wide[:, ::2]                                           # x stride 2
    m_step2.copy_(m)
    variants = {
        "contiguous, flow HW2, mask i32": (d, fl, m),
        "contiguous, flow 2HW, mask i64": (d, fl_2hw, m64),
        "crops, flow HW2 crop, mask i64 crop": (_crop(d), _crop(fl), _crop(m64)),
        "depth crop, flow 2HW view of HW2, mask i32 x-stride 2": (_crop(d), fl.permute(2, 0, 1), m_step2),
        "flow 2HW crop, mask i32 crop": (d, _crop_chw(fl_2hw), _crop(m)),
    }
    for what, (dv, fv, mv) in variants.items():
        Fd = capi.Frame(ctx, W, H)
        Fd.upload_tensors(image=g, depth=dv, flow=fv, mask=mv)
        _assert_outputs_equal(_frame_outputs(Fd), ref, what)
    # a NULL plane keeps what is resident
    Fp = capi.Frame(ctx, W, H)
    Fp.upload(gray=f["gray"], flow=f["flow"])
    Fp.upload_tensors(depth=d, mask=m)
    _assert_outputs_equal(_frame_outputs(Fp), ref, "depth + mask only")


# ------------------------------------------------------------------------------------------------ 3. whole tracker
def _device_inputs(t, bgr, f):
    """rotate layouts per frame: BGR HWC (rgb=False), RGB CHW, BGRA HWC crop; flow HW2 / 2HW; mask i32 / i64; some planes as crops"""
    k = t % 3
    if k == 0:
        img, rgb = _dev(bgr), False
    elif k == 1:
        img, rgb = _dev(np.ascontiguousarray(bgr[..., ::-1].transpose(2, 0, 1))), True
    else:
        img, rgb = _crop(_dev(cv2.cvtColor(bgr, cv2.COLOR_BGR2BGRA))), False
    fl = _dev(f["flow"])
    if t % 2:
        fl = fl.permute(2, 0, 1).contiguous()
    d = _dev(f["depth_raw"])
    if t % 4 >= 2:
        d = _crop(d)
    m = _dev(f["mask"]).to(torch.int64 if (t // 2) % 2 else torch.int32)
    if t % 3 == 2:
        m = _crop(m)
    return img, rgb, d, fl, m


def _assert_trackers_equal(td, th, t):
    for name in GET_NAMES:
        np.testing.assert_array_equal(td.get(name), th.get(name), err_msg=f"frame {t}: {name}")


def test_tracker_device_input_equals_host_input(ctx, sequence):
    """11 frames, WINDOW 6 / OVERLAP 2 (the windowed BA runs twice inside the loop).  Mid-sequence, frames the device tracker must refuse
    (an i64 label of 2**31, a zero-stride write-back target, a size mismatch) are offered first; the sequence must go on as if they never came."""
    H, W = sequence[0]["gray"].shape
    td = capi.Tracker(ctx, window_size=6, overlap_size=2)
    th = capi.Tracker(ctx, window_size=6, overlap_size=2)
    for t, f in enumerate(sequence):
        bgr = colour_from_gray(f["gray"], seed=t)                           # the host tracker gets cv2.cvtColor of it: the same gray
        img, rgb, d, fl, m = _device_inputs(t, bgr, f)
        if t in (0, 4, 7):
            bad = m.to(torch.int64).clone()
            bad[H // 2, W // 3] = 2 ** 31
            d_before = d.clone()
            with pytest.raises(capi.VdoError, match=r"\(-2\).*int32"):
                td.track_tensors(img, d, fl, bad, f["obj_ids"], rgb=rgb)
            assert torch.equal(d, d_before)                                  # a refused frame writes nothing back
            with pytest.raises(capi.VdoError, match=r"\(-2\).*stride"):
                td.track_tensors(img, d, fl, torch.zeros(W, dtype=torch.int32, device=DEV).expand(H, W), f["obj_ids"], rgb=rgb)
            planes = [capi._dev_plane(ctx, k, v, W, H, rgb) for k, v in (("image", img), ("depth", d), ("flow", fl), ("mask", m))]
            T = np.zeros((4, 4), np.float32)
            rc = ctx.L.vdo_tracker_track_dev(td.h_, C.c_int(W + 1), C.c_int(H), *[C.byref(p) for p in planes], C.c_int(0), None, C.c_int(1), C.c_uint64(0),
                                             T.ctypes.data_as(C.POINTER(C.c_float)))
            assert rc == ERR_ARG
        d_host, m_host = f["depth_raw"].copy(), f["mask"].copy()
        T_h = th.track(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), d_host, f["flow"], m_host, f["obj_ids"], writeback=True)
        T_d = td.track_tensors(img, d, fl, m, f["obj_ids"], writeback=True, rgb=rgb)
        assert np.array_equal(T_d, T_h), f"frame {t}: Tcw"
        _assert_trackers_equal(td, th, t)
        assert np.array_equal(d.cpu().numpy(), d_host), f"frame {t}: written-back depth"
        assert np.array_equal(m.cpu().numpy(), m_host), f"frame {t}: written-back mask"
    assert td.get("local_ba")[0] == 2
    for name in MAP_NAMES:
        np.testing.assert_array_equal(td.map_get(name), th.map_get(name), err_msg=name)
    # the full batch: its graph is the same bit for bit; the solve sums with double atomics, so two runs on one graph may differ in the
    # last bits (up to 7e-12 seen on an H100 with the graphs asserted identical here)
    gd, gh = td.graph_export(1), th.graph_export(1)
    for k in gh:
        np.testing.assert_array_equal(gd[k], gh[k], err_msg=f"full-batch graph: {k}")
    rd, rh = td.batch_optimize(1), th.batch_optimize(1)
    assert rd["iterations"] == rh["iterations"]
    for name in ("vmCameraPose_RF", "vmRigidMotion_RF"):
        assert np.abs(td.map_get(name) - th.map_get(name)).max() <= 1e-8, name


# ------------------------------------------------------------------------------------------------ 4. stream ordering
def test_inputs_produced_on_a_side_stream_are_seen_without_a_synchronise(ctx, sequence):
    H, W = sequence[0]["gray"].shape
    td = capi.Tracker(ctx)
    th = capi.Tracker(ctx)
    side = torch.cuda.Stream(DEV)
    junk = torch.ones(1 << 27, device=DEV)                                 # 512 MB of element-wise work queued before the inputs
    for t, f in enumerate(sequence[:4]):
        src = [_dev(f["gray"]), _dev(f["depth_raw"]), _dev(f["flow"]).permute(2, 0, 1).contiguous(), _dev(f["mask"]).to(torch.int64)]
        dst = [torch.full_like(s, 7) for s in src]                         # wrong values until the side stream's copies land
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            for _ in range(6):
                junk.mul_(1.0001).add_(0.5)
            for a, b in zip(dst, src):
                a.copy_(b)
            T_d = td.track_tensors(*dst, f["obj_ids"], writeback=True)
            d_dev, m_dev = dst[1].cpu().numpy(), dst[3].cpu().numpy()
        d_host, m_host = f["depth_raw"].copy(), f["mask"].copy()
        T_h = th.track(f["gray"], d_host, f["flow"], m_host, f["obj_ids"], writeback=True)
        assert np.array_equal(T_d, T_h), f"frame {t}: Tcw"
        _assert_trackers_equal(td, th, t)
        assert np.array_equal(d_dev, d_host) and np.array_equal(m_dev, m_host), f"frame {t}: write-back"
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 5. refusals
def _plane(data_ptr, dtype, channels, sy, sx, sc=0, rgb=1):
    return capi.DevPlane(data_ptr, dtype, channels, sy, sx, sc, rgb)


def test_refusals(ctx):
    W, H = 320, 240
    F = capi.Frame(ctx, W, H)
    tr = capi.Tracker(ctx, width=W, height=H, cx=160.0, cy=110.0)
    img = torch.zeros((H, W, 3), dtype=torch.uint8, device=DEV)
    d = torch.ones((H, W), device=DEV)
    fl = torch.zeros((H, W, 2), device=DEV)
    m = torch.zeros((H, W), dtype=torch.int32, device=DEV)
    # Python: CPU tensors, wrong dtype / shape / layout
    for kw in (dict(depth=d.cpu()), dict(depth=d.double()), dict(depth=d[:-1]), dict(mask=m.float()), dict(flow=fl[..., :1]), dict(image=img[..., :2]),
               dict(image=img.float()), dict(flow=np.zeros((H, W, 2), np.float32))):
        with pytest.raises(ValueError):
            F.upload_tensors(**kw)
    with pytest.raises(ValueError):
        tr.track_tensors(img.cpu(), d, fl, m, [])
    # C ABI: host memory (pinned and pageable) is not device memory
    pinned = torch.zeros((H, W), device="cpu").pin_memory()
    pageable = np.zeros((H, W), np.float32)
    for ptr in (pinned.data_ptr(), pageable.ctypes.data):
        p = _plane(ptr, capi.VDO_DT_F32, 1, W, 1)
        assert ctx.L.vdo_frame_upload_dev(F.h_, None, C.byref(p), None, None, C.c_uint64(0)) == ERR_ARG
    assert "device memory" in ctx.L.vdo_last_error(ctx.h).decode()
    # C ABI: dtype / channel combinations outside the accepted set, and a misaligned pointer
    bad = [("image", _plane(img.data_ptr(), capi.VDO_DT_F32, 3, 3 * W, 3, 1)), ("image", _plane(img.data_ptr(), capi.VDO_DT_U8, 2, 3 * W, 3, 1)),
           ("depth", _plane(d.data_ptr(), capi.VDO_DT_F32, 2, W, 1, 1)), ("depth", _plane(d.data_ptr(), capi.VDO_DT_I32, 1, W, 1)),
           ("flow", _plane(fl.data_ptr(), capi.VDO_DT_F32, 1, 2 * W, 2)), ("flow", _plane(fl.data_ptr(), capi.VDO_DT_I64, 2, 2 * W, 2, 1)),
           ("mask", _plane(m.data_ptr(), capi.VDO_DT_U8, 1, W, 1)), ("mask", _plane(m.data_ptr(), capi.VDO_DT_I32, 2, W, 1, 1)),
           ("mask", _plane(m.data_ptr() + 2, capi.VDO_DT_I32, 1, W, 1)), ("depth", _plane(0, capi.VDO_DT_F32, 1, W, 1))]
    order = ("image", "depth", "flow", "mask")
    for kind, p in bad:
        args = [C.byref(p) if k == kind else None for k in order]
        assert ctx.L.vdo_frame_upload_dev(F.h_, *args, C.c_uint64(0)) == ERR_ARG, kind
    # C ABI: width / height mismatch, missing planes
    good = [capi._dev_plane(ctx, k, v, W, H) for k, v in zip(order, (img, d, fl, m))]
    T = np.zeros((4, 4), np.float32)
    Tp = T.ctypes.data_as(C.POINTER(C.c_float))
    for w, h in ((W - 1, H), (W, H + 1)):
        assert ctx.L.vdo_tracker_track_dev(tr.h_, C.c_int(w), C.c_int(h), *[C.byref(p) for p in good], C.c_int(0), None, C.c_int(0), C.c_uint64(0), Tp) == ERR_ARG
    args = [C.byref(p) for p in good]
    args[2] = None
    assert ctx.L.vdo_tracker_track_dev(tr.h_, C.c_int(W), C.c_int(H), *args, C.c_int(0), None, C.c_int(0), C.c_uint64(0), Tp) == ERR_ARG
    # zero-stride write-back targets; the same broadcast planes are fine as inputs only
    with pytest.raises(capi.VdoError, match=r"\(-2\)"):
        tr.track_tensors(img, d, fl, torch.zeros(W, dtype=torch.int32, device=DEV).expand(H, W), [], writeback=True)
    with pytest.raises(capi.VdoError, match=r"\(-2\)"):
        tr.track_tensors(img, torch.ones(H, 1, device=DEV).expand(H, W), fl, m, [], writeback=True)
    assert int(tr.get("f_id")[0]) == 0 and len(tr.map_get("vmCameraPose")) == 0           # nothing above reached the tracker's state
    tr.track_tensors(img, d, fl, torch.zeros(W, dtype=torch.int32, device=DEV).expand(H, W), [], writeback=False)
    assert len(tr.map_get("vmCameraPose")) == 16
