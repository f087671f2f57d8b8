"""Several sequences in one call (vdo_tracker_track_batch_dev through capi.track_tensors_batch): every tracker of a batch must end up
exactly where separate vdo_tracker_track_dev calls take it, bit for bit, whatever point of its sequence it is at, and a refused batch
must leave every tracker as it was.  test_device_input_gpu.py pins the single-tracker device path to the host path."""
import ctypes as C

import numpy as np
import pytest
import torch

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_sequence_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG, ERR_STATE = -2, -4
BF = 387.5744

GET_NAMES = ("Tcw", "mVelocity", "mvKeys", "mvStatKeys", "mvStatKeysTmp", "mvStatDepth", "mvStatDepthTmp", "mvCorres", "mvFlowNext", "mvStat3DPointTmp",
             "nStaInlierID", "mvObjKeys", "mvObjDepth", "mvObjCorres", "mvObjFlowNext", "mvObj3DPoint", "vSemObjLabel", "vObjLabel", "nDynInlierID",
             "vFlow_3d", "nModLabel", "nSemPosition", "TemperalMatch_subset", "bObjStat", "vObjCentre3D", "vObjMod", "max_id", "f_id", "local_ba")
MAP_NAMES = ("vmCameraPose", "vmCameraPose_RF", "vmRigidMotion", "vmRigidMotion_RF", "vmRigidCentre", "n_per_frame", "vp3DPointSta", "vp3DPointDyn",
             "vnRMLabel", "n_frames")

# three sequences that differ in seed, intrinsics, ThDepthBG, dataset (the second is VirtualKITTI: metric depth, no disparity conversion)
# and window, so the windowed optimisation fires on different steps
SEQS = (dict(seed=0, K=None, params=dict(th_depth_bg=40.0, window_size=6, overlap_size=2)),
        dict(seed=1, K=(700.0, 705.0, 600.0, 180.0), params=dict(th_depth_bg=35.0, dataset=3, window_size=8, overlap_size=3)),
        dict(seed=2, K=(730.0, 730.0, 615.0, 170.0), params=dict(th_depth_bg=45.0, window_size=6, overlap_size=2)))
N_FRAMES = 14


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.fixture(scope="module")
def frames():
    out = []
    for s in SEQS:
        seq = [make_sequence_frame(t, seed=s["seed"], K=s["K"]) for t in range(N_FRAMES)]
        if s["params"].get("dataset") == 3:
            for f in seq:
                raw = f["depth_raw"]
                f["depth_raw"] = np.where(raw > 0, np.float32(BF) / (raw / np.float32(256.0)), raw).astype(np.float32)
        out.append(seq)
    return out


def _tracker(ctx, s):
    kw = dict(s["params"])
    if s["K"] is not None:
        kw.update(fx=s["K"][0], fy=s["K"][1], cx=s["K"][2], cy=s["K"][3])
    return capi.Tracker(ctx, **kw)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _crop(t, pad=(3, 5)):
    shape = list(t.shape)
    big = torch.zeros([shape[0] + 2 * pad[0], shape[1] + 2 * pad[1]] + shape[2:], dtype=t.dtype, device=t.device)
    v = big[pad[0]:pad[0] + shape[0], pad[1]:pad[1] + shape[1]]
    v.copy_(t)
    return v


def _inputs(f, t, i):
    """fresh device inputs of one frame, layouts rotated by frame and sequence: gray HW / RGB CHW / BGR HWC crop, flow HW2 / 2HW,
    mask i32 / i64 (some cropped), depth contiguous / cropped"""
    k = (t + i) % 3
    g = f["gray"]
    if k == 0:
        img, rgb = _dev(g), True
    elif k == 1:
        img, rgb = _dev(np.stack([g, g, g])), True
    else:
        img, rgb = _crop(_dev(np.stack([g, g, g], axis=-1))), False
    fl = _dev(f["flow"])
    if (t + i) % 2:
        fl = fl.permute(2, 0, 1).contiguous()
    d = _dev(f["depth_raw"])
    if (t + i) % 4 >= 2:
        d = _crop(d)
    m = _dev(f["mask"]).to(torch.int64 if (t + i) // 2 % 2 else torch.int32)
    if (t + i) % 3 == 2:
        m = _crop(m)
    return img, rgb, d, fl, m


def _batch(trackers, ins, gts):
    """one track_tensors_batch call; the image layouts differ per element, so all take the gray value from one rgb flag per call when the
    layouts agree -- here every colour image is a gray replica, so rgb does not change the result"""
    return capi.track_tensors_batch(trackers, [x[0] for x in ins], [x[2] for x in ins], [x[3] for x in ins], [x[4] for x in ins], gts)


def _alone(tr, inp, gt):
    img, rgb, d, fl, m = inp
    return tr.track_tensors(img, d, fl, m, gt, rgb=rgb)


def _assert_same(tb, ts, what):
    for name in GET_NAMES:
        np.testing.assert_array_equal(tb.get(name), ts.get(name), err_msg=f"{what}: {name}")


def _assert_maps_same(tb, ts, what):
    for name in MAP_NAMES:
        np.testing.assert_array_equal(tb.map_get(name), ts.map_get(name), err_msg=f"{what}: {name}")
    gb, gs = tb.graph_export(1), ts.graph_export(1)
    for k in gs:
        np.testing.assert_array_equal(gb[k], gs[k], err_msg=f"{what}: full-batch graph {k}")


def test_batch_equals_separate_trackers(ctx, frames):
    B = len(SEQS)
    tb = [_tracker(ctx, s) for s in SEQS]
    ts = [_tracker(ctx, s) for s in SEQS]
    for t in range(N_FRAMES):
        fr = [frames[i][t] for i in range(B)]
        ins_b = [_inputs(fr[i], t, i) for i in range(B)]
        ins_s = [_inputs(fr[i], t, i) for i in range(B)]
        Tb = _batch(tb, ins_b, [f["obj_ids"] for f in fr])
        for i in range(B):
            Ts = _alone(ts[i], ins_s[i], fr[i]["obj_ids"])
            assert np.array_equal(Tb[i], Ts), f"frame {t} sequence {i}: Tcw"
            _assert_same(tb[i], ts[i], f"frame {t} sequence {i}")
            assert torch.equal(ins_b[i][2], ins_s[i][2]), f"frame {t} sequence {i}: written-back depth"
            assert torch.equal(ins_b[i][4], ins_s[i][4]), f"frame {t} sequence {i}: written-back mask"
    runs = [int(tb[i].get("local_ba")[0]) for i in range(B)]
    assert runs[0] >= 2 and runs[1] >= 1 and runs[0] != runs[1]           # the windows fire on different steps
    for i in range(B):
        _assert_maps_same(tb[i], ts[i], f"sequence {i}")
        st = tb[i].get("stage_ms")
        assert np.all(st[:8] > 0), f"sequence {i}: every batched stage is timed"


def test_staggered_starts(ctx, frames):
    """tracker 2 joins at step 3 (its first frame inside a batch call); tracker 1 is tracked alone at steps 5 and 6 and rejoins at 7"""
    B = len(SEQS)
    tb = [_tracker(ctx, s) for s in SEQS]
    ts = [_tracker(ctx, s) for s in SEQS]
    pos = [0] * B
    for step in range(10):
        members = [i for i in range(B) if not (i == 2 and step < 3)]
        alone = [i for i in members if i == 1 and step in (5, 6)]
        batch = [i for i in members if i not in alone]
        ins_b = {i: _inputs(frames[i][pos[i]], pos[i], i) for i in members}
        ins_s = {i: _inputs(frames[i][pos[i]], pos[i], i) for i in members}
        Tb = _batch([tb[i] for i in batch], [ins_b[i] for i in batch], [frames[i][pos[i]]["obj_ids"] for i in batch])
        for i in alone:
            _alone(tb[i], ins_b[i], frames[i][pos[i]]["obj_ids"])
        for i in members:
            Ts = _alone(ts[i], ins_s[i], frames[i][pos[i]]["obj_ids"])
            if i in batch:
                assert np.array_equal(Tb[batch.index(i)], Ts), f"step {step} sequence {i}: Tcw"
            _assert_same(tb[i], ts[i], f"step {step} sequence {i}")
            assert torch.equal(ins_b[i][2], ins_s[i][2]) and torch.equal(ins_b[i][4], ins_s[i][4]), f"step {step} sequence {i}: write-back"
            pos[i] += 1
    for i in range(B):
        _assert_maps_same(tb[i], ts[i], f"sequence {i}")


def test_refused_batch_changes_no_tracker(ctx, frames):
    B = len(SEQS)
    tb = [_tracker(ctx, s) for s in SEQS]
    ts = [_tracker(ctx, s) for s in SEQS]
    H, W = frames[0][0]["gray"].shape
    for t in range(6):
        fr = [frames[i][t] for i in range(B)]
        if t == 3:
            ins = [_inputs(fr[i], t, i) for i in range(B)]
            bad = ins[1][4].to(torch.int64).clone()
            bad[H // 2, W // 3] = 2 ** 31
            ins[1] = ins[1][:4] + (bad,)
            before = [(tr.get("f_id").copy(), tr.get("Tcw").copy(), tr.get("mvKeys").copy(), len(tr.map_get("vmCameraPose"))) for tr in tb]
            d_before = [x[2].clone() for x in ins]
            m_before = [x[4].clone() for x in ins]
            with pytest.raises(capi.VdoError, match=r"\(-2\).*trackers\[1\].*int32"):
                _batch(tb, ins, [f["obj_ids"] for f in fr])
            for i, tr in enumerate(tb):
                f_id, Tcw, keys, n_map = before[i]
                assert np.array_equal(tr.get("f_id"), f_id) and np.array_equal(tr.get("Tcw"), Tcw) and np.array_equal(tr.get("mvKeys"), keys)
                assert len(tr.map_get("vmCameraPose")) == n_map
                assert torch.equal(ins[i][2], d_before[i]) and torch.equal(ins[i][4], m_before[i]), f"sequence {i}: a refused call writes nothing back"
        ins_b = [_inputs(fr[i], t, i) for i in range(B)]
        Tb = _batch(tb, ins_b, [f["obj_ids"] for f in fr])
        for i in range(B):
            Ts = _alone(ts[i], _inputs(fr[i], t, i), fr[i]["obj_ids"])
            assert np.array_equal(Tb[i], Ts), f"frame {t} sequence {i}: Tcw"
            _assert_same(tb[i], ts[i], f"frame {t} sequence {i}")


def test_refused_orb_settings_change_no_tracker(ctx, frames):
    """n_features = 50 000 gives level 0 an octree capacity over the extractor's 8192: the frame build's extractor refuses the settings,
    and the batch is refused before any tracker or input changes"""
    B = len(SEQS)
    tb = [_tracker(ctx, dict(s, params=dict(s["params"], n_features=50000))) for s in SEQS]
    fr = [frames[i][0] for i in range(B)]
    ins = [_inputs(fr[i], 0, i) for i in range(B)]
    before = [(tr.get("f_id").copy(), tr.get("Tcw").copy(), tr.get("mvKeys").copy(), len(tr.map_get("vmCameraPose"))) for tr in tb]
    d_before = [x[2].clone() for x in ins]
    m_before = [x[4].clone() for x in ins]
    with pytest.raises(capi.VdoError, match=r"\(-3\).*ORB"):
        _batch(tb, ins, [f["obj_ids"] for f in fr])
    with pytest.raises(capi.VdoError, match=r"\(-3\).*ORB"):
        _alone(tb[0], ins[0], fr[0]["obj_ids"])
    for i, tr in enumerate(tb):
        f_id, Tcw, keys, n_map = before[i]
        assert np.array_equal(tr.get("f_id"), f_id) and np.array_equal(tr.get("Tcw"), Tcw) and np.array_equal(tr.get("mvKeys"), keys)
        assert len(tr.map_get("vmCameraPose")) == n_map
        assert torch.equal(ins[i][2], d_before[i]) and torch.equal(ins[i][4], m_before[i]), f"sequence {i}: a refused call writes nothing back"


def _raw_call(ctx, trackers, planes, gt_begin, gt_ids=None):
    B = len(trackers)
    arr = [(capi.DevPlane * B)(*[planes[k] for _ in range(B)]) for k in range(4)]
    handles = (C.c_void_p * B)(*[t.h_.value for t in trackers])
    gb = np.asarray(gt_begin, np.int32)
    gi = np.asarray(gt_ids if gt_ids is not None else [0], np.int32)
    T = np.zeros((B, 4, 4), np.float32)
    return ctx.L.vdo_tracker_track_batch_dev(handles, C.c_int(B), *arr, gb.ctypes.data_as(C.POINTER(C.c_int)), gi.ctypes.data_as(C.POINTER(C.c_int)),
                                             C.c_int(0), C.c_uint64(0), T.ctypes.data_as(C.POINTER(C.c_float)))


def test_argument_refusals(ctx):
    W, H = 320, 240
    mk = lambda c=ctx, **kw: capi.Tracker(c, width=W, height=H, cx=160.0, cy=110.0, **kw)
    a, b = mk(), mk()
    img = torch.zeros((H, W), dtype=torch.uint8, device=DEV)
    d = torch.ones((H, W), device=DEV)
    fl = torch.zeros((H, W, 2), device=DEV)
    m = torch.zeros((H, W), dtype=torch.int32, device=DEV)
    planes = [capi._dev_plane(ctx, k, v, W, H) for k, v in (("image", img), ("depth", d), ("flow", fl), ("mask", m))]
    cases = {
        "duplicate": ([a, b, a], [0, 0, 0, 0], ERR_ARG, "repeats"),
        "two contexts": ([a, mk(capi.Context(0))], [0, 0, 0], ERR_ARG, "context"),
        "map-only": ([a, capi.Tracker(ctx, width=0, height=0)], [0, 0, 0], ERR_STATE, "map-only"),
        "width": ([a, capi.Tracker(ctx, width=W + 2, height=H)], [0, 0, 0], ERR_ARG, "ORB settings"),
        "ORB settings": ([a, mk(n_features=2000)], [0, 0, 0], ERR_ARG, "ORB settings"),
        "gt_begin not from 0": ([a, b], [1, 1, 1], ERR_ARG, "gt_begin"),
        "gt_begin decreasing": ([a, b], [0, 2, 1], ERR_ARG, "gt_begin"),
    }
    for what, (trs, gb, rc, msg) in cases.items():
        assert _raw_call(ctx, trs, planes, gb, [1, 2]) == rc, what
        assert msg in ctx.L.vdo_tracker_last_error(trs[0].h_).decode(), what
    assert int(a.get("f_id")[0]) == 0 and len(a.map_get("vmCameraPose")) == 0 and len(b.map_get("vmCameraPose")) == 0
    with pytest.raises(ValueError):
        capi.track_tensors_batch([a, b], [img], [d, d], [fl, fl], [m, m], [[], []])
    with pytest.raises(ValueError):
        capi.track_tensors_batch([a, b], torch.stack([img, img]), torch.stack([d, d]), [fl, fl], [m, m], [[]])
    T = capi.track_tensors_batch([a, b], torch.stack([img, img]), torch.stack([d, d]), torch.stack([fl, fl]), torch.stack([m, m]), [[], []], writeback=False)
    assert T.shape == (2, 4, 4) and len(a.map_get("vmCameraPose")) == 16 and len(b.map_get("vmCameraPose")) == 16


def test_batch_of_one_equals_track_tensors(ctx, frames):
    s = SEQS[2]
    tb, ts = _tracker(ctx, s), _tracker(ctx, s)
    for t in range(5):
        f = frames[2][t]
        ib, is_ = _inputs(f, t, 2), _inputs(f, t, 2)
        Tb = capi.track_tensors_batch([tb], [ib[0]], [ib[2]], [ib[3]], [ib[4]], [f["obj_ids"]], rgb=ib[1])
        Ts = _alone(ts, is_, f["obj_ids"])
        assert np.array_equal(Tb[0], Ts), f"frame {t}: Tcw"
        _assert_same(tb, ts, f"frame {t}")
        assert torch.equal(ib[2], is_[2]) and torch.equal(ib[4], is_[4]), f"frame {t}: write-back"
