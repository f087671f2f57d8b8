"""Sequences of different image sizes and ORB settings in one call (vdo_tracker_track_mixed_dev through capi.track_tensors_mixed): every
tracker of a mixed batch must end up exactly where separate vdo_tracker_track_dev calls take it, bit for bit, whatever its size, its ORB
settings and the point of its sequence it is at; a batch of one geometry must give what track_tensors_batch gives; and a refused call
must leave every tracker and every input as it was."""
import ctypes as C

import numpy as np
import pytest
import torch

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_sequence_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG, ERR_STATE = -2, -4

GET_NAMES = ("Tcw", "mVelocity", "mvKeys", "mvStatKeys", "mvStatKeysTmp", "mvStatDepth", "mvStatDepthTmp", "mvCorres", "mvFlowNext", "mvStat3DPointTmp",
             "nStaInlierID", "mvObjKeys", "mvObjDepth", "mvObjCorres", "mvObjFlowNext", "mvObj3DPoint", "vSemObjLabel", "vObjLabel", "nDynInlierID",
             "vFlow_3d", "nModLabel", "nSemPosition", "TemperalMatch_subset", "bObjStat", "vObjCentre3D", "vObjMod", "max_id", "f_id", "local_ba")
MAP_NAMES = ("vmCameraPose_RF", "vmRigidMotion_RF", "vmRigidCentre", "n_per_frame", "vnRMLabel", "n_frames")
# what the windowed optimisations write back: the batch solver sums with fp64 atomics, so two solves of one window already differ in the
# last bits (test_full_batch_gpu.py), and these are compared at its tolerance
SOLVED_NAMES = ("vmCameraPose", "vmRigidMotion", "vp3DPointSta", "vp3DPointDyn")
OMD_K = (618.3587036132812, 618.5924072265625, 328.9866333007812, 237.7507629394531)

# Four geometries: KITTI (option I), KITTI-like one pixel off in each direction with other intrinsics, OMD (640x480, 3 000 features,
# sampled background features, DepthMapFactor 1000), and a size of its own with other n_levels, scale_factor and FAST thresholds.  They
# start at steps 0, 2, 4 and 1; with these windows the windowed optimisation of the first three fires on the same call (step 9).
SEQS = (dict(seed=0, w=1242, h=375, K=None, start=0, params=dict(n_features=2500, window_size=6, overlap_size=2)),
        dict(seed=1, w=1241, h=376, K=(700.0, 705.0, 600.0, 180.0), start=2, params=dict(th_depth_bg=35.0, window_size=8, overlap_size=3)),
        dict(seed=2, w=640, h=480, K=OMD_K, start=4, factor=1000.0,
             params=dict(n_features=3000, use_sample_feature=1, sample_seed=7, dataset=1, is_kitti=0, sf_mg_thres=0.02, sf_ds_thres=0.99,
                         window_size=6, overlap_size=2)),
        dict(seed=3, w=960, h=400, K=(650.0, 650.0, 470.0, 190.0), start=1,
             params=dict(n_features=2000, n_levels=6, scale_factor=1.3, ini_th_fast=15, min_th_fast=5, window_size=10, overlap_size=4)))
N_STEPS = 32


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def _frames(s, n):
    out = []
    for t in range(n):
        f = make_sequence_frame(t, seed=s["seed"], width=s["w"], height=s["h"], K=s["K"])
        if "factor" in s:                       # the synthetic depth is disparity * 256: rescale it to this DepthMapFactor
            raw = f["depth_raw"]
            f["depth_raw"] = np.where(raw > 0, raw * np.float32(s["factor"] / 256.0), raw).astype(np.float32)
        out.append(f)
    return out


def _tracker(ctx, s):
    kw = dict(s["params"], width=s["w"], height=s["h"])
    if s["K"] is not None:
        kw.update(fx=s["K"][0], fy=s["K"][1], cx=s["K"][2], cy=s["K"][3])
    if "factor" in s:
        kw["depth_factor"] = s["factor"]
    return capi.Tracker(ctx, **kw)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _inputs(f, t, i):
    """fresh device inputs of one frame, layouts rotated by frame and sequence: gray HW / gray-replica CHW, flow HW2 / 2HW, mask i32 / i64,
    depth contiguous / a strided view"""
    g = f["gray"]
    img = _dev(g) if (t + i) % 2 == 0 else _dev(np.stack([g, g, g]))
    fl = _dev(f["flow"])
    if (t + i) % 3 == 1:
        fl = fl.permute(2, 0, 1).contiguous()
    d = _dev(f["depth_raw"])
    if (t + i) % 4 >= 2:
        big = torch.zeros((d.shape[0] + 4, d.shape[1] + 6), device=DEV)
        d = big[2:2 + d.shape[0], 3:3 + d.shape[1]]
        d.copy_(_dev(f["depth_raw"]))
    m = _dev(f["mask"]).to(torch.int64 if (t + i) // 2 % 2 else torch.int32)
    return img, d, fl, m


def _mixed(trackers, ins, gts):
    return capi.track_tensors_mixed(trackers, [x[0] for x in ins], [x[1] for x in ins], [x[2] for x in ins], [x[3] for x in ins], gts)


def _alone(tr, inp, gt):
    return tr.track_tensors(*inp, gt)


def _assert_same(ta, tb, what):
    for name in GET_NAMES:
        np.testing.assert_array_equal(ta.get(name), tb.get(name), err_msg=f"{what}: {name}")


def _assert_maps_same(ta, tb, what):
    for name in MAP_NAMES:
        np.testing.assert_array_equal(ta.map_get(name), tb.map_get(name), err_msg=f"{what}: {name}")
    for name in SOLVED_NAMES:
        a, b = ta.map_get(name), tb.map_get(name)
        assert a.shape == b.shape, f"{what}: {name}"
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-5, err_msg=f"{what}: {name}")


def _state(tr):
    return tr.get("f_id").copy(), tr.get("Tcw").copy(), tr.get("mvKeys").copy(), len(tr.map_get("vmCameraPose"))


def _assert_state(tr, st, what):
    f_id, Tcw, keys, n_map = st
    assert np.array_equal(tr.get("f_id"), f_id) and np.array_equal(tr.get("Tcw"), Tcw) and np.array_equal(tr.get("mvKeys"), keys), what
    assert len(tr.map_get("vmCameraPose")) == n_map, what


@pytest.fixture(scope="module")
def seq_frames():
    return [_frames(s, N_STEPS - s["start"]) for s in SEQS]


@pytest.fixture(scope="module")
def mixed_run(ctx, seq_frames):
    """the four sequences with staggered starts, one track_tensors_mixed call per step; each checked step by step against its twin driven
    by track_tensors.  Returns (mixed trackers, twins, windowed optimisations that fired per step)"""
    frames = seq_frames
    tm = [_tracker(ctx, s) for s in SEQS]
    ts = [_tracker(ctx, s) for s in SEQS]
    fired = []
    for step in range(N_STEPS):
        live = [i for i, s in enumerate(SEQS) if step >= s["start"]]
        pos = {i: step - SEQS[i]["start"] for i in live}
        ins_m = [_inputs(frames[i][pos[i]], pos[i], i) for i in live]
        ins_s = [_inputs(frames[i][pos[i]], pos[i], i) for i in live]
        runs0 = [int(tm[i].get("local_ba")[0]) for i in live]
        Tm = _mixed([tm[i] for i in live], ins_m, [frames[i][pos[i]]["obj_ids"] for i in live])
        fired.append([i for i, r0 in zip(live, runs0) if int(tm[i].get("local_ba")[0]) > r0])
        for j, i in enumerate(live):
            what = f"step {step} sequence {i} ({SEQS[i]['w']}x{SEQS[i]['h']})"
            Ts = _alone(ts[i], ins_s[j], frames[i][pos[i]]["obj_ids"])
            assert np.array_equal(Tm[j], Ts), f"{what}: Tcw"
            _assert_same(tm[i], ts[i], what)
            assert torch.equal(ins_m[j][1], ins_s[j][1]), f"{what}: written-back depth"
            assert torch.equal(ins_m[j][3], ins_s[j][3]), f"{what}: written-back mask"
    return tm, ts, fired


def test_each_tracker_equals_tracking_it_alone(mixed_run):
    tm, ts, fired = mixed_run
    assert any(len(f) >= 3 for f in fired), f"windows of several trackers fire on one call: {fired}"
    for i in range(len(SEQS)):
        assert int(tm[i].get("local_ba")[0]) >= 2, f"sequence {i}: windowed optimisations"
        assert len(tm[i].get("mvKeys")) > 0, f"sequence {i}: keypoints"
        _assert_maps_same(tm[i], ts[i], f"sequence {i}")
        assert np.all(tm[i].get("stage_ms")[:8] > 0), f"sequence {i}: every batched stage is timed"


@pytest.fixture(scope="module")
def unwindowed(ctx, seq_frames):
    """the four sequences over 20 steps with staggered starts and no windowed optimisation, so that the mixed trackers and their twins
    hold bit-identical maps: mixed through track_tensors_mixed, twins through track_tensors"""
    seqs = [dict(s, params=dict(s["params"], local_batch=0, window_size=6, overlap_size=2)) for s in SEQS]
    tm = [_tracker(ctx, s) for s in seqs]
    ts = [_tracker(ctx, s) for s in seqs]
    for step in range(20):
        live = [i for i, s in enumerate(seqs) if step >= s["start"]]
        fr = [seq_frames[i][step - seqs[i]["start"]] for i in live]
        ins = [_inputs(f, step, i) for f, i in zip(fr, live)]
        Tm = _mixed([tm[i] for i in live], ins, [f["obj_ids"] for f in fr])
        for j, i in enumerate(live):
            assert np.array_equal(Tm[j], _alone(ts[i], _inputs(fr[j], step, i), fr[j]["obj_ids"])), f"step {step} sequence {i}: Tcw"
    for i in range(len(seqs)):
        assert int(tm[i].get("local_ba")[0]) == 0
        for name in MAP_NAMES + SOLVED_NAMES:
            np.testing.assert_array_equal(tm[i].map_get(name), ts[i].map_get(name), err_msg=f"sequence {i}: {name}")
    return tm, ts


@pytest.mark.parametrize("mode", [1, 0])
def test_full_batch_over_the_mixed_set(unwindowed, mode):
    """batch_optimize_trackers over the mixed set against each twin's own batch_optimize, at test_full_batch_gpu.py's tolerances for
    PCG-path graphs"""
    tm, ts = unwindowed
    rs = capi.batch_optimize_trackers(tm, mode)
    r1 = [t.batch_optimize(mode) for t in ts]
    for i, (a, b, r, r0) in enumerate(zip(tm, ts, rs, r1)):
        what = f"mode {mode} tracker {i}"
        for k in SOLVED_NAMES + ("vmCameraPose_RF", "vmRigidMotion_RF"):
            x, y = a.map_get(k), b.map_get(k)
            assert x.shape == y.shape, f"{what}: {k}"
            np.testing.assert_allclose(x, y, rtol=0, atol=1e-5, err_msg=f"{what}: {k}")
        for k in ("iterations", "trials"):
            assert r[k] == r0[k], f"{what}: {k}"
        assert abs(r["pcg_iterations"] - r0["pcg_iterations"]) <= r0["pcg_iterations"] // 1000, f"{what}: pcg_iterations"
        assert r["sizes"] == r0["sizes"]
    if mode == 1:
        assert all(r["pcg_iterations"] > 0 for r in rs)


def test_chunk_of_several_geometries(ctx):
    """70 small trackers of four sizes and two ORB settings in one call: the extractor's 64-frame chunks each hold several geometries"""
    sizes = ((160, 120, 500), (200, 96, 700), (128, 128, 500), (176, 144, 700))
    n, steps = 70, 3
    cfg = []
    for k in range(n):
        w, h, nf = sizes[k % 4]
        cfg.append(dict(seed=100 + k, w=w, h=h, K=(0.9 * w, 0.9 * w, w / 2 - 0.5, h / 2 - 0.5), start=0, params=dict(n_features=nf)))
    frames = [_frames(s, steps) for s in cfg]
    tm = [_tracker(ctx, s) for s in cfg]
    ts = [_tracker(ctx, s) for s in cfg]
    for t in range(steps):
        ins_m = [_inputs(frames[k][t], t, k) for k in range(n)]
        ins_s = [_inputs(frames[k][t], t, k) for k in range(n)]
        Tm = _mixed(tm, ins_m, [frames[k][t]["obj_ids"] for k in range(n)])
        for k in range(n):
            Ts = _alone(ts[k], ins_s[k], frames[k][t]["obj_ids"])
            assert np.array_equal(Tm[k], Ts), f"frame {t} tracker {k}: Tcw"
            _assert_same(tm[k], ts[k], f"frame {t} tracker {k}")
            assert torch.equal(ins_m[k][1], ins_s[k][1]) and torch.equal(ins_m[k][3], ins_s[k][3]), f"frame {t} tracker {k}: write-back"
    assert sum(len(t.get("mvKeys")) > 0 for t in tm) == n


def test_uniform_batch_equals_track_tensors_batch(ctx):
    cfg = [dict(seed=s, w=1242, h=375, K=K, start=0, params=dict(th_depth_bg=th, window_size=6, overlap_size=2))
           for s, K, th in ((0, None, 40.0), (1, (700.0, 705.0, 600.0, 180.0), 35.0), (2, (730.0, 730.0, 615.0, 170.0), 45.0))]
    frames = [_frames(s, 8) for s in cfg]
    tm = [_tracker(ctx, s) for s in cfg]
    tb = [_tracker(ctx, s) for s in cfg]
    for t in range(8):
        ins_m = [_inputs(frames[i][t], t, i) for i in range(3)]
        ins_b = [_inputs(frames[i][t], t, i) for i in range(3)]
        gts = [frames[i][t]["obj_ids"] for i in range(3)]
        Tm = _mixed(tm, ins_m, gts)
        Tb = capi.track_tensors_batch(tb, [x[0] for x in ins_b], [x[1] for x in ins_b], [x[2] for x in ins_b], [x[3] for x in ins_b], gts)
        assert np.array_equal(Tm, Tb), f"frame {t}: Tcw"
        for i in range(3):
            _assert_same(tm[i], tb[i], f"frame {t} sequence {i}")
            assert torch.equal(ins_m[i][1], ins_b[i][1]) and torch.equal(ins_m[i][3], ins_b[i][3]), f"frame {t} sequence {i}: write-back"
    for i in range(3):
        _assert_maps_same(tm[i], tb[i], f"sequence {i}")


def test_refusals_write_nothing(ctx, monkeypatch):
    """an extractor refusal of one tracker's ORB settings and a device-side label-range refusal of one frame, each in an otherwise valid
    mix, leave every tracker and input unchanged; tracking then goes on as if they never came"""
    seqs = SEQS[:3]
    frames = [_frames(s, 5) for s in seqs]
    tm = [_tracker(ctx, s) for s in seqs]
    ts = [_tracker(ctx, s) for s in seqs]
    big = _tracker(ctx, dict(SEQS[3], params=dict(SEQS[3]["params"], n_features=50000)))   # level 0 over the octree's 8192 nodes
    for t in range(5):
        fr = [frames[i][t] for i in range(3)]
        gts = [f["obj_ids"] for f in fr]
        if t in (2, 3):
            trs, ins = list(tm), [_inputs(fr[i], t, i) for i in range(3)]
            if t == 2:
                f4 = _frames(SEQS[3], 1)[0]
                trs.insert(1, big); ins.insert(1, _inputs(f4, 0, 3)); g = list(gts); g.insert(1, f4["obj_ids"])
                match, bad = r"\(-3\).*trackers\[1\].*ORB", big
            else:
                m = ins[2][3].to(torch.int64).clone()
                m[fr[2]["mask"].shape[0] // 2, fr[2]["mask"].shape[1] // 3] = 2 ** 31
                ins[2] = ins[2][:3] + (m,)
                g, match, bad = gts, r"\(-2\).*trackers\[2\].*int32", None
            before = [_state(tr) for tr in trs]
            d_before = [x[1].clone() for x in ins]
            m_before = [x[3].clone() for x in ins]
            with pytest.raises(capi.VdoError, match=match):
                _mixed(trs, ins, g)
            for i, tr in enumerate(trs):
                _assert_state(tr, before[i], f"frame {t} tracker {i}")
                assert torch.equal(ins[i][1], d_before[i]) and torch.equal(ins[i][3], m_before[i]), f"frame {t} tracker {i}: a refused call writes nothing back"
            if bad is not None:
                with pytest.raises(capi.VdoError, match=r"\(-3\).*ORB"):
                    _alone(bad, ins[1], g[1])
        ins_m = [_inputs(fr[i], t, i) for i in range(3)]
        Tm = _mixed(tm, ins_m, gts)
        for i in range(3):
            Ts = _alone(ts[i], _inputs(fr[i], t, i), gts[i])
            assert np.array_equal(Tm[i], Ts), f"frame {t} sequence {i}: Tcw"
            _assert_same(tm[i], ts[i], f"frame {t} sequence {i}")
    # the Python front refuses before the C call: a plane of another tracker's size, a wrong dtype, a host tensor
    calls = []
    real = ctx.L.vdo_tracker_track_mixed_dev
    monkeypatch.setattr(ctx.L, "vdo_tracker_track_mixed_dev", lambda *a: calls.append(a) or real(*a))
    fr = [frames[i][0] for i in range(3)]
    ins = [_inputs(fr[i], 0, i) for i in range(3)]
    before = [_state(tr) for tr in tm]
    cases = {"size of another tracker": (ins[0][0],) + ins[1][1:], "dtype": (ins[1][0].float(),) + ins[1][1:], "host tensor": (ins[1][0].cpu(),) + ins[1][1:],
             "mask dtype": ins[1][:3] + (ins[1][3].to(torch.int16),)}
    for what, bad_in in cases.items():
        trial = [ins[0], tuple(bad_in), ins[2]]
        with pytest.raises(ValueError, match=r"trackers\[1\]"):
            _mixed(tm, trial, [f["obj_ids"] for f in fr])
        assert not calls, what
    with pytest.raises(ValueError):
        capi.track_tensors_mixed(tm, [x[0] for x in ins[:2]], [x[1] for x in ins], [x[2] for x in ins], [x[3] for x in ins], [[], [], []])
    with pytest.raises(ValueError):
        capi.track_tensors_mixed([], [], [], [], [], [])
    assert not calls
    for tr, st in zip(tm, before):
        _assert_state(tr, st, "after the Python refusals")


def _raw_call(ctx, trackers, planes, gt_begin, gt_ids=None):
    B = len(trackers)
    arr = [(capi.DevPlane * B)(*[planes[k] for _ in range(B)]) for k in range(4)]
    handles = (C.c_void_p * B)(*[t.h_.value for t in trackers])
    gb = np.asarray(gt_begin, np.int32)
    gi = np.asarray(gt_ids if gt_ids is not None else [0], np.int32)
    T = np.zeros((B, 4, 4), np.float32)
    return ctx.L.vdo_tracker_track_mixed_dev(handles, C.c_int(B), *arr, gb.ctypes.data_as(C.POINTER(C.c_int)), gi.ctypes.data_as(C.POINTER(C.c_int)),
                                             C.c_int(0), C.c_uint64(0), T.ctypes.data_as(C.POINTER(C.c_float)))


def test_argument_refusals(ctx):
    """the checks of vdo_tracker_track_batch_dev except the geometry rule"""
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
        "gt_begin not from 0": ([a, b], [1, 1, 1], ERR_ARG, "gt_begin"),
        "gt_begin decreasing": ([a, b], [0, 2, 1], ERR_ARG, "gt_begin"),
    }
    for what, (trs, gb, rc, msg) in cases.items():
        assert _raw_call(ctx, trs, planes, gb, [1, 2]) == rc, what
        err = ctx.L.vdo_tracker_last_error(trs[0].h_).decode()
        assert msg in err and "vdo_tracker_track_mixed_dev" in err, what
    assert int(a.get("f_id")[0]) == 0 and len(a.map_get("vmCameraPose")) == 0 and len(b.map_get("vmCameraPose")) == 0
    # trackers that differ in size and ORB settings are accepted, each with planes of its own size
    c = capi.Tracker(ctx, width=W + 2, height=H + 4, cx=161.0, cy=112.0, n_features=2000, n_levels=5)
    z = lambda t, s: torch.zeros(s, dtype=t.dtype, device=DEV)
    T = capi.track_tensors_mixed([a, c], [img, z(img, (H + 4, W + 2))], [d, z(d, (H + 4, W + 2)) + 1], [fl, z(fl, (H + 4, W + 2, 2))],
                                 [m, z(m, (H + 4, W + 2))], [[], []], writeback=False)
    assert T.shape == (2, 4, 4) and len(a.map_get("vmCameraPose")) == 16 and len(c.map_get("vmCameraPose")) == 16
