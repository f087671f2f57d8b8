"""Object features carried across frame pairs on the device (capi.ObjectMotion.renew / vdo_obj_renew_batch_dev, and the samples= sets of
track() and update_mask(): vdo_obj_track_set_batch_dev, vdo_obj_update_mask_set_batch_dev).

Two references, both compared bit for bit:
  * the tracker: capi.Tracker.track over whole synth.make_sequence_frame sequences (every object ID in gt_ids, so the ground-truth gate
    never fires), whose per-frame object state (mvObjKeys ... nDynInlierID, the dynamic objects, the written-back mask) the chain
    update_mask -> track -> renew must reproduce frame after frame from the tracker's own metric depth and poses;
  * the host route per pair: capi.renew_frame_info (vdo_renew_frame_info, with an empty static part) fed with the device track() result
    and Frame.sample_objects of the current frame."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from tests.object_motion_reference import inv4
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
CAP = ((W + 3) // 4) * ((H + 3) // 4)
M = 8
FILL = 7
SET_COLS = ("x", "y", "label", "depth", "cx", "cy", "flow", "inlier_id", "obj_label", "point")


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


def tens(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host_of(o):
    return {k: v.cpu().numpy() for k, v in o.items()}


def filled(d):
    for v in d.values():
        v.fill_(FILL)
    return d


def dropped(seed):
    """the object missing from frame 5's mask: the larger of objects 1 and 3 there"""
    m = make_sequence_frame(5, seed=seed, width=W, height=H, n_obj=4, parked=(2,))["mask"]
    return 1 if (m == 1).sum() > (m == 3).sum() else 3


@functools.lru_cache(maxsize=None)
def frames(seed, n=12, n_obj=4):
    """a sequence with the events the renewal has to follow: object 2 parked; the larger of objects 1 and 3 missing from frame 5's mask
    (UpdateMask recovers it); object 4 absent from the masks before frame 6 (it enters mid-sequence); object 1's flow scrambled in frame 8
    (it fails the gate)"""
    out = []
    rng = np.random.default_rng(seed + 77)
    for t in range(n):
        f = make_sequence_frame(t, seed=seed, width=W, height=H, n_obj=n_obj, parked=(2,))
        mask, flow = f["mask"].copy(), f["flow"].copy()
        if t == 5:
            mask[mask == dropped(seed)] = 0
        if t < 6:
            mask[mask == 4] = 0
        if t == 8:
            sel = f["mask"] == 1
            flow[sel] += rng.normal(0.0, 6.0, (int(sel.sum()), 2)).astype(np.float32)
        out.append(dict(gray=f["gray"], depth_raw=f["depth_raw"], flow=flow, mask=mask.astype(np.int32), ids=list(range(1, n_obj + 1))))
    return out


TRACKER_F = ("mvObjKeys", "mvObjDepth", "mvObjCorres", "mvObjFlowNext", "mvObj3DPoint", "vObjMod", "vObjCentre3D")
TRACKER_I = ("vSemObjLabel", "vObjLabel", "nDynInlierID", "nModLabel", "nSemPosition", "bObjStat", "max_id")


@functools.lru_cache(maxsize=None)
def tracked(ctx, seed):
    """the tracker over the sequence: per frame its metric depth, written-back mask, Tcw and object state"""
    tr = capi.Tracker(ctx, local_batch=0)
    res = []
    for f in frames(seed):
        d, m = f["depth_raw"].copy(), f["mask"].copy()
        T = tr.track(f["gray"], d, f["flow"], m, f["ids"], writeback=True)
        res.append(dict(depth=d, mask=m, Tcw=T.copy(), **{k: tr.get(k) for k in TRACKER_F + TRACKER_I}))
    return res


def set_rows(S, p=0):
    n = int(S["count"][p])
    return {k: S[k][p, :n] for k in SET_COLS}


def assert_set_equals_tracker(S, ref, what):
    r = set_rows(S)
    keys = ref["mvObjKeys"].reshape(-1, 2)
    assert len(keys) == len(r["x"]), (what, len(keys), len(r["x"]))
    assert np.array_equal(np.stack([r["x"], r["y"]], 1).astype(np.float32), keys), what
    assert np.array_equal(r["depth"], ref["mvObjDepth"]), what
    assert np.array_equal(np.stack([r["cx"], r["cy"]], 1), ref["mvObjCorres"].reshape(-1, 2)), what
    assert np.array_equal(r["flow"], ref["mvObjFlowNext"].reshape(-1, 2)), what
    assert np.array_equal(r["point"], ref["mvObj3DPoint"].reshape(-1, 3)), what
    assert np.array_equal(r["label"], ref["vSemObjLabel"]), what
    assert np.array_equal(r["obj_label"], ref["vObjLabel"]), what
    assert np.array_equal(r["inlier_id"], ref["nDynInlierID"]), what


def dynamic_slots(o, p=0):
    return [s for s in range(o["cls"].shape[1]) if o["cls"][p, s] == capi.OT_DYNAMIC]


def assert_track_equals_tracker(o, ref, what):
    dyn = dynamic_slots(o)
    assert np.array_equal(o["id"][0, dyn], ref["nModLabel"]), what
    assert np.array_equal(o["label"][0, dyn], ref["nSemPosition"]), what
    assert np.array_equal(o["stat"][0, dyn], ref["bObjStat"]), what
    assert np.array_equal(o["H"][0, dyn].reshape(-1), ref["vObjMod"]), what
    assert np.array_equal(o["centre"][0, dyn].reshape(-1), ref["vObjCentre3D"]), what
    assert int(o["max_id"][0]) == int(ref["max_id"][0]), what


def chain(est, seq, with_sets, check=None):
    """update_mask -> track -> renew over the sequence on the tracker's depth and poses; check(t, mask, track result, set) per pair"""
    depth = [tens(r["depth"]) for r in seq["ref"]]
    flow = [tens(f["flow"]) for f in seq["frames"]]
    mask = [tens(f["mask"]) for f in seq["frames"]]
    T = [tens(r["Tcw"][None]) for r in seq["ref"]]
    S, prev = None, None
    outs = [est.empty_outputs(1, track=True) for _ in range(2)]
    sets = [est.empty_outputs(1, renew=True) for _ in range(2)]
    um = est.empty_outputs(1, update_mask=True)
    for t in range(len(depth) - 1):
        est.update_mask([depth[t]], [flow[t]], [mask[t]], [mask[t + 1]], samples=S, out=um)
        obj = est.track([depth[t]], [flow[t]], [mask[t]], [depth[t + 1]], [mask[t + 1]], KITTI_K, Tcw_last=T[t], Tcw_cur=T[t + 1], prev=prev,
                        samples=S, out=outs[t % 2])
        if with_sets:
            S = est.renew(obj, [depth[t + 1]], [flow[t + 1]], [mask[t + 1]], KITTI_K, Tcw_cur=T[t + 1], out=sets[t % 2])
        prev = obj
        torch.cuda.synchronize()
        if check:
            check(t, mask[t + 1].cpu().numpy(), host_of(obj), None if S is None else host_of(S))


# ------------------------------------------------------------------------------------------------ 1. equal to the tracker, whole sequences
@pytest.mark.parametrize("seed", [0, 5])
def test_sequence_equals_the_tracker(ctx, seed):
    seq = dict(frames=frames(seed), ref=tracked(ctx, seed))
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    seen = dict(recovered=0, entered=0, failed=0, parked=0, carried=0)

    def check(t, mask, o, S):
        ref = seq["ref"][t + 1]
        what = f"seed {seed}, frame {t + 1}"
        assert np.array_equal(mask, ref["mask"]), what
        assert_track_equals_tracker(o, ref, what)
        assert_set_equals_tracker(S, ref, what)
        assert S["status"][0] == 0
        seen["recovered"] += t == 4 and bool((mask == dropped(seed)).any())
        seen["entered"] += int(((set_rows(S)["label"] == 4) & (set_rows(S)["obj_label"] == -2)).any()) if t == 5 else 0
        seen["failed"] += int(any(o["stat"][0, s] == 0 for s in dynamic_slots(o)))
        seen["parked"] += int(any(o["label"][0, s] == 2 and o["cls"][0, s] == capi.OT_STATIC for s in range(M)))
        seen["carried"] += int((set_rows(S)["inlier_id"] >= 0).any())            # carried points have identities

    chain(est, seq, True, check)
    assert all(v > 0 for v in seen.values()) and seen["carried"] >= 6, seen

    # without the carried sets the same loop leaves the tracker from the second pair on
    diff = []
    chain(est, seq, False, lambda t, mask, o, S: diff.append(t >= 1 and not np.array_equal(
        o["H"][0, dynamic_slots(o)].reshape(-1), seq["ref"][t + 1]["vObjMod"])))
    assert any(diff), diff


# ------------------------------------------------------------------------------------------------ 2. equal to the host route, per pair
def host_renew(ctx, g, p, depth_c, flow_c, mask_c, Tcw_cur, max_obj, step=4, th=25.0):
    """the object part of vdo_renew_frame_info on pair p of a D2H'd track() result and Frame.sample_objects of the current frame"""
    fr = capi.Frame(ctx, W, H)
    fr.upload(depth=depth_c, flow=flow_c, mask=np.asarray(mask_c).astype(np.int32))
    s = fr.sample_objects(th, step)
    n = int(g["n_samples"][p])
    keys = np.stack([(g["sample_x"][p, :n] + g["sample_flow_ref"][p, :n, 0]).astype(np.float32),
                     (g["sample_y"][p, :n] + g["sample_flow_ref"][p, :n, 1]).astype(np.float32)], 1)
    slots = [j for j in range(M) if g["label"][p, j] != -1]
    inl = [[k for k in range(n) if g["sample_slot"][p, k] == j and g["sample_flags"][p, k] & 2] for j in slots]
    _, o = capi.renew_frame_info(fr, [], np.zeros((0, 2)), np.zeros((0, 2)), 0, inl, g["stat"][p, slots], g["label"][p, slots], g["id"][p, slots], keys,
                                 g["obj_label"][p, :n], np.stack([s["x"], s["y"]], 1).astype(np.float32), s["depth"], s["label"],
                                 np.stack([s["fx"], s["fy"]], 1), np.stack([s["cx"], s["cy"]], 1), max_obj, np.asarray(KITTI_K, np.float32),
                                 inv4(Tcw_cur))
    fr.close()
    return o


def assert_set_equals_host(S, p, o, what, cap=CAP):
    n = min(len(o["keys"]), cap)
    assert S["count"][p] == n and S["status"][p] == (capi.OM_PAIR_FEATURE_CAP if len(o["keys"]) > cap else 0), (what, S["count"][p], len(o["keys"]))
    r = set_rows(S, p)
    for got, want in ((np.stack([r["x"], r["y"]], 1).astype(np.float32), o["keys"]), (r["depth"], o["depth"]), (np.stack([r["cx"], r["cy"]], 1), o["corres"]),
                      (r["flow"], o["flow"]), (r["label"], o["sem"]), (r["inlier_id"], o["inlier_id"]), (r["obj_label"], o["label"]), (r["point"], o["p3d"])):
        assert np.array_equal(got, want[:n]), what


@functools.lru_cache(maxsize=None)
def pair_inputs(seed, t):
    f0, f1 = (make_sequence_frame(t + k, seed=seed, width=W, height=H, n_obj=4) for k in (0, 1))
    dep = lambda f: np.where(f["depth_raw"] < 0, np.float32(0), KITTI_BF / (f["depth_raw"] / KITTI_DEPTH_FACTOR)).astype(np.float32)
    Tc = lambda f: np.linalg.inv(f["Twc"]).astype(np.float32)
    return dict(d0=dep(f0), f0=f0["flow"], m0=f0["mask"], T0=Tc(f0), d1=dep(f1), f1=f1["flow"], m1=f1["mask"], T1=Tc(f1))


def layout(a, kind, how):
    """a plane in one of the strided layouts the calls accept"""
    if kind == "flow" and how == "chw":
        return tens(np.ascontiguousarray(a.transpose(2, 0, 1)))
    if how == "strided":
        big = np.zeros((a.shape[0] + 3, a.shape[1] + 5) + a.shape[2:], a.dtype)
        big[1:1 + a.shape[0], 2:2 + a.shape[1]] = a
        return tens(big)[1:1 + a.shape[0], 2:2 + a.shape[1]]
    return tens(a)


@pytest.mark.parametrize("max_obj", [0, 50, 800])
@pytest.mark.parametrize("how", ["plain", "i64_chw", "strided"])
def test_pair_equals_host_route(ctx, max_obj, how):
    seeds = [(0, 2), (1, 4), (3, 1)]
    P = len(seeds)
    est = capi.ObjectMotion(ctx, P, M, CAP)
    ins = [pair_inputs(s, t) for s, t in seeds]
    mdt = np.int64 if how == "i64_chw" else np.int32
    fl_how = "chw" if how == "i64_chw" else how
    obj = est.track([tens(x["d0"]) for x in ins], [tens(x["f0"]) for x in ins], [tens(x["m0"]) for x in ins], [tens(x["d1"]) for x in ins],
                    [tens(x["m1"]) for x in ins], KITTI_K, Tcw_last=tens(np.stack([x["T0"] for x in ins])), Tcw_cur=tens(np.stack([x["T1"] for x in ins])))
    S = filled(est.empty_outputs(P, renew=True))
    est.renew(obj, [layout(x["d1"], "depth", how if how == "strided" else "plain") for x in ins], [layout(x["f1"], "flow", fl_how) for x in ins],
              [layout(x["m1"].astype(mdt), "mask", how if how == "strided" else "plain") for x in ins], KITTI_K,
              Tcw_cur=tens(np.stack([x["T1"] for x in ins])), max_track_obj=max_obj, out=S)
    torch.cuda.synchronize()
    g, S = host_of(obj), host_of(S)
    for p, x in enumerate(ins):
        o = host_renew(ctx, g, p, x["d1"], x["f1"], x["m1"], x["T1"], max_obj)
        assert_set_equals_host(S, p, o, (how, max_obj, p))
        if max_obj == 800:
            assert (o["inlier_id"] >= 0).any() and (o["label"] >= 1).any()
        assert (S["x"][p, S["count"][p]:] == FILL).all()                  # rows past count untouched


# ------------------------------------------------------------------------------------------------ 3. limits
def plane_pair(w=256, h=128, flow=(10.5, 0.5), depth=10.0):
    """one object filling the frame: a fronto-parallel plane at `depth` translating parallel to the image, so its flow is the same
    everywhere and the motion is exactly rigid (identity camera poses)"""
    d = np.full((h, w), depth, np.float32)
    f = np.empty((h, w, 2), np.float32)
    f[..., 0], f[..., 1] = flow
    m = np.ones((h, w), np.int32)
    return d, f, m


def host_route_plane(ctx, est_track, d, f, m, max_obj):
    h, w = d.shape
    fr = capi.Frame(ctx, w, h)
    fr.upload(depth=d, flow=f, mask=m)
    s = fr.sample_objects(25.0, 4)
    g = est_track
    n = int(g["n_samples"][0])
    keys = np.stack([(g["sample_x"][0, :n] + g["sample_flow_ref"][0, :n, 0]).astype(np.float32),
                     (g["sample_y"][0, :n] + g["sample_flow_ref"][0, :n, 1]).astype(np.float32)], 1)
    slots = [j for j in range(M) if g["label"][0, j] != -1]
    inl = [[k for k in range(n) if g["sample_slot"][0, k] == j and g["sample_flags"][0, k] & 2] for j in slots]
    _, o = capi.renew_frame_info(fr, [], np.zeros((0, 2)), np.zeros((0, 2)), 0, inl, g["stat"][0, slots], g["label"][0, slots], g["id"][0, slots], keys,
                                 g["obj_label"][0, :n], np.stack([s["x"], s["y"]], 1).astype(np.float32), s["depth"], s["label"],
                                 np.stack([s["fx"], s["fy"]], 1), np.stack([s["cx"], s["cy"]], 1), max_obj, np.asarray(KITTI_K, np.float32),
                                 np.eye(4, dtype=np.float32))
    fr.close()
    return o


@pytest.mark.parametrize("flow", [(10.5, 0.5), (12.0, 4.0)])
def test_plane_object_cap_and_pixel_reuse(ctx, flow):
    """an object filling the frame, carried and topped up without a quota: (10.5, 0.5) puts every carried key off the raster, so the set
    holds about twice the raster and is cut at the cap (VDO_OM_PAIR_FEATURE_CAP), equal to the host route's first C rows; (12, 4) puts every
    carried key on a raster position, which the top-up must then skip (the reference's "closer than 1 px")"""
    d, f, m = plane_pair(flow=flow)
    h, w = d.shape
    cap = ((w + 3) // 4) * ((h + 3) // 4)
    est = capi.ObjectMotion(ctx, 1, M, cap)
    o = est.track([tens(d)], [tens(f)], [tens(m)], [tens(d)], [tens(m)], KITTI_K, shrink=(0, 0))
    S = filled(est.empty_outputs(1, renew=True))
    est.renew(o, [tens(d)], [tens(f)], [tens(m)], KITTI_K, max_track_obj=100000, out=S)
    torch.cuda.synchronize()
    g, S = host_of(o), host_of(S)
    assert g["stat"][0, 0] == 1, (g["cls"][0], g["status"][0])
    ref = host_route_plane(ctx, g, d, f, m, 100000)
    assert_set_equals_host(S, 0, ref, flow, cap=cap)
    r = set_rows(S)
    carried = r["inlier_id"] >= 0
    if flow[0] == 10.5:
        assert len(ref["keys"]) > cap and S["status"][0] == capi.OM_PAIR_FEATURE_CAP
    else:
        assert S["status"][0] == 0 and carried.sum() > 1000
        taken = set(zip(r["x"][carried].tolist(), r["y"][carried].tolist()))
        topped = ~carried & (r["obj_label"] >= 1)
        assert all((a % 4, b % 4) == (0, 0) for a, b in taken)
        assert topped.any() and not any(q in taken for q in zip(r["x"][topped].tolist(), r["y"][topped].tolist()))


def test_64_pairs_with_staggered_starts(ctx):
    """64 pairs of mixed sizes, each a sequence of its own; pair p restarts at step p % 3 (its set's count -1, its prev row the reset state):
    every step of every pair equals the same pair run alone"""
    P, steps = 64, 3
    sizes = [(W, H), (640, 256), (400, 160), (1000, 300)]
    est = capi.ObjectMotion(ctx, P, M, CAP)
    solo = capi.ObjectMotion(ctx, 1, M, CAP)
    dep = lambda f: np.where(f["depth_raw"] < 0, np.float32(0), KITTI_BF / (f["depth_raw"] / KITTI_DEPTH_FACTOR)).astype(np.float32)
    seqs = []
    for p in range(P):
        w, h = sizes[p % 4]
        fs = [make_sequence_frame(t + p % 3, seed=p % 7, width=w, height=h, n_obj=1 + p % 4) for t in range(steps + 1)]
        seqs.append([dict(d=tens(dep(f)), f=tens(f["flow"]), m=tens(f["mask"]), T=tens(np.linalg.inv(f["Twc"]).astype(np.float32)[None])) for f in fs])
    sets = [est.empty_outputs(P, renew=True) for _ in range(2)]
    outs = [est.empty_outputs(P, track=True) for _ in range(2)]
    S, prev = None, None
    solo_S, solo_prev = [None] * P, [None] * P
    for t in range(steps):
        pl = lambda k, i: [seqs[p][t + i][k] for p in range(P)]
        start = [t == 0 or p % 3 == t for p in range(P)]
        for p in range(P):
            if start[p] and S is not None:
                S["count"][p] = -1
                prev["label"][p] = -1; prev["id"][p] = -1; prev["stat"][p] = 0; prev["max_id"][p] = 1
                prev["H"][p] = torch.eye(4, device=DEV)
        obj = est.track(pl("d", 0), pl("f", 0), pl("m", 0), pl("d", 1), pl("m", 1), KITTI_K, Tcw_last=torch.cat(pl("T", 0)), Tcw_cur=torch.cat(pl("T", 1)),
                        prev=prev, samples=S, out=outs[t % 2])
        S = est.renew(obj, pl("d", 1), pl("f", 1), pl("m", 1), KITTI_K, Tcw_cur=torch.cat(pl("T", 1)), out=sets[t % 2])
        prev = obj
        torch.cuda.synchronize()
        g, Sh = host_of(obj), host_of(S)
        for p in range(P):
            if start[p]:
                solo_S[p], solo_prev[p] = None, None
            q = seqs[p]
            so = solo.track([q[t]["d"]], [q[t]["f"]], [q[t]["m"]], [q[t + 1]["d"]], [q[t + 1]["m"]], KITTI_K, Tcw_last=q[t]["T"], Tcw_cur=q[t + 1]["T"],
                            prev=solo_prev[p], samples=solo_S[p])
            ss = solo.renew(so, [q[t + 1]["d"]], [q[t + 1]["f"]], [q[t + 1]["m"]], KITTI_K, Tcw_cur=q[t + 1]["T"])
            torch.cuda.synchronize()
            solo_S[p], solo_prev[p] = {k: v.clone() for k, v in ss.items()}, {k: v.clone() for k, v in so.items()}
            sh, go = host_of(ss), host_of(so)
            for k in ("label", "id", "stat", "H", "max_id", "n_samples"):
                assert np.array_equal(g[k][p], go[k][0]), (t, p, k)
            assert Sh["count"][p] == sh["count"][0] and Sh["status"][p] == sh["status"][0], (t, p)
            n = int(sh["count"][0])
            for k in SET_COLS:
                assert np.array_equal(Sh[k][p, :n], sh[k][0, :n]), (t, p, k)


# ------------------------------------------------------------------------------------------------ 4. capture
def test_cuda_graph_of_the_step_equals_eager(ctx):
    seed = 0
    seq = dict(frames=frames(seed), ref=tracked(ctx, seed))
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    n = 7
    depth = [tens(r["depth"]) for r in seq["ref"][:n]]
    flow = [tens(f["flow"]) for f in seq["frames"][:n]]
    masks = [tens(f["mask"]) for f in seq["frames"][:n]]
    T = [tens(r["Tcw"][None]) for r in seq["ref"][:n]]
    # eager reference
    eager = []
    S, prev = None, None
    for t in range(n - 1):
        mc = masks[t + 1].clone()
        ml = masks[t] if t == 0 else eager[-1]["mask"]
        est.update_mask([depth[t]], [flow[t]], [ml], [mc], samples=S)
        o = est.track([depth[t]], [flow[t]], [ml], [depth[t + 1]], [mc], KITTI_K, Tcw_last=T[t], Tcw_cur=T[t + 1], prev=prev, samples=S)
        S = est.renew(o, [depth[t + 1]], [flow[t + 1]], [mc], KITTI_K, Tcw_cur=T[t + 1])
        prev = o
        eager.append(dict(mask=mc, obj={k: v.clone() for k, v in o.items()}, set={k: v.clone() for k, v in S.items()}))
    # the step captured once: static inputs, double-buffered sets and outputs (one graph per parity)
    dl, fl, ml, dc, mc, fc, Tl, Tc = (x.clone() for x in (depth[0], flow[0], masks[0], depth[1], masks[1], flow[1], T[0], T[1]))
    sets = [est.empty_outputs(1, renew=True) for _ in range(2)]
    outs = [est.empty_outputs(1, track=True) for _ in range(2)]
    um = est.empty_outputs(1, update_mask=True)
    for s in sets:
        s["count"].fill_(-1)
    graphs = []
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        for k in range(2):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                est.update_mask([dl], [fl], [ml], [mc], samples=sets[1 - k], out=um)
                o = est.track([dl], [fl], [ml], [dc], [mc], KITTI_K, Tcw_last=Tl, Tcw_cur=Tc, prev=outs[1 - k], samples=sets[1 - k], out=outs[k])
                est.renew(o, [dc], [fc], [mc], KITTI_K, Tcw_cur=Tc, out=sets[k])
            graphs.append(g)
    torch.cuda.current_stream(DEV).wait_stream(side)
    # the first pair starts a sequence: reset prev row of outs[1], count -1 in sets[1]
    outs[1]["label"].fill_(-1); outs[1]["id"].fill_(-1); outs[1]["stat"].fill_(0); outs[1]["max_id"].fill_(1)
    outs[1]["H"].copy_(torch.eye(4, device=DEV).expand_as(outs[1]["H"]))
    sets[1]["count"].fill_(-1)
    for t in range(n - 1):
        dl.copy_(depth[t]); fl.copy_(flow[t]); ml.copy_(masks[t] if t == 0 else eager[t - 1]["mask"]); dc.copy_(depth[t + 1]); mc.copy_(masks[t + 1])
        fc.copy_(flow[t + 1]); Tl.copy_(T[t]); Tc.copy_(T[t + 1])
        graphs[t % 2].replay()
        torch.cuda.synchronize()
        e = eager[t]
        assert torch.equal(mc, e["mask"]), t
        ns = int(e["obj"]["n_samples"][0])
        for k, v in e["obj"].items():
            per_sample = v.dim() >= 2 and v.shape[1] == CAP
            got = outs[t % 2][k]
            assert torch.equal(got[:, :ns] if per_sample else got, v[:, :ns] if per_sample else v), (t, k)
        cnt = int(e["set"]["count"][0])
        assert int(sets[t % 2]["count"][0]) == cnt
        for k in SET_COLS:
            assert torch.equal(sets[t % 2][k][0, :cnt], e["set"][k][0, :cnt]), (t, k)


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_python_refusals_write_nothing(ctx):
    x = pair_inputs(0, 0)
    est = capi.ObjectMotion(ctx, 2, M, CAP)
    obj = est.track([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [tens(x["d1"])], [tens(x["m1"])], KITTI_K)
    S = filled(est.empty_outputs(1, renew=True))
    d, f, m = tens(x["d1"]), tens(x["f1"]), tens(x["m1"])
    ok = dict(track_result=obj, depths_cur=[d], flows_cur=[f], masks_cur=[m], K=KITTI_K, out=S)
    other = capi.ObjectMotion(ctx, 1, M + 1, CAP).empty_outputs(1, track=True)
    bad = [dict(max_track_obj=-1), dict(step=0), dict(th_depth_obj=float("nan")), dict(track_result=other), dict(track_result=[]),
           dict(depths_cur=[d, d], flows_cur=[f, f], masks_cur=[m, m]), dict(masks_cur=[m.float()]), dict(flows_cur=[d]),
           dict(out=dict(S, point=S["point"][:, :, :2])), dict(Tcw_cur=torch.eye(4)), dict(K=np.zeros(3))]
    for b in bad:
        with pytest.raises(ValueError):
            est.renew(**dict(ok, **b))
    torch.cuda.synchronize()
    for k, t in S.items():
        assert (t == FILL).all(), k
    tout = filled(est.empty_outputs(1, track=True))
    with pytest.raises(ValueError):
        est.track([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [d], [m], KITTI_K, samples=dict(S, label=S["label"][:, :5]), out=tout)
    with pytest.raises(ValueError):
        est.update_mask([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [m.clone()], samples="set")
    torch.cuda.synchronize()
    for k, t in tout.items():
        assert (t == FILL).all(), k


def test_c_refusals_write_nothing(ctx):
    x = pair_inputs(0, 0)
    est = capi.ObjectMotion(ctx, 2, M, CAP)
    obj = est.track([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [tens(x["d1"])], [tens(x["m1"])], KITTI_K)
    torch.cuda.synchronize()
    d, f, m = tens(x["d1"]), tens(x["f1"]), tens(x["m1"])
    pl = {k: capi._dev_plane(ctx, kd, v, W, H) for k, kd, v in (("d", "depth", d), ("f", "flow", f), ("m", "mask", m))}
    S = filled(est.empty_outputs(1, renew=True))
    host_buf = np.zeros(1 << 16, np.int32)
    shapes = est._shapes(1, capi._OT_OUT)
    tp = capi._out_ptrs(ctx, obj, shapes, capi._OT_OUT)
    Kp = np.ascontiguousarray(np.asarray(KITTI_K, np.float32)[None])
    wh1 = np.array([[W, H]], np.int32)

    def set_with(**kw):
        ptr = {k: S[k].data_ptr() for k in capi._OS_SET}
        ptr.update(kw)
        return capi.ObjFeatSet(*[ptr[k] for k in capi._OS_SET])

    def track_with(**kw):
        ptr = dict(zip(capi._OT_OUT, tp))
        ptr.update(kw)
        v = [ptr[k] for k in capi._OT_OUT]
        return capi.ObjTrackOut(capi.ObjMotionOut(*v[:len(capi._OM_OUT)]), *v[len(capi._OM_OUT):])

    def call(P=1, step=4, th=25.0, mx=800, so=None, to=None, mp=None, wh=None, null_t=False):
        arr = lambda p_: (capi.DevPlane * P)(*([p_] * P))
        whp = np.tile(wh1, (P, 1)) if wh is None else wh
        Kx = np.tile(Kp, (P, 1))
        return ctx.L.vdo_obj_renew_batch_dev(est.h_, C.c_int(P), None if null_t else C.byref(to or track_with()), arr(pl["d"]), arr(pl["f"]),
                                             arr(mp or pl["m"]), whp.ctypes.data_as(C.POINTER(C.c_int32)), Kx.ctypes.data_as(C.POINTER(C.c_float)), None,
                                             C.c_int32(step), C.c_float(th), C.c_int32(mx), C.byref(so or set_with()), C.c_uint64(0))

    plane = lambda p_, **kw: capi.DevPlane(**dict(dict(data_dev=p_.data_dev, dtype=p_.dtype, channels=1, stride_y=p_.stride_y, stride_x=p_.stride_x,
                                                       stride_c=0, rgb=1), **kw))
    bad = {"P 0": dict(P=0), "P 3": dict(P=3), "step 0": dict(step=0), "th NaN": dict(th=float("nan")), "max_track_obj -1": dict(mx=-1),
           "track_out NULL": dict(null_t=True), "mask f32": dict(mp=plane(pl["m"], dtype=capi.VDO_DT_F32)),
           "size above the cap": dict(wh=np.array([[W + 8, H]], np.int32)), "width 0": dict(wh=np.array([[0, H]], np.int32)),
           "set point NULL": dict(so=set_with(point=None)), "set count host memory": dict(so=set_with(count=host_buf.ctypes.data)),
           "set x misaligned": dict(so=set_with(x=S["x"].data_ptr() + 2)),
           "track stat NULL": dict(to=track_with(stat=None)), "track flow_ref misaligned": dict(to=track_with(sample_flow_ref=tp[list(capi._OT_OUT).index("sample_flow_ref")] + 4))}
    torch.cuda.synchronize()
    for what, kw in bad.items():
        assert call(**kw) == ERR_ARG, what
        assert ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_obj_renew_batch_dev"), what
    torch.cuda.synchronize()
    for k, t in S.items():
        assert (t == FILL).all(), k
    assert call() == 0
    torch.cuda.synchronize()
    # the set entries refuse a NULL set and a foreign set field, writing nothing
    tout = filled(est.empty_outputs(1, track=True))
    o = track_with(**{k: tout[k].data_ptr() for k in capi._OT_OUT})
    opts = capi.ObjTrackOpts(4, 25.0, 500, 50, 0.4, 0.98, 1, 0.12, 0.3, 25, 50, 0)
    d0, f0, m0 = (capi._dev_plane(ctx, k, tens(x[v]), W, H) for k, v in (("depth", "d0"), ("flow", "f0"), ("mask", "m0")))
    one = lambda p_: (capi.DevPlane * 1)(p_)
    for last in (None, set_with(cx=host_buf.ctypes.data)):
        rc = ctx.L.vdo_obj_track_set_batch_dev(est.h_, C.c_int(1), one(d0), one(f0), one(m0), one(pl["d"]), one(pl["m"]), wh1.ctypes.data_as(C.POINTER(C.c_int32)),
                                               Kp.ctypes.data_as(C.POINTER(C.c_float)), None, None, None, None, None, None, None,
                                               None if last is None else C.byref(last), C.byref(opts), C.byref(o), C.c_uint64(0))
        assert rc == ERR_ARG and ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_obj_track_set_batch_dev")
        uo = est.empty_outputs(1, update_mask=True)
        rc = ctx.L.vdo_obj_update_mask_set_batch_dev(est.h_, C.c_int(1), one(d0), one(f0), one(m0), one(pl["m"]), wh1.ctypes.data_as(C.POINTER(C.c_int32)),
                                                     C.c_int32(4), C.c_float(25.0), None if last is None else C.byref(last),
                                                     C.byref(capi.ObjMaskOut(*[uo[k].data_ptr() for k in capi._OU_OUT])), C.c_uint64(0))
        assert rc == ERR_ARG and ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_obj_update_mask_set_batch_dev")
    torch.cuda.synchronize()
    for k, t in tout.items():
        assert (t == FILL).all(), k


def test_set_count_out_of_range_is_flagged(ctx):
    x = pair_inputs(0, 0)
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    S = est.empty_outputs(1, renew=True)
    S["count"].fill_(CAP + 1)
    o = est.track([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [tens(x["d1"])], [tens(x["m1"])], KITTI_K, samples=S)
    u = est.update_mask([tens(x["d0"])], [tens(x["f0"])], [tens(x["m0"])], [tens(x["m1"])], samples=S)
    torch.cuda.synchronize()
    assert int(o["n_samples"][0]) == 0 and int(o["pair_status"][0]) & capi.OM_PAIR_SET_COUNT
    assert int(u["n_samples"][0]) == 0 and int(u["pair_status"][0]) & capi.OM_PAIR_SET_COUNT
