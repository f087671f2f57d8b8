"""Tracked objects between frame pairs on the device (capi.ObjectMotion.track / vdo_obj_track_batch_dev).

Every output is compared with the host route of tests/object_track_reference.py (vdo_frame_sample_objects, the look-up in numpy,
capi.scene_flow, capi.dyn_obj_tracking, capi.init_model_batch with the ID-keyed motion model, capi.pose_opt_flow2 mode 1): it must be
identical.  Inputs: synth.make_sequence_frame pairs (t, t + 1), 1242x375, whose current masks are relabelled at random, so that the
objects' identities come only from the IDs.  Also: oracle parity of the IDs, classes and votes, a chained sequence of calls (persistent IDs,
a parked object, boundary and far objects, a failed gate, a split object), batch independence at 64 pairs with staggered resets, the edge
cases, a CUDA graph of extract -> match -> PnP -> refine -> track replayed over frames, and the refusals."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import tracking_ops as to
from tests import object_track_reference as R
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame, make_view_pair

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
STEP = 4
CAP = ((W + STEP - 1) // STEP) * ((H + STEP - 1) // STEP)
FILL = 7
EYE = np.eye(4, dtype=np.float32)
PER_SLOT = ("label", "H", "X", "T_init", "centre", "velocity", "info", "stats", "status", "id", "cls", "vote", "stat")


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@functools.lru_cache(maxsize=None)
def seq(seed, t, n_obj, parked=()):
    """frame t of sequence seed: metric depth, flow, mask (relabelled at random per frame: label = 10 * perm + 3), true Tcw"""
    f = make_sequence_frame(t, seed=seed, width=W, height=H, n_obj=n_obj, parked=parked)
    raw = f["depth_raw"]
    depth = np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
    perm = np.random.default_rng(100 * seed + t).permutation(n_obj) + 1
    relab = np.concatenate([[0], 10 * perm + 3]).astype(np.int32)
    return dict(depth=depth, flow=f["flow"], mask=relab[f["mask"]], true_of=dict(zip(relab[1:].tolist(), range(1, n_obj + 1))),
                Tcw=np.linalg.inv(f["Twc"]).astype(np.float32), gray=f["gray"])


def tens(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def filled(est, P):
    o = est.empty_outputs(P, track=True)
    for t in o.values():
        t.fill_(FILL)
    return o


def host_of(o):
    return {k: v.cpu().numpy() for k, v in o.items()}


def run(est, last, cur, poses=True, prev=None, **kw):
    P = len(last)
    Tl = tens(np.stack([f["Tcw"] for f in last])) if poses else None
    Tc = tens(np.stack([f["Tcw"] for f in cur])) if poses else None
    out = filled(est, P)
    est.track([tens(f["depth"]) for f in last], [tens(f["flow"]) for f in last], [tens(f["mask"]) for f in last],
              [tens(f["depth"]) for f in cur], [tens(f["mask"]) for f in cur], KITTI_K, Tcw_last=Tl, Tcw_cur=Tc,
              prev=None if prev is None else {k: tens(v) for k, v in prev.items()}, out=out, **kw)
    torch.cuda.synchronize()
    return host_of(out)


def prev_of(g):
    return {k: g[k] for k in ("label", "id", "stat", "H", "max_id")}


def row(prev, p):
    return None if prev is None else {k: v[p] for k, v in prev.items()}


def host_pair(ctx, f, c, M, poses=True, prev=None, **kw):
    return R.host_track(ctx, f["depth"], f["flow"], f["mask"], c["depth"], c["mask"], KITTI_K, M, f["Tcw"] if poses else None,
                        c["Tcw"] if poses else None, prev, **kw)


def assert_pair_equal(g, p, r, what=""):
    n = int(r["n_samples"])
    assert g["n_samples"][p] == n and g["pair_status"][p] == r["pair_status"] and g["max_id"][p] == r["max_id"], what
    for k in [k for k in r if k.startswith("sample_")] + ["label_cur", "depth_cur", "flow3d", "obj_label"]:
        assert np.array_equal(g[k][p, :n], r[k]), (what, k)
        assert (g[k][p, n:] == FILL).all(), (what, k)
    for k in PER_SLOT:
        assert np.array_equal(g[k][p], r[k]), (what, k)


CASES = [(0, 0, 3), (1, 0, 4), (2, 1, 5)]      # (seed, t, objects)


# ------------------------------------------------------------------------------------------------ 1. equal to the host route
@pytest.mark.parametrize("shrink", [(25, 50), (0, 0)])
@pytest.mark.parametrize("sf", [(0.12, 0.3), (0.5, 0.6)])
@pytest.mark.parametrize("quirk", [0, 1])
@pytest.mark.parametrize("poses", [True, False])
def test_equal_to_host_route(ctx, poses, quirk, sf, shrink):
    """two chained calls (t -> t+1, t+1 -> t+2): the second looks the IDs and motion models up in the first's result"""
    M = 8
    est = capi.ObjectMotion(ctx, len(CASES), M, CAP)
    kw = dict(quirk=quirk, sf_mg_thres=sf[0], sf_ds_thres=sf[1], shrink=shrink)
    prev = None
    for k in range(2):
        last = [seq(s, t + k, n) for s, t, n in CASES]
        cur = [seq(s, t + k + 1, n) for s, t, n in CASES]
        g = run(est, last, cur, poses, prev, **kw)
        for p, (f, c) in enumerate(zip(last, cur)):
            assert_pair_equal(g, p, host_pair(ctx, f, c, M, poses, row(prev, p), **kw), (k, p))
        prev = prev_of(g)
    if poses and sf == (0.12, 0.3):
        assert (g["cls"] == capi.OT_DYNAMIC).sum() >= 6 and (g["stat"] == 1).sum() >= 6


def test_oracle_parity(ctx):
    """the device's per-sample arrays through oracle/tracking_ops.dyn_obj_tracking give the same IDs, classes and votes"""
    M = 8
    est = capi.ObjectMotion(ctx, 3, M, CAP)
    prev = None
    for k in range(2):
        last = [seq(s, t + k, n) for s, t, n in CASES]
        cur = [seq(s, t + k + 1, n) for s, t, n in CASES]
        g = run(est, last, cur, True, prev)
        for p in range(3):
            n = g["n_samples"][p]
            sel = np.nonzero(g["sample_slot"][p, :n] >= 0)[0]
            pv = R.reset_state(M) if prev is None else row(prev, p)
            ol, objs, ml, sp, mid = to.dyn_obj_tracking(
                g["label_cur"][p, sel], np.zeros(len(sel), np.int32), np.stack([g["sample_cx"][p, sel], g["sample_cy"][p, sel]], 1),
                g["depth_cur"][p, sel], g["flow3d"][p, sel], g["sample_label"][p, sel], pv["label"], pv["stat"], pv["id"], H, W, 25, 50, 0.12,
                0.3, 25.0, 1 if prev is None else 2, int(pv["max_id"]))
            dyn = g["cls"][p] == capi.OT_DYNAMIC
            assert g["label"][p][dyn].tolist() == list(sp) and g["id"][p][dyn].tolist() == list(ml) and g["max_id"][p] == mid
            for j in np.nonzero(dyn)[0]:
                assert g["vote"][p, j] == to._majority(g["sample_label"][p, :n][g["sample_slot"][p, :n] == j].tolist())
        prev = prev_of(g)


# ------------------------------------------------------------------------------------------------ 2. a sequence of calls
def test_sequence_keeps_ids(ctx):
    """8 chained calls with a new random relabelling every frame: each moving object keeps one ID, the parked one is static"""
    M = 8
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    prev, id_of = None, {}
    for t in range(8):
        f, c = seq(3, t, 4, (2,)), seq(3, t + 1, 4, (2,))
        g = run(est, [f], [c], True, prev)
        assert_pair_equal(g, 0, host_pair(ctx, f, c, M, True, row(prev, 0)), t)
        for j in range(M):
            if g["label"][0, j] == -1:
                continue
            true = c["true_of"][int(g["label"][0, j])]
            if true == 2:
                assert g["cls"][0, j] == capi.OT_STATIC and g["id"][0, j] == -1
                n = g["n_samples"][0]
                assert (g["obj_label"][0, :n][g["sample_slot"][0, :n] == j] == 0).all()
            elif g["cls"][0, j] == capi.OT_DYNAMIC:
                assert id_of.setdefault(true, int(g["id"][0, j])) == g["id"][0, j], (t, true)
        prev = prev_of(g)
    assert len(id_of) >= 2 and len(set(id_of.values())) == len(id_of)


def test_classes_gate_and_shared_ids(ctx):
    M = 8
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    f, c = seq(0, 0, 3), seq(0, 1, 3)
    g = run(est, [f], [c], shrink=(H // 2, W // 2))                # the border band covers the image: every object is boundary
    assert set(g["cls"][0][g["label"][0] != -1].tolist()) == {capi.OT_BOUNDARY}
    g = run(est, [f], [c], step=16)                                 # fewer than 150 points each: far / small
    assert set(g["cls"][0][g["label"][0] != -1].tolist()) == {capi.OT_FAR}
    assert_pair_equal(g, 0, host_pair(ctx, f, c, M, step=16))
    # a gate that fails: stat 0, so the next call hands the same objects new IDs (the reference looks IDs up only where bObjStat)
    g0 = run(est, [f], [c], min_inliers=10 ** 6)
    dyn = g0["cls"][0] == capi.OT_DYNAMIC
    assert dyn.sum() >= 2 and (g0["stat"][0][dyn] == 0).all()
    g1 = run(est, [c], [seq(0, 2, 3)], prev=prev_of(g0))
    assert_pair_equal(g1, 0, host_pair(ctx, c, seq(0, 2, 3), M, prev=row(prev_of(g0), 0)))
    d1 = g1["cls"][0] == capi.OT_DYNAMIC
    assert not set(g1["id"][0][d1].tolist()) & set(g0["id"][0][dyn].tolist())
    # one object split into two current instances: both vote for its last label and share its ID
    f0, f1, f2 = seq(0, 0, 3), seq(0, 1, 3), seq(0, 2, 3)
    g0 = run(est, [f0], [f1])
    labs, cnt = np.unique(f2["mask"][f2["mask"] != 0], return_counts=True)
    L = int(labs[np.argmax(cnt)])
    c2 = dict(f2, mask=f2["mask"].copy())
    ys, xs = np.nonzero(c2["mask"] == L)
    right = xs > np.median(xs)
    c2["mask"][ys[right], xs[right]] = 999
    g1 = run(est, [f1], [c2], prev=prev_of(g0))
    assert_pair_equal(g1, 0, host_pair(ctx, f1, c2, M, prev=row(prev_of(g0), 0)))
    ja, jb = list(g1["label"][0]).index(L), list(g1["label"][0]).index(999)
    assert g1["cls"][0, ja] == g1["cls"][0, jb] == capi.OT_DYNAMIC
    assert g1["id"][0, ja] == g1["id"][0, jb] and g1["vote"][0, ja] == g1["vote"][0, jb]


# ------------------------------------------------------------------------------------------------ 3. batch independence
def test_batch_of_64_with_staggered_resets(ctx):
    M = 8
    cases = [(s % 4, s // 4 % 3, 3 + s % 3) for s in range(64)]
    est = capi.ObjectMotion(ctx, 64, M, CAP)
    one = capi.ObjectMotion(ctx, 1, M, CAP)
    last = [seq(*c) for c in cases]
    cur = [seq(s, t + 1, n) for s, t, n in cases]
    g0 = run(est, last, cur)
    prev = prev_of(g0)
    for p in range(0, 64, 3):                                       # these pairs start a new sequence
        for k, v in R.reset_state(M).items():
            prev[k][p] = v
    nxt = [seq(s, t + 2, n) for s, t, n in cases]
    g = run(est, cur, nxt, prev=prev)
    for p in range(64):
        a = run(one, [cur[p]], [nxt[p]], prev={k: v[p:p + 1] for k, v in prev.items()})
        for k in g:
            assert np.array_equal(g[k][p], a[k][0]), (p, k)


# ------------------------------------------------------------------------------------------------ 4. edge cases
def test_edge_cases(ctx):
    M = 2
    est = capi.ObjectMotion(ctx, 1, M, CAP)
    f, c = seq(2, 1, 5), seq(2, 2, 5)
    g = run(est, [f], [c])                                          # five objects, two slots
    assert g["pair_status"][0] & capi.OM_PAIR_OBJECT_CAP
    assert_pair_equal(g, 0, host_pair(ctx, f, c, M))
    n = g["n_samples"][0]
    assert (g["obj_label"][0, :n] == -2).sum() > 0
    g = run(est, [f], [dict(c, mask=np.zeros_like(c["mask"]))])     # no object in the current frame
    assert (g["label"][0] == -1).all() and (g["obj_label"][0, :g["n_samples"][0]] == -1).all() and g["max_id"][0] == 1
    m64 = c["mask"].astype(np.int64)
    m64[m64 != 0] += 1 << 33                                        # an i64 label outside int32
    est.track([tens(f["depth"])], [tens(f["flow"])], [tens(f["mask"])], [tens(c["depth"])], [tens(m64)], KITTI_K, out=(o := filled(est, 1)))
    torch.cuda.synchronize()
    assert o["pair_status"][0].item() & capi.OM_PAIR_LABEL_RANGE and (o["label"][0] == -1).all()
    # CHW flow, cropped and transposed planes equal the contiguous ones
    big = lambda a: torch.zeros((a.shape[0] + 8, a.shape[1] + 16) + a.shape[2:], dtype=a.dtype, device=DEV)
    crop = lambda a: (lambda b: (b[3:3 + a.shape[0], 5:5 + a.shape[1]].copy_(a), b[3:3 + a.shape[0], 5:5 + a.shape[1]])[1])(big(a))
    tr = lambda a: a.t().contiguous().t() if a.dim() == 2 else a
    ref = run(est, [f], [c], poses=False)
    for mk in (crop, tr):
        o = filled(est, 1)
        est.track([mk(tens(f["depth"]))], [tens(f["flow"]).permute(2, 0, 1).contiguous()], [mk(tens(f["mask"]))], [mk(tens(c["depth"]))],
                  [mk(tens(c["mask"]))], KITTI_K, out=o)
        torch.cuda.synchronize()
        got = host_of(o)
        for k in ref:
            assert np.array_equal(got[k], ref[k]), k


# ------------------------------------------------------------------------------------------------ 5. CUDA graph of the whole chain
def test_cuda_graph_of_the_chain_equals_eager(ctx):
    """extract -> match -> PnP -> refine -> track captured once; replays over frames alternate two out / prev sets"""
    pairs = [(0, 1), (2, 3)]
    seeds = [(0, 3), (1, 4)]
    ex = capi.OrbExtractor(ctx, W, H, 4, n_features=3000)
    solver, refiner, est = capi.PnpSolver(ctx, 2, ex.capacity), capi.PoseRefiner(ctx, 2, ex.capacity), capi.ObjectMotion(ctx, 2, 8, CAP)
    vs_of = lambda t: [make_view_pair(t=t, seed=s, width=W, height=H) for s, _ in seeds]
    gray_of = lambda vv: tens(np.stack([g for v in vv for g in (v["gray_a"], v["gray_b"])]))
    fr = lambda t, k: tens(np.stack([seq(s, t, n)[k] for s, n in seeds]))
    vv = vs_of(0)
    img, dcam = gray_of(vv), tens(np.stack([v["depth_a"] for v in vv]))
    d, fl, mk, dc, mc = fr(0, "depth"), fr(0, "flow"), fr(0, "mask"), fr(1, "depth"), fr(1, "mask")
    Tq = tens(np.stack([v["Tcw_a"] for v in vv]).astype(np.float32))
    Tq_h = Tq.cpu().numpy()
    eo, mo = ex.empty_outputs(4), capi.orb_match_empty_outputs(ctx, 2, ex.capacity, ex.capacity, 2)
    po_, ro = solver.empty_outputs(2, ex.capacity), refiner.empty_outputs(2, ex.capacity)
    outs = [est.empty_outputs(2, track=True), est.empty_outputs(2, track=True)]
    prev0 = {k: tens(np.stack([v] * 2)) for k, v in R.reset_state(8).items()}

    def chain(images, dcq, Tl, oo, prev, eo=None, mo=None, po_=None, ro=None, planes=None):
        r = ex.extract(images, out=eo)
        m = capi.orb_match(ctx, r, r, pairs, k=2, out=mo)
        s = solver.solve(r, r, pairs, m, dcq, KITTI_K, Tcw_query=Tq_h, ratio=0.8, out=po_)
        t = refiner.refine(r, r, pairs, m, dcq, KITTI_K, T_init=s["T"], mask=s["inlier"], Tcw_query=Tq_h, ratio=0.8, out=ro)
        return est.track(*(planes or (d, fl, mk, dc, mc)), KITTI_K, Tcw_last=Tl, Tcw_cur=t["T"], prev=prev, out=oo)

    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    graphs = [torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()]
    with torch.cuda.stream(side):
        for i, gr in enumerate(graphs):          # graph i writes outs[i] and takes outs[1 - i] as prev
            chain(img, dcam, Tq, outs[i], prev_of_t(outs[1 - i]), eo, mo, po_, ro)
            with torch.cuda.graph(gr, stream=side):
                chain(img, dcam, Tq, outs[i], prev_of_t(outs[1 - i]), eo, mo, po_, ro)
    torch.cuda.current_stream(DEV).wait_stream(side)
    for k, v in prev0.items():                   # the first replay starts the sequences
        outs[1][k].copy_(v)
    eager_prev = {k: v.clone() for k, v in prev0.items()}
    for t in range(4):
        vv = vs_of(t)
        img.copy_(gray_of(vv)); dcam.copy_(tens(np.stack([v["depth_a"] for v in vv])))
        d.copy_(fr(t, "depth")); fl.copy_(fr(t, "flow")); mk.copy_(fr(t, "mask")); dc.copy_(fr(t + 1, "depth")); mc.copy_(fr(t + 1, "mask"))
        Tq.copy_(tens(np.stack([v["Tcw_a"] for v in vv]).astype(np.float32)))
        for v in outs[t % 2].values():           # the set this replay writes (the other one is its prev)
            v.fill_(FILL)
        graphs[t % 2].replay()
        torch.cuda.synchronize()
        got = host_of(outs[t % 2])
        planes = tuple(x.clone() for x in (d, fl, mk, dc, mc))
        eager = host_of(chain(gray_of(vv), tens(np.stack([v["depth_a"] for v in vv])), Tq.clone(), filled(est, 2), eager_prev, planes=planes))
        for k in eager:
            assert np.array_equal(got[k], eager[k]), (t, k)
        eager_prev = {k: tens(eager[k]) for k in ("label", "id", "stat", "H", "max_id")}
        assert (got["cls"] == capi.OT_DYNAMIC).sum() >= 3
    assert (got["id"][got["cls"] == capi.OT_DYNAMIC] < 6).all()          # the IDs persisted: no ID was handed out per frame


def prev_of_t(o):
    return {k: o[k] for k in ("label", "id", "stat", "H", "max_id")}


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_python_refusals_write_nothing(ctx):
    f, c = seq(0, 0, 3), seq(0, 1, 3)
    est = capi.ObjectMotion(ctx, 2, 4, CAP)
    d, fl, mk, dc, mc = tens(f["depth"]), tens(f["flow"]), tens(f["mask"]), tens(c["depth"]), tens(c["mask"])
    out = filled(est, 1)
    ok = dict(depths=[d], flows=[fl], masks=[mk], depths_cur=[dc], masks_cur=[mc], K=KITTI_K, out=out)
    est_prev = est.empty_outputs(1)
    tr_prev = est.empty_outputs(1, track=True)
    bad = [dict(depths_cur=[]), dict(depths_cur=[dc[:100]]), dict(masks_cur=[mc[:, :100]]), dict(masks_cur=[mc.float()]), dict(depths_cur=[dc.cpu()]),
           dict(sf_mg_thres=float("nan")), dict(sf_ds_thres=float("nan")), dict(shrink=(-1, 0)), dict(step=0), dict(quirk=2),
           dict(prev=est_prev), dict(prev=dict(tr_prev, id=tr_prev["id"][:, :2])), dict(prev={k: v for k, v in tr_prev.items() if k != "stat"}),
           dict(out=est.empty_outputs(1)), dict(out=dict(out, flow3d=out["flow3d"][..., :2]))]
    for b in bad:
        with pytest.raises(ValueError):
            est.track(**dict(ok, **b))
    torch.cuda.synchronize()
    for k, t in out.items():
        assert (t == FILL).all(), k


def test_c_refusals_write_nothing(ctx):
    f, c = seq(0, 0, 3), seq(0, 1, 3)
    M = 4
    est = capi.ObjectMotion(ctx, 2, M, CAP)
    out = filled(est, 1)
    d, fl, mk, dc, mc = tens(f["depth"]), tens(f["flow"]), tens(f["mask"]), tens(c["depth"]), tens(c["mask"])
    pl = {k: capi._dev_plane(ctx, kd, v, W, H) for k, kd, v in (("d", "depth", d), ("f", "flow", fl), ("m", "mask", mk), ("dc", "depth", dc),
                                                                 ("mc", "mask", mc))}
    prev = {k: tens(np.stack([v])) for k, v in R.reset_state(M).items()}
    host_buf = np.zeros(1 << 16, np.int32)
    keys = list(out)
    om_keys = keys[:len(capi.ObjMotionOut._fields_)]

    def o_with(**kw):
        ptr = {k: out[k].data_ptr() for k in keys}
        ptr.update(kw)
        return capi.ObjTrackOut(capi.ObjMotionOut(*[ptr[k] for k in om_keys]), *[ptr[k] for k in keys[len(om_keys):]])

    opt = lambda **kw: capi.ObjTrackOpts(**dict(dict(step=4, th_depth_obj=25.0, iters=500, min_inliers=50, thr=0.4, conf=0.98, quirk=1, sf_mg_thres=0.12,
                                                     sf_ds_thres=0.3, shrink_row=25, shrink_col=50), **kw))

    def call(opts=None, o=None, dcp=None, mcp=None, pv=None):
        arr = lambda p_: (capi.DevPlane * 1)(p_)
        wh = np.array([[W, H]], np.int32)
        K = np.asarray([KITTI_K], np.float32)
        p = dict({k: v.data_ptr() for k, v in prev.items()}, **(pv or {}))
        return ctx.L.vdo_obj_track_batch_dev(est.h_, C.c_int(1), arr(pl["d"]), arr(pl["f"]), arr(pl["m"]), arr(dcp or pl["dc"]), arr(mcp or pl["mc"]),
                                             wh.ctypes.data_as(C.POINTER(C.c_int32)), K.ctypes.data_as(C.POINTER(C.c_float)), None, None,
                                             *[C.c_void_p(p[k]) for k in ("label", "id", "stat", "H", "max_id")], C.byref(opts or opt()),
                                             C.byref(o or o_with()), C.c_uint64(0))

    bad = {
        "sf_mg NaN": dict(opts=opt(sf_mg_thres=float("nan"))), "sf_ds NaN": dict(opts=opt(sf_ds_thres=float("nan"))),
        "shrink < 0": dict(opts=opt(shrink_col=-1)), "step 0": dict(opts=opt(step=0)),
        "prev partly given": dict(pv=dict(stat=None)), "prev_max_id host memory": dict(pv=dict(max_id=host_buf.ctypes.data)),
        "depth_cur u8": dict(dcp=capi.DevPlane(pl["dc"].data_dev, capi.VDO_DT_U8, 1, W, 1, 0, 1)),
        "mask_cur misaligned": dict(mcp=capi.DevPlane(pl["mc"].data_dev + 2, capi.VDO_DT_I32, 1, W, 1, 0, 1)),
        "out.id NULL": dict(o=o_with(id=None)), "out.flow3d host memory": dict(o=o_with(flow3d=host_buf.ctypes.data)),
        "out.motion.H misaligned": dict(o=o_with(H=out["H"].data_ptr() + 2)),
    }
    torch.cuda.synchronize()
    for what, kw in bad.items():
        assert call(**kw) == ERR_ARG, what
        assert ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_obj_track_batch_dev"), what
    torch.cuda.synchronize()
    for k, t in out.items():
        assert (t == FILL).all(), k
    assert call() == 0
    torch.cuda.synchronize()
    assert out["n_samples"][0] > 0 and out["max_id"][0] >= 1
