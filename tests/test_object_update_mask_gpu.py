"""Objects the segmentation missed, recovered in the current masks on the device (capi.ObjectMotion.update_mask /
vdo_obj_update_mask_batch_dev).

Every result is compared with the host route: Frame.upload + Frame.sample_objects on the last frame, then capi.update_mask
(vdo_update_mask) on resident frames with the samples of the kept slots.  The host route reports the updated mask and the recovered
labels; a slot's vote is checked against the mask the host route leaves after the slots below it (the route run on their samples only).
Inputs: synth.make_sequence_frame pairs with stable labels, where objects are dropped from the current mask by zeroing their label, and
small hand-made planes for the slot order and the vote boundaries."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from tests import object_track_reference as R
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame, make_view_pair

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
CAP = ((W + 3) // 4) * ((H + 3) // 4)
CAP2 = ((W + 1) // 2) * ((H + 1) // 2)
FILL = 7
MASK_FILL = 123456


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@functools.lru_cache(maxsize=None)
def seq(seed, t, n_obj, w=W, h=H):
    """frame t of sequence seed with its stable labels 1 .. n_obj: metric depth, flow, mask, true Tcw"""
    f = make_sequence_frame(t, seed=seed, width=w, height=h, n_obj=n_obj)
    raw = f["depth_raw"]
    depth = np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
    return dict(depth=depth, flow=f["flow"], mask=f["mask"], Tcw=np.linalg.inv(f["Twc"]).astype(np.float32), vel=f["obj_vel"], gray=f["gray"])


def dropped(mask, labels):
    m = mask.copy()
    m[np.isin(m, list(labels))] = 0
    return m


def visible(f):
    labs, cnt = np.unique(f["mask"][f["mask"] != 0], return_counts=True)
    return [int(v) for v in labs[np.argsort(-cnt)]]


def tens(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def filled(est, P):
    o = est.empty_outputs(P, update_mask=True)
    for t in o.values():
        t.fill_(FILL)
    return o


def host_of(o):
    return {k: v.cpu().numpy() for k, v in o.items()}


def host_route(ctx, depth, flow, mask, mask_cur, M, step=4, th=25.0, upto=None):
    """(updated mask, recovered labels, samples, kept slot labels): vdo_frame_sample_objects + vdo_update_mask on the first `upto` slots"""
    h, w = depth.shape
    last, cur = capi.Frame(ctx, w, h), capi.Frame(ctx, w, h)
    last.upload(depth=depth, flow=flow, mask=mask)
    cur.upload(mask=np.asarray(mask_cur).astype(np.int32))
    s = last.sample_objects(th, step)
    slots = sorted(set(s["label"].tolist()))[:M]
    keep = np.isin(s["label"], slots[:upto])
    out, warped = capi.update_mask(cur, last, s["label"][keep], np.stack([s["cx"][keep], s["cy"][keep]], 1))
    last.close(); cur.close()
    return out, warped, s, slots


def expected(ctx, depth, flow, mask, mask_cur, M, step=4, th=25.0):
    """one pair's result as the host route gives it: the updated mask and update_mask()'s per-slot and per-pair outputs"""
    h, w = depth.shape
    out, warped, s, slots = host_route(ctx, depth, flow, mask, mask_cur, M, step, th)
    r = dict(mask=out, label=np.full(M, -1, np.int32), n_vote=np.zeros(M, np.int32), vote=np.zeros(M, np.int32), recovered=np.zeros(M, np.int32),
             n_samples=len(s["x"]), pair_status=capi.OM_PAIR_OBJECT_CAP if len(set(s["label"].tolist())) > M else 0)
    u, v = s["cx"].astype(np.int64), s["cy"].astype(np.int64)
    inside = (u < w) & (u > 0) & (v < h) & (v > 0)
    for j, L in enumerate(slots):
        sel = inside & (s["label"] == L)
        r["label"][j], r["n_vote"][j], r["recovered"][j] = L, sel.sum(), int(L in warped)
        if sel.sum() >= 100:
            seen = host_route(ctx, depth, flow, mask, mask_cur, M, step, th, upto=j)[0] if j else np.asarray(mask_cur).astype(np.int32)
            r["vote"][j] = R.majority(seen[v[sel], u[sel]])
            assert (r["vote"][j] == 0) == bool(r["recovered"][j])
    return r


def run(est, last, masks_cur, step=4, th=25.0, out=None):
    """update_mask on tensors; returns (result, updated masks as numpy)"""
    out = filled(est, len(last)) if out is None else out
    est.update_mask([tens(f["depth"]) for f in last], [tens(f["flow"]) for f in last], [tens(f["mask"]) for f in last], masks_cur, step=step,
                    th_depth_obj=th, out=out)
    torch.cuda.synchronize()
    return host_of(out), [m.cpu().numpy() for m in masks_cur]


def assert_pair_equal(g, p, mask_got, r, what=""):
    assert np.array_equal(mask_got.astype(np.int64), r["mask"].astype(np.int64)), what
    assert g["n_samples"][p] == r["n_samples"] and g["pair_status"][p] == r["pair_status"], what
    for k in ("label", "n_vote", "vote", "recovered"):
        assert np.array_equal(g[k][p], r[k]), (what, k, g[k][p], r[k])


# ------------------------------------------------------------------------------------------------ 1. equal to the host route
@pytest.mark.parametrize("th", [25.0, 14.0])
@pytest.mark.parametrize("step", [4, 2])
def test_equal_to_host_route(ctx, step, th):
    """pairs with 0, 1 and 2 dropped objects, i32 and i64 masks, HWC and CHW flow, contiguous, cropped and transposed planes, and a strided
    mask_cur (every other column of a wider tensor, or a transposed one)"""
    M = 8
    cases = [(0, 0, 3, 0), (1, 0, 4, 1), (2, 1, 5, 2), (3, 2, 4, 1), (0, 3, 3, 2), (1, 4, 4, 0)]
    P = len(cases)
    est = capi.ObjectMotion(ctx, P, M, CAP2 if step == 2 else CAP)
    big = lambda a: torch.zeros((a.shape[0] + 8, a.shape[1] + 16) + a.shape[2:], dtype=a.dtype, device=DEV)
    crop = lambda a: (lambda b: (b[3:3 + a.shape[0], 5:5 + a.shape[1]].copy_(a), b[3:3 + a.shape[0], 5:5 + a.shape[1]])[1])(big(a))
    tr = lambda a: a.transpose(0, 1).contiguous().transpose(0, 1)
    d, fl, mk, mc, refs, wides = [], [], [], [], [], []
    for p, (s, t, n, drop) in enumerate(cases):
        f, c = seq(s, t, n), seq(s, t + 1, n)
        cm = dropped(c["mask"], visible(c)[:drop])
        dt = torch.int64 if p % 2 else torch.int32
        lay = [lambda a: a, crop, tr][p % 3]
        d.append(lay(tens(f["depth"])))
        fl.append(tens(f["flow"]).permute(2, 0, 1).contiguous() if p % 2 else lay(tens(f["flow"])))
        mk.append(lay(tens(f["mask"]).to(dt)))
        if p % 3 == 1:
            wides.append(torch.full((H, 2 * W), MASK_FILL, dtype=dt, device=DEV))
            mc.append(wides[-1][:, ::2])
            mc[-1].copy_(tens(cm).to(dt))
        else:
            mc.append(tr(tens(cm).to(dt)) if p % 3 == 2 else tens(cm).to(dt))
        refs.append(expected(ctx, f["depth"], f["flow"], f["mask"], cm, M, step, th))
    out = filled(est, P)
    est.update_mask(d, fl, mk, mc, step=step, th_depth_obj=th, out=out)
    torch.cuda.synchronize()
    g = host_of(out)
    for p in range(P):
        assert_pair_equal(g, p, mc[p].cpu().numpy(), refs[p], p)
    for wd in wides:                                               # the other columns of the wide tensors are untouched
        assert (wd[:, 1::2] == MASK_FILL).all()
    rec = sum(int(g["recovered"][p].sum()) for p in range(P))
    assert rec >= sum(c[3] for c in cases) - 2, rec                # the dropped objects come back (a far or hidden one may not vote)


# ------------------------------------------------------------------------------------------------ 2. the slot order
def planes(w=320, h=120):
    return dict(depth=np.full((h, w), 10.0, np.float32), flow=np.zeros((h, w, 2), np.float32), mask=np.zeros((h, w), np.int32))


def one(ctx, f, cm, M=8):
    est = capi.ObjectMotion(ctx, 1, M, ((f["depth"].shape[1] + 3) // 4) * ((f["depth"].shape[0] + 3) // 4))
    mc = tens(cm)
    g, m = run(est, [f], [mc])
    r = expected(ctx, f["depth"], f["flow"], f["mask"], cm, M)
    assert_pair_equal(g, 0, m[0], r)
    return g, m[0]


def test_earlier_recovery_decides_a_later_slot(ctx):
    """A (5) and B (7) are both missing; A's push covers B's targets, so B sees 5 and is not recovered"""
    f = planes()
    f["mask"][20:60, 20:100] = 5
    f["flow"][20:60, 20:100, 0] = 130.0                            # A lands on columns 150 .. 229
    f["mask"][20:60, 150:230] = 7                                  # B stays where it is
    g, m = one(ctx, f, np.zeros_like(f["mask"]))
    assert g["label"][0, :2].tolist() == [5, 7] and g["recovered"][0, :2].tolist() == [1, 0] and g["vote"][0, 1] == 5
    assert (m[20:60, 150:230] == 5).all() and (m == 7).sum() == 0


def test_the_higher_slot_wins_a_shared_pixel(ctx):
    """A (5) and B (7) are both recovered and their pushes share columns 150 .. 169; a higher label (50) there before loses to B"""
    f = planes()
    f["mask"][70:110, 20:90] = 5
    f["flow"][70:110, 20:90, 0] = 80.0                             # A -> columns 100 .. 169
    f["mask"][70:110, 150:230] = 7                                 # B stays: columns 150 .. 229
    cm = np.zeros_like(f["mask"])
    cm[70:110, 160:164] = 50
    g, m = one(ctx, f, cm)
    assert g["recovered"][0, :2].tolist() == [1, 1]
    assert (m[70:110, 100:150] == 5).all() and (m[70:110, 150:230] == 7).all()


# ------------------------------------------------------------------------------------------------ 3. vote boundaries
def test_vote_boundaries(ctx):
    """100 samples per object (a 40 x 40 box on the step-4 raster, zero flow): 99 voters (one target on the u = 0 edge) are skipped, 100
    vote; 0 tied with 9 recovers, 0 tied with -5 does not; a target with v = 0 does not vote"""
    f = planes(400, 120)
    boxes = {3: (8, 4), 4: (8, 80), 6: (8, 160), 8: (8, 240), 10: (64, 320)}
    for L, (y, x) in boxes.items():
        f["mask"][y:y + 40, x:x + 40] = L
    f["flow"][8, 4, 0] = -3.5                                      # label 3: target x 0.5, a sample whose u = 0 does not vote
    f["flow"][64, 320, 1] = -63.5                                  # label 10: target y 0.5, v = 0
    cm = np.zeros_like(f["mask"])
    cm[8:28, 160:200] = 9                                          # label 6: half 9, half 0
    cm[8:28, 240:280] = -5                                         # label 8: half -5, half 0
    g, m = one(ctx, f, cm)
    got = dict(zip(g["label"][0].tolist(), zip(g["n_vote"][0].tolist(), g["vote"][0].tolist(), g["recovered"][0].tolist())))
    assert got[3] == (99, 0, 0) and got[4] == (100, 0, 1) and got[6] == (100, 0, 1) and got[8] == (100, -5, 0) and got[10] == (99, 0, 0)
    assert (m[8:48, 4:44] == 0).all() and (m[8:48, 80:120] == 4).all()


# ------------------------------------------------------------------------------------------------ 4. caps and ranges
def test_object_cap_and_label_range(ctx):
    f, c = seq(2, 1, 5), seq(2, 2, 5)
    cm = dropped(c["mask"], visible(c)[:3])
    est = capi.ObjectMotion(ctx, 1, 2, CAP)
    mc = tens(cm)
    g, m = run(est, [f], [mc])
    assert g["pair_status"][0] & capi.OM_PAIR_OBJECT_CAP
    assert_pair_equal(g, 0, m[0], expected(ctx, f["depth"], f["flow"], f["mask"], cm, 2))
    est = capi.ObjectMotion(ctx, 1, 8, CAP)
    m64 = f["mask"].astype(np.int64)
    m64[m64 == visible(f)[0]] += 1 << 33                           # an out-of-range label in the last mask, at its largest object
    mc = tens(cm.astype(np.int64))
    o = filled(est, 1)
    est.update_mask([tens(f["depth"])], [tens(f["flow"])], [tens(m64)], [mc], out=o)
    torch.cuda.synchronize()
    assert o["pair_status"][0].item() & capi.OM_PAIR_LABEL_RANGE and (o["recovered"][0] == 0).all()
    assert np.array_equal(mc.cpu().numpy(), cm)
    c64 = cm.astype(np.int64)
    c64[c["mask"] == visible(c)[0]] = 1 << 33                      # an out-of-range label in the current mask, under the dropped object's voters
    mc = tens(c64)
    o = filled(est, 1)
    est.update_mask([tens(f["depth"])], [tens(f["flow"])], [tens(f["mask"])], [mc], out=o)
    torch.cuda.synchronize()
    assert o["pair_status"][0].item() & capi.OM_PAIR_LABEL_RANGE and (o["recovered"][0] == 0).all()
    assert np.array_equal(mc.cpu().numpy(), c64)


# ------------------------------------------------------------------------------------------------ 5. idempotent
def test_second_call_changes_nothing(ctx):
    cases = [(0, 0, 3, 1), (1, 0, 4, 2)]
    est = capi.ObjectMotion(ctx, 2, 8, CAP)
    last = [seq(s, t, n) for s, t, n, _ in cases]
    mc = [tens(dropped(seq(s, t + 1, n)["mask"], visible(seq(s, t + 1, n))[:k])) for s, t, n, k in cases]
    g, m1 = run(est, last, mc)
    assert g["recovered"].sum() >= 2
    g2, m2 = run(est, last, mc)
    assert g2["recovered"].sum() == 0
    for a, b in zip(m1, m2):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ 6. batch independence
def test_batch_of_64_mixed_sizes(ctx):
    sizes = [(W, H), (640, 192)]
    cases = [(s % 4, s // 4 % 3, 3 + s % 3, sizes[s % 2], s % 3) for s in range(64)]
    est, alone = capi.ObjectMotion(ctx, 64, 8, CAP), capi.ObjectMotion(ctx, 1, 8, CAP)
    last = [seq(s, t, n, *wh) for s, t, n, wh, _ in cases]
    cms = [dropped(seq(s, t + 1, n, *wh)["mask"], visible(seq(s, t + 1, n, *wh))[:k]) for s, t, n, wh, k in cases]
    mc = [tens(m) for m in cms]
    g, m = run(est, last, mc)
    assert g["recovered"].sum() >= 20
    for p in range(64):
        a, ma = run(alone, [last[p]], [tens(cms[p])])
        assert np.array_equal(m[p], ma[0]), p
        for k in g:
            assert np.array_equal(g[k][p], a[k][0]), (p, k)


# ------------------------------------------------------------------------------------------------ 7. the dropout, end to end
def test_dropout_keeps_the_object_id(ctx):
    """an 8-frame sequence with stable labels where a moving object is missing from frame 4's mask: update_mask then track per pair keeps its
    ID and gives it a motion at the dropout pair; track alone hands it a new ID after the gap"""
    M, seed, n = 8, 3, 4
    frames = [dict(seq(seed, t, n)) for t in range(9)]
    L = visible(frames[4])[0]
    frames[4]["mask"] = dropped(frames[4]["mask"], [L])
    est = capi.ObjectMotion(ctx, 1, M, CAP)

    def sequence(with_update):
        prev, ids, masks = None, [], [f["mask"] for f in frames]
        for t in range(8):
            f, c = dict(frames[t], mask=masks[t]), frames[t + 1]
            cm = c["mask"]
            if with_update:
                mc = tens(cm)
                g, _ = run(est, [f], [mc])
                cm = mc.cpu().numpy()
                host_cm = expected(ctx, f["depth"], f["flow"], f["mask"], c["mask"], M)["mask"]
                assert np.array_equal(cm, host_cm), t
                masks[t + 1] = cm
            cc = dict(c, mask=cm)
            o = est.empty_outputs(1, track=True)
            est.track([tens(f["depth"])], [tens(f["flow"])], [tens(f["mask"])], [tens(cc["depth"])], [tens(cm)], KITTI_K, Tcw_last=tens(f["Tcw"][None]),
                      Tcw_cur=tens(cc["Tcw"][None]), prev=None if prev is None else {k: tens(v) for k, v in prev.items()}, out=o)
            torch.cuda.synchronize()
            tr = host_of(o)
            ref = R.host_track(ctx, f["depth"], f["flow"], f["mask"], cc["depth"], cm, KITTI_K, M, f["Tcw"], cc["Tcw"],
                               None if prev is None else {k: v[0] for k, v in prev.items()})
            for k in ("label", "id", "cls", "vote", "stat", "H", "velocity"):
                assert np.array_equal(tr[k][0], ref[k]), (t, k)
            j = [s for s in range(M) if tr["label"][0, s] == L and tr["cls"][0, s] == capi.OT_DYNAMIC]
            ids.append((int(tr["id"][0, j[0]]), tr["velocity"][0, j[0]], int(tr["stat"][0, j[0]])) if j else None)
            prev = {k: tr[k] for k in ("label", "id", "stat", "H", "max_id")}
        return ids

    ids = sequence(True)
    assert all(ids[t] is not None for t in (2, 3, 4, 5)) and len({x[0] for x in ids if x is not None}) == 1, ids
    vel = frames[3]["vel"][L]
    assert ids[3][2] == 1 and np.linalg.norm(ids[3][1] - vel) < 0.2, (ids[3], vel)
    plain = sequence(False)
    assert plain[3] is None                                        # the object has no slot at the dropout
    assert plain[2] is not None and plain[5] is not None and plain[2][0] != plain[5][0], plain    # and comes back under a new ID


# ------------------------------------------------------------------------------------------------ 8. CUDA graph of the whole chain
def test_cuda_graph_of_the_chain_equals_eager(ctx):
    """extract -> match -> PnP -> refine -> update_mask -> track captured once and replayed over frames with a dropped object"""
    pairs = [(0, 1), (2, 3)]
    seeds = [(0, 3), (1, 4)]
    ex = capi.OrbExtractor(ctx, W, H, 4, n_features=3000)
    solver, refiner, est = capi.PnpSolver(ctx, 2, ex.capacity), capi.PoseRefiner(ctx, 2, ex.capacity), capi.ObjectMotion(ctx, 2, 8, CAP)
    vs_of = lambda t: [make_view_pair(t=t, seed=s, width=W, height=H) for s, _ in seeds]
    gray_of = lambda vv: tens(np.stack([g for v in vv for g in (v["gray_a"], v["gray_b"])]))
    fr = lambda t, k: tens(np.stack([seq(s, t, n)[k] for s, n in seeds]))
    cur_mask = lambda t: tens(np.stack([dropped(seq(s, t, n)["mask"], visible(seq(s, t, n))[:1]) for s, n in seeds]))
    vv = vs_of(0)
    img, dcam = gray_of(vv), tens(np.stack([v["depth_a"] for v in vv]))
    d, fl, mk, dc, mc = fr(0, "depth"), fr(0, "flow"), fr(0, "mask"), fr(1, "depth"), cur_mask(1)
    Tq = tens(np.stack([v["Tcw_a"] for v in vv]).astype(np.float32))
    Tq_h = Tq.cpu().numpy()
    eo, mo = ex.empty_outputs(4), capi.orb_match_empty_outputs(ctx, 2, ex.capacity, ex.capacity, 2)
    po_, ro = solver.empty_outputs(2, ex.capacity), refiner.empty_outputs(2, ex.capacity)
    uo, to_ = est.empty_outputs(2, update_mask=True), est.empty_outputs(2, track=True)

    def chain(images, dcq, planes, uo=None, to_=None, eo=None, mo=None, po_=None, ro=None):
        r = ex.extract(images, out=eo)
        m = capi.orb_match(ctx, r, r, pairs, k=2, out=mo)
        s = solver.solve(r, r, pairs, m, dcq, KITTI_K, Tcw_query=Tq_h, ratio=0.8, out=po_)
        t = refiner.refine(r, r, pairs, m, dcq, KITTI_K, T_init=s["T"], mask=s["inlier"], Tcw_query=Tq_h, ratio=0.8, out=ro)
        u = est.update_mask(*planes[:3], planes[4], out=uo)
        return u, est.track(*planes, KITTI_K, Tcw_cur=t["T"], out=to_)

    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        chain(img, dcam, (d, fl, mk, dc, mc.clone()), uo, to_, eo, mo, po_, ro)
        with torch.cuda.graph(graph, stream=side):
            chain(img, dcam, (d, fl, mk, dc, mc), uo, to_, eo, mo, po_, ro)
    torch.cuda.current_stream(DEV).wait_stream(side)
    for t in range(3):
        vv = vs_of(t)
        img.copy_(gray_of(vv)); dcam.copy_(tens(np.stack([v["depth_a"] for v in vv])))
        d.copy_(fr(t, "depth")); fl.copy_(fr(t, "flow")); mk.copy_(fr(t, "mask")); dc.copy_(fr(t + 1, "depth")); mc.copy_(cur_mask(t + 1))
        planes = tuple(x.clone() for x in (d, fl, mk, dc, mc))
        for v in list(uo.values()) + list(to_.values()):
            v.fill_(FILL)
        graph.replay()
        torch.cuda.synchronize()
        got_u, got_t, got_m = host_of(uo), host_of(to_), mc.cpu().numpy()
        eu, et = chain(gray_of(vv), tens(np.stack([v["depth_a"] for v in vv])), planes, filled(est, 2),
                       {k: v.fill_(FILL) for k, v in est.empty_outputs(2, track=True).items()})
        torch.cuda.synchronize()
        assert np.array_equal(got_m, planes[4].cpu().numpy()), t
        for k, v in host_of(eu).items():
            assert np.array_equal(got_u[k], v), (t, k)
        for k, v in host_of(et).items():
            assert np.array_equal(got_t[k], v), (t, k)
        assert got_u["recovered"].sum() >= 2


# ------------------------------------------------------------------------------------------------ 9. refusals
def test_python_refusals_write_nothing(ctx):
    f, c = seq(0, 0, 3), seq(0, 1, 3)
    est = capi.ObjectMotion(ctx, 2, 4, CAP)
    d, fl, mk = tens(f["depth"]), tens(f["flow"]), tens(f["mask"])
    cm = dropped(c["mask"], visible(c)[:1])
    mc = tens(cm)
    out, out2 = filled(est, 1), filled(est, 2)
    ok = dict(depths=[d], flows=[fl], masks=[mk], masks_cur=[mc], out=out)
    zero = torch.as_strided(tens(cm), (H, W), (0, 1))                       # every row on one row
    fold = torch.as_strided(torch.zeros(2 * W * H, dtype=torch.int32, device=DEV), (H, W), (W // 2, 1))   # rows overlap
    mc2 = tens(cm)
    bad = [dict(masks_cur=[]), dict(masks_cur=[mc[:100]]), dict(masks_cur=[mc.float()]), dict(masks_cur=[mc.cpu()]), dict(step=0),
           dict(th_depth_obj=float("nan")), dict(out=est.empty_outputs(1)), dict(out=dict(out, vote=out["vote"][:, :2])),
           dict(masks_cur=[zero]), dict(masks_cur=[fold]),
           dict(masks_cur=[mk]),                                                 # the last mask as the current one
           dict(depths=[d, d], flows=[fl, fl], masks=[mk, mk], masks_cur=[mc2, mc2], out=out2),       # one current mask for two pairs
           dict(depths=[d, d], flows=[fl, fl], masks=[mk, mc2], masks_cur=[mc, mc2], out=out2)]       # pair 1's last mask is its current
    msgs = []
    for b in bad:
        with pytest.raises(ValueError) as e:
            est.update_mask(**dict(ok, **b))
        msgs.append(str(e.value))
    assert "pair 0" in msgs[-3] and "pair 0" in msgs[-2] and "mask_cur" in msgs[-1] and "pair" in msgs[-1]
    torch.cuda.synchronize()
    for k, t in list(out.items()) + list(out2.items()):
        assert (t == FILL).all(), k
    for m in (mc, mc2):
        assert np.array_equal(m.cpu().numpy(), cm)


def test_c_refusals_write_nothing(ctx):
    f, c = seq(0, 0, 3), seq(0, 1, 3)
    est = capi.ObjectMotion(ctx, 2, 4, CAP)
    out = filled(est, 1)
    cm = dropped(c["mask"], visible(c)[:1])
    d, fl, mk, mc = tens(f["depth"]), tens(f["flow"]), tens(f["mask"]), tens(cm)
    pl = {k: capi._dev_plane(ctx, kd, v, W, H) for k, kd, v in (("d", "depth", d), ("f", "flow", fl), ("m", "mask", mk), ("mc", "mask", mc))}
    host_buf = np.zeros(1 << 16, np.int32)
    keys = list(out)
    wh1 = np.array([[W, H]], np.int32)

    def o_with(**kw):
        ptr = {k: out[k].data_ptr() for k in keys}
        ptr.update(kw)
        return capi.ObjMaskOut(*[ptr[k] for k in keys])

    def call(P=1, step=4, th=25.0, o=None, mcp=None, mp=None, wh=None, nullcur=False):
        arr = lambda p_: (capi.DevPlane * P)(*([p_] * P))
        whp = np.tile(wh1, (P, 1)) if wh is None else wh
        return ctx.L.vdo_obj_update_mask_batch_dev(est.h_, C.c_int(P), arr(pl["d"]), arr(pl["f"]), arr(mp or pl["m"]), None if nullcur else arr(mcp or pl["mc"]),
                                                   whp.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int32(step), C.c_float(th), C.byref(o or o_with()),
                                                   C.c_uint64(0))

    plane = lambda p_, **kw: capi.DevPlane(**dict(dict(data_dev=p_.data_dev, dtype=p_.dtype, channels=1, stride_y=p_.stride_y, stride_x=p_.stride_x,
                                                       stride_c=0, rgb=1), **kw))
    bad = {
        "P 0": dict(P=0), "P 3": dict(P=3), "step 0": dict(step=0), "th NaN": dict(th=float("nan")), "mask_cur NULL": dict(nullcur=True),
        "mask_cur f32": dict(mcp=plane(pl["mc"], dtype=capi.VDO_DT_F32)), "mask_cur 2 channels": dict(mcp=plane(pl["mc"], channels=2)),
        "mask_cur misaligned": dict(mcp=plane(pl["mc"], data_dev=pl["mc"].data_dev + 2)),
        "mask_cur host memory": dict(mcp=plane(pl["mc"], data_dev=host_buf.ctypes.data)),
        "mask_cur zero stride": dict(mcp=plane(pl["mc"], stride_y=0)), "mask_cur rows overlap": dict(mcp=plane(pl["mc"], stride_y=W - 1)),
        "mask_cur zero x stride": dict(mcp=plane(pl["mc"], stride_x=0, stride_y=W)),
        "mask_cur on the last mask": dict(mcp=pl["m"]), "mask_cur shared by two pairs": dict(P=2),
        "size above the cap": dict(wh=np.array([[W + 8, H]], np.int32)), "width 0": dict(wh=np.array([[0, H]], np.int32)),
        "out.vote NULL": dict(o=o_with(vote=None)), "out.n_vote host memory": dict(o=o_with(n_vote=host_buf.ctypes.data)),
        "out.label misaligned": dict(o=o_with(label=out["label"].data_ptr() + 2)),
    }
    torch.cuda.synchronize()
    for what, kw in bad.items():
        assert call(**kw) == ERR_ARG, what
        assert ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_obj_update_mask_batch_dev"), what
    torch.cuda.synchronize()
    for k, t in out.items():
        assert (t == FILL).all(), k
    assert np.array_equal(mc.cpu().numpy(), cm)
    assert call(mcp=plane(pl["mc"], stride_y=-W, data_dev=pl["mc"].data_dev + 4 * W * (H - 1))) == 0    # rows upside down: distinct
    torch.cuda.synchronize()
    assert out["n_samples"][0] > 0 and out["recovered"][0].sum() >= 0
