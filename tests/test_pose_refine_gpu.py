"""Refined poses of matched ORB frame pairs on the device (capi.PoseRefiner / vdo_pose_refine_batch_dev).

The problems the device gathers from the matches are gathered again on the host (tests/pnp_match_reference.gather, restricted by the mask)
and given to capi.pose_opt_flow2 (mode 0): pose, LM statistics, flows and inlier flags must be identical.  Inputs: the synth.make_view_pair
views of tests/test_pnp_match_gpu.py refined from PnpSolver's result, and synthetic keypoint sets large enough for the single-CTA kernel.
Also: oracle parity, accuracy against the synthetic truth, batch independence at 64 pairs, the edge cases, a CUDA graph of
extract -> match -> PnP -> refine, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle as po
from tests import pnp_match_reference as R
from tests.test_pnp_match_gpu import SETTINGS, VIEWS
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_K, make_view_pair

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
FILL = 7                                  # fill of the output tensors: slots the call must not write keep it
CL_MAX_N = 11376                          # VDO_FLOW2_CLUSTER_MAX_N
EYE = np.eye(4, dtype=np.float32)


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.fixture(scope="module")
def views(ctx):
    """frames a0, b0, a1, b1, ... of the view pairs: ORB keypoints (host copies too) and depths of every frame"""
    vs = [make_view_pair(width=W, height=H, **kw) for kw in VIEWS]
    grays = [g for v in vs for g in (v["gray_a"], v["gray_b"])]
    ex = capi.OrbExtractor(ctx, W, H, len(grays), n_features=3000)
    r = ex.extract(torch.from_numpy(np.stack(grays)).to(DEV))
    S = {k: r[k].clone() for k in ("descriptors", "x", "y", "count")}
    torch.cuda.synchronize()
    assert (r["status"] == 0).all() and (S["count"] > 1000).all()
    depths = [torch.from_numpy(d).to(DEV) for v in vs for d in (v["depth_a"], v["depth_b"])]
    depths_h = [d for v in vs for d in (v["depth_a"], v["depth_b"])]
    return dict(vs=vs, S=S, Sh={k: S[k].cpu().numpy() for k in S}, depths=depths, depths_h=depths_h, cap=ex.capacity)


def filled(refiner, P, qcap):
    o = refiner.empty_outputs(P, qcap)
    for t in o.values():
        t.fill_(FILL)
    return o


def host_of(o):
    return {k: v.cpu().numpy() for k, v in o.items()}


def host_problems(Sh, pairs, idx, dist, depths_h, K, Tcw, T_init, mask, ratio, max_depth):
    """per pair: (query indices of the problem's points, the problem as capi.pose_opt_flow2 takes it)"""
    out = []
    for p, (q, t) in enumerate(pairs):
        sel, obj, img = R.gather(Sh["x"][q], Sh["y"][q], Sh["count"][q], Sh["x"][t], Sh["y"][t], Sh["count"][t], idx[p], dist[p], depths_h[p], K,
                                 None, ratio, max_depth)
        keep = np.ones(len(sel), bool) if mask is None else mask[p][sel] != 0
        sel, z, img = sel[keep], obj[keep, 2], img[keep]
        pts = np.stack([Sh["x"][q][sel], Sh["y"][q][sel]], 1).astype(np.float32)
        out.append((sel, dict(pts=pts, depth=z.astype(np.float32), flow=(img - pts).astype(np.float32), K=np.asarray(K, np.float32),
                              Tcw_last=EYE if Tcw is None else np.asarray(Tcw[p], np.float32), T_init=np.asarray(T_init[p], np.float32))))
    return out


def assert_equal_to_host(ctx, g, probs, counts, quirk):
    ref = capi.pose_opt_flow2(ctx, [pb for _, pb in probs], quirk=quirk, modes=[0] * len(probs))
    for p, ((sel, _), r) in enumerate(zip(probs, ref)):
        nq = int(counts[p])
        assert g["n_points"][p] == len(sel), p
        assert np.array_equal(g["T"][p], r["T"]), p
        assert np.array_equal(g["stats"][p], r["stats"]), p
        assert np.array_equal(g["flow"][p, sel], r["flow"]), p
        assert np.array_equal(g["inlier"][p, sel], r["inlier"].astype(np.uint8)), p
        rest = np.setdiff1d(np.arange(nq), sel)
        assert (g["inlier"][p, rest] == 0).all() and (g["inlier"][p, nq:] == FILL).all(), p
        assert (g["flow"][p, rest] == FILL).all() and (g["flow"][p, nq:] == FILL).all(), p
    return ref


def pnp(ctx, views, pairs, m, Tcw, ratio, max_depth, k, thr=0.4):
    solver = capi.PnpSolver(ctx, len(pairs), views["cap"], 500)
    return solver.solve(views["S"], views["S"], pairs, m, [views["depths"][q] for q, _ in pairs], KITTI_K, Tcw_query=Tcw, ratio=ratio,
                        max_depth=max_depth, thr=thr)


def match(ctx, S, pairs, k):
    return capi.orb_match(ctx, S, S, pairs, k=k, cross_check=k == 1)


def view_pairs(views):
    nv = len(views["vs"])
    return [(2 * i, 2 * i + 1) for i in range(nv)]


# ------------------------------------------------------------------------------------------------ 1. equal to the host entry
@pytest.mark.parametrize("quirk", [0, 1])
@pytest.mark.parametrize("use_mask", [True, False])
@pytest.mark.parametrize("k,ratio,max_depth,use_tcw,iters,thr", SETTINGS)
def test_equal_to_host_entry(ctx, views, k, ratio, max_depth, use_tcw, iters, thr, use_mask, quirk):
    pairs = view_pairs(views)
    P = len(pairs)
    m = match(ctx, views["S"], pairs, k)
    Tcw = np.stack([v["Tcw_a"] for v in views["vs"]]).astype(np.float32) if use_tcw else None
    res = pnp(ctx, views, pairs, m, Tcw, ratio, max_depth, k, thr)
    refiner = capi.PoseRefiner(ctx, 8, views["cap"])
    out = filled(refiner, P, views["cap"])
    refiner.refine(views["S"], views["S"], pairs, m, [views["depths"][q] for q, _ in pairs], KITTI_K, T_init=res["T"],
                   mask=res["inlier"] if use_mask else None, Tcw_query=Tcw, ratio=ratio, max_depth=max_depth, quirk=quirk, out=out)
    g = host_of(out)
    mask = res["inlier"].cpu().numpy() if use_mask else None
    probs = host_problems(views["Sh"], pairs, m["idx"].cpu().numpy(), m["dist"].cpu().numpy(), [views["depths_h"][q] for q, _ in pairs], KITTI_K,
                          Tcw, res["T"].cpu().numpy(), mask, ratio, max_depth)
    assert all(len(sel) > 10 for sel, _ in probs)
    assert_equal_to_host(ctx, g, probs, [views["Sh"]["count"][q] for q, _ in pairs], quirk)
    assert (g["status"] == 0).all() and (g["stats"][:, 0] > 0).all()


# ------------------------------------------------------------------------------------------------ 2. oracle parity, 3. accuracy
def _rot_err_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))))


def test_oracle_parity(ctx, views):
    pairs = view_pairs(views)[:1]
    m = match(ctx, views["S"], pairs, 2)
    Tcw = np.stack([views["vs"][0]["Tcw_a"]]).astype(np.float32)
    res = pnp(ctx, views, pairs, m, Tcw, 0.8, None, 2)
    g = host_of(capi.PoseRefiner(ctx, 1, views["cap"]).refine(views["S"], views["S"], pairs, m, [views["depths"][0]], KITTI_K, T_init=res["T"],
                                                                mask=res["inlier"], Tcw_query=Tcw, ratio=0.8))
    (_, pb), = host_problems(views["Sh"], pairs, m["idx"].cpu().numpy(), m["dist"].cpu().numpy(), [views["depths_h"][0]], KITTI_K, Tcw,
                             res["T"].cpu().numpy(), res["inlier"].cpu().numpy(), 0.8, None)
    o = po.flow2(pb, mode=0, quirk=1)
    assert np.abs(g["T"][0] - o["T"]).max() <= 1e-4


def test_accuracy_from_pnp(ctx, views):
    pairs = view_pairs(views)
    m = match(ctx, views["S"], pairs, 2)
    refiner = capi.PoseRefiner(ctx, 8, views["cap"])
    Tcw = np.stack([v["Tcw_a"] for v in views["vs"]]).astype(np.float32)
    dp = [views["depths"][q] for q, _ in pairs]
    for tcw in (None, Tcw):
        res = pnp(ctx, views, pairs, m, tcw, 0.8, None, 2, thr=2.0)
        g = host_of(refiner.refine(views["S"], views["S"], pairs, m, dp, KITTI_K, T_init=res["T"], mask=res["inlier"], Tcw_query=tcw, ratio=0.8))
        for p, v in enumerate(views["vs"]):
            truth = v["T_ba"] if tcw is None else v["Tcw_b"]
            T = g["T"][p].astype(np.float64)
            assert g["status"][p] == 0 and g["n_points"][p] > 200 and g["stats"][p, 0] > 0, p
            assert _rot_err_deg(T[:3, :3], truth[:3, :3]) < 0.2, p
            assert np.linalg.norm(T[:3, 3] - truth[:3, 3]) < 0.05, p


# ------------------------------------------------------------------------------------------------ 4. batch independence
def test_batch_of_64_equals_each_pair_alone(ctx, views):
    F = 2 * len(views["vs"])
    pairs = [(q, t) for q in range(F) for t in range(F)]
    assert len(pairs) == 64
    m = match(ctx, views["S"], pairs, 2)
    Tcw = np.stack([views["vs"][q // 2]["Tcw_a" if q % 2 == 0 else "Tcw_b"] for q, _ in pairs]).astype(np.float32)
    depths = [views["depths"][q] for q, _ in pairs]
    res = capi.PnpSolver(ctx, 64, views["cap"], 500).solve(views["S"], views["S"], pairs, m, depths, KITTI_K, Tcw_query=Tcw, ratio=0.8, max_depth=40.0, thr=2.0)
    refiner = capi.PoseRefiner(ctx, 64, views["cap"])
    kw = dict(Tcw_query=Tcw, ratio=0.8, max_depth=40.0)
    gb = host_of(refiner.refine(views["S"], views["S"], pairs, m, depths, KITTI_K, T_init=res["T"], mask=res["inlier"], out=filled(refiner, 64, views["cap"]), **kw))
    assert (gb["n_points"] > 200).any() and (gb["n_points"] < 3).any()     # pairs of one view pair, and unrelated frames with few PnP inliers
    for p, pr in enumerate(pairs):
        ms = {k: m[k][p:p + 1] for k in ("idx", "dist")}
        g1 = host_of(refiner.refine(views["S"], views["S"], [pr], ms, [depths[p]], KITTI_K, T_init=res["T"][p:p + 1], mask=res["inlier"][p:p + 1],
                                    out=filled(refiner, 1, views["cap"]), **dict(kw, Tcw_query=Tcw[p:p + 1])))
        for k in g1:
            assert np.array_equal(g1[k][0], gb[k][p]), (p, k)


# ------------------------------------------------------------------------------------------------ 5. both kernel shapes in one call
def synthetic_sets(counts, cap, seed=5, noise=0.3):
    """F = len(counts) query frames of cap keypoints at distinct pixels over a random depth plane, train frames holding their projections
    under a known small motion (plus noise in px); idx[p, i] = i for pair p = (p, p)"""
    rng = np.random.default_rng(seed)
    K = KITTI_K.astype(np.float64)
    depth = rng.uniform(4, 40, (H, W)).astype(np.float32)
    Rm = np.eye(3); t = np.array([0.02, -0.01, -0.8])
    c = 0.01; Rm[0, 0] = Rm[2, 2] = np.cos(c); Rm[0, 2] = np.sin(c); Rm[2, 0] = -np.sin(c)
    qx, qy, tx, ty = (np.zeros((len(counts), cap), np.float32) for _ in range(4))
    for f in range(len(counts)):
        pix = rng.choice(W * H, cap, replace=False)
        u = (pix % W + rng.uniform(0, 0.99, cap)).astype(np.float32); v = (pix // W + rng.uniform(0, 0.99, cap)).astype(np.float32)
        z = depth[v.astype(int), u.astype(int)].astype(np.float64)
        X = np.stack([(u - K[2]) * z / K[0], (v - K[3]) * z / K[1], z], 1) @ Rm.T + t
        qx[f], qy[f] = u, v
        tx[f] = K[0] * X[:, 0] / X[:, 2] + K[2] + rng.normal(0, noise, cap)
        ty[f] = K[1] * X[:, 1] / X[:, 2] + K[3] + rng.normal(0, noise, cap)
    T = np.eye(4, dtype=np.float32); T[:3, :3] = Rm; T[:3, 3] = t
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    q = {"x": torch.from_numpy(qx).to(DEV), "y": torch.from_numpy(qy).to(DEV), "count": cnt}
    tr = {"x": torch.from_numpy(tx).to(DEV), "y": torch.from_numpy(ty).to(DEV), "count": cnt.clone()}
    P = len(counts)
    idx = torch.arange(cap, dtype=torch.int32, device=DEV).reshape(1, cap, 1).repeat(P, 1, 1).contiguous()
    return dict(q=q, t=tr, m={"idx": idx, "dist": torch.zeros_like(idx)}, depth=depth, depth_t=torch.from_numpy(depth).to(DEV), T=T,
                h={"x": qx, "y": qy, "count": np.asarray(counts)}, th={"x": tx, "y": ty})


def test_both_kernel_shapes_in_one_call(ctx):
    cap = 12000
    counts = [cap, 700, CL_MAX_N, CL_MAX_N + 1, 2]
    d = synthetic_sets(counts, cap)
    P = len(counts)
    pairs = [(p, p) for p in range(P)]
    refiner = capi.PoseRefiner(ctx, P, cap)
    T0 = torch.from_numpy(np.stack([EYE] * P)).to(DEV)
    for quirk in (0, 1):
        out = filled(refiner, P, cap)
        refiner.refine(d["q"], d["t"], pairs, d["m"], [d["depth_t"]] * P, KITTI_K, T_init=T0, quirk=quirk, out=out)
        g = host_of(out)
        Sh = {"x": np.concatenate([d["h"]["x"], d["th"]["x"]]), "y": np.concatenate([d["h"]["y"], d["th"]["y"]]),
              "count": np.concatenate([counts, counts])}
        hp = [(p, P + p) for p in range(P)]                  # host view: train frame p is row P + p
        idx, dist = d["m"]["idx"].cpu().numpy(), d["m"]["dist"].cpu().numpy()
        probs = host_problems(Sh, hp, idx, dist, [d["depth"]] * P, KITTI_K, None, np.stack([EYE] * P), None, None, None)
        assert [len(s) for s, _ in probs] == counts
        assert_equal_to_host(ctx, g, probs, counts, quirk)
        for p in range(P - 1):
            assert np.abs(g["T"][p][:3, 3] - d["T"][:3, 3]).max() < 0.05, p


# ------------------------------------------------------------------------------------------------ 6. edge cases
def test_edge_cases(ctx, views):
    pairs = view_pairs(views)[:2]
    m = match(ctx, views["S"], pairs, 2)
    res = pnp(ctx, views, pairs, m, None, 0.8, None, 2)
    refiner = capi.PoseRefiner(ctx, 2, views["cap"])
    dp = [views["depths"][q] for q, _ in pairs]
    cap, nq = views["cap"], [int(views["Sh"]["count"][q]) for q, _ in pairs]

    def run(S=views["S"], T_init=res["T"], mask=res["inlier"]):
        out = filled(refiner, 2, cap)
        refiner.refine(S, S, pairs, m, dp, KITTI_K, T_init=T_init, mask=mask, ratio=0.8, out=out)
        return host_of(out)

    # n < 3: an empty mask, and a mask of two correspondences: identity, stats[0] = -1, the prior flows, no inliers
    two = torch.zeros_like(res["inlier"])
    sel2 = [np.nonzero(res["inlier"][p].cpu().numpy())[0][:2] for p in range(2)]
    for p in range(2):
        two[p, torch.from_numpy(sel2[p]).to(DEV)] = 1
    for mask, n in ((torch.zeros_like(res["inlier"]), 0), (two, 2)):
        g = run(mask=mask)
        for p, (q, t) in enumerate(pairs):
            assert g["n_points"][p] == n and g["status"][p] == 0
            assert np.array_equal(g["T"][p], EYE) and g["stats"][p, 0] == -1 and (g["stats"][p, 1:] == 0).all()
            assert (g["inlier"][p, :nq[p]] == 0).all() and (g["inlier"][p, nq[p]:] == FILL).all()
            if n:
                i = sel2[p]
                j = m["idx"][p, i, 0].cpu().numpy()
                prior = np.stack([views["Sh"]["x"][t][j] - views["Sh"]["x"][q][i], views["Sh"]["y"][t][j] - views["Sh"]["y"][q][i]], 1)
                assert np.array_equal(g["flow"][p, i], prior.astype(np.float64))
    # counts outside 0 .. cap set the status bits and give no points; the query row is not written when count[q] is out of range
    for bad in (-1, cap + 1):
        cnt = views["S"]["count"].clone()
        cnt[pairs[0][0]] = bad
        cnt[pairs[1][1]] = bad
        g = run(S=dict(views["S"], count=cnt))
        assert g["status"][0] == capi.PNP_STATUS_QUERY_COUNT and g["status"][1] == capi.PNP_STATUS_TRAIN_COUNT
        assert (g["n_points"] == 0).all() and (g["stats"][:, 0] == -1).all()
        assert (g["inlier"][0] == FILL).all() and (g["inlier"][1, :nq[1]] == 0).all()
    # an initial pose from a motion model (not PnP) is accepted and refined as the host entry refines it
    mm = res["T"].clone()
    mm[:, :3, 3] *= 0.9
    g = run(T_init=mm)
    probs = host_problems(views["Sh"], pairs, m["idx"].cpu().numpy(), m["dist"].cpu().numpy(), [views["depths_h"][q] for q, _ in pairs], KITTI_K,
                          None, mm.cpu().numpy(), res["inlier"].cpu().numpy(), 0.8, None)
    assert_equal_to_host(ctx, g, probs, nq, 1)


# ------------------------------------------------------------------------------------------------ 7. capture of the whole chain
def test_cuda_graph_of_the_chain_equals_eager(ctx):
    vs = [make_view_pair(width=W, height=H, **kw) for kw in VIEWS[:2]]
    vs2 = [make_view_pair(width=W, height=H, **dict(kw, seed=kw["seed"] + 10)) for kw in VIEWS[:2]]
    frames = lambda vv: torch.from_numpy(np.stack([g for v in vv for g in (v["gray_a"], v["gray_b"])])).to(DEV)
    depth_of = lambda vv: torch.from_numpy(np.stack([v["depth_a"] for v in vv])).to(DEV)
    pairs = [(0, 1), (2, 3)]
    Tcw_of = lambda vv: np.stack([v["Tcw_a"] for v in vv]).astype(np.float32)
    ex = capi.OrbExtractor(ctx, W, H, 4, n_features=3000)
    solver, refiner = capi.PnpSolver(ctx, 2, ex.capacity, 500), capi.PoseRefiner(ctx, 2, ex.capacity)
    img, dep = frames(vs), depth_of(vs)
    Tq = Tcw_of(vs)                                          # host parameters: captured with the call
    eo, mo = ex.empty_outputs(4), capi.orb_match_empty_outputs(ctx, 2, ex.capacity, ex.capacity, 2)
    po_, ro = solver.empty_outputs(2, ex.capacity), refiner.empty_outputs(2, ex.capacity)

    def chain(images, depths, Tcw, eo=None, mo=None, po_=None, ro=None):
        r = ex.extract(images, out=eo)
        m = capi.orb_match(ctx, r, r, pairs, k=2, out=mo)
        s = solver.solve(r, r, pairs, m, depths, KITTI_K, Tcw_query=Tcw, ratio=0.8, out=po_)
        return refiner.refine(r, r, pairs, m, depths, KITTI_K, T_init=s["T"], mask=s["inlier"], Tcw_query=Tcw, ratio=0.8, out=ro)

    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        chain(img, dep, Tq, eo, mo, po_, ro)                 # warm-up on the side stream
        with torch.cuda.graph(g, stream=side):
            chain(img, dep, Tq, eo, mo, po_, ro)
    torch.cuda.current_stream(DEV).wait_stream(side)
    for vv in (vs, vs2):
        img.copy_(frames(vv)); dep.copy_(depth_of(vv))
        for t in ro.values():
            t.fill_(FILL)
        g.replay()
        torch.cuda.synchronize()
        got = host_of(ro)
        eager = host_of(chain(frames(vv), depth_of(vv), Tq, ro=filled(refiner, 2, ex.capacity)))
        assert (got["n_points"] > 50).all()
        for k in eager:
            assert np.array_equal(got[k], eager[k]), k


# ------------------------------------------------------------------------------------------------ 8. refusals
def test_python_refusals(ctx, views):
    S, cap = views["S"], views["cap"]
    pairs = [(0, 1)]
    m = match(ctx, S, pairs, 2)
    m1 = match(ctx, S, pairs, 1)
    refiner = capi.PoseRefiner(ctx, 2, cap)
    d = [views["depths"][0]]
    T0 = torch.from_numpy(EYE[None].copy()).to(DEV)
    mk = torch.ones((1, cap), dtype=torch.uint8, device=DEV)
    ok = dict(query=S, train=S, pairs=pairs, matches=m, depths=d, K=KITTI_K, T_init=T0, mask=mk)
    bad = [dict(pairs=[]), dict(pairs=[(0, 1)] * 3), dict(pairs=[(0, 99)]), dict(depths=[d[0].double()]), dict(depths=[d[0].cpu()]),
           dict(depths=[d[0], d[0]]), dict(matches={"idx": m["idx"].long(), "dist": m["dist"]}), dict(matches={"idx": m["idx"][:, :100], "dist": m["dist"]}),
           dict(matches=m1, ratio=0.8), dict(ratio=float("nan")), dict(max_depth=float("nan")), dict(quirk=2), dict(quirk=-1),
           dict(T_init=None), dict(T_init=T0.double()), dict(T_init=T0.cpu()), dict(T_init=T0[:, :3]), dict(mask=mk.bool()), dict(mask=mk[:, :10]),
           dict(mask=mk.cpu()), dict(K=np.zeros(3)), dict(Tcw_query=np.eye(3)), dict(query=dict(S, x=S["x"].cpu())),
           dict(train=dict(S, count=S["count"].long())), dict(out=dict(refiner.empty_outputs(1), T=torch.empty((1, 4, 4), dtype=torch.float64, device=DEV))),
           dict(out=dict(refiner.empty_outputs(1), flow=torch.empty((1, cap, 2), dtype=torch.float32, device=DEV)))]
    for b in bad:
        with pytest.raises(ValueError):
            refiner.refine(**dict(ok, **b))
    with pytest.raises(ValueError):
        capi.PoseRefiner(ctx, 1, 100).refine(**ok)            # query capacity above the refiner's cap


def test_c_refusals_write_nothing(ctx, views):
    S, cap = views["S"], views["cap"]
    m = match(ctx, S, [(0, 1)], 2)
    refiner = capi.PoseRefiner(ctx, 2, cap)
    out = filled(refiner, 2, cap)
    T0 = torch.from_numpy(np.stack([EYE] * 2)).to(DEV)
    mk = torch.ones((2, cap), dtype=torch.uint8, device=DEV)
    L = ctx.L
    host_buf = np.zeros(1 << 20, np.int32)
    nf = S["x"].shape[0]
    dp = capi._dev_plane(ctx, "depth", views["depths"][0], W, H)

    def call(P=1, pr=((0, 1),), qs=None, ts=None, idx=None, dist=None, plane=None, wh=(W, H), opts=None, o=None, Ti=None, mask=None):
        qs = qs or capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), nf, cap)
        ts = ts or capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), nf, cap)
        plane = plane or dp
        n = max(P, 1)
        planes = (capi.DevPlane * n)(*([plane] * n))
        pa = np.ascontiguousarray(np.array(list(pr) * n, np.int32)[:n])
        whs = np.ascontiguousarray(np.tile(np.array(wh, np.int32), (n, 1)))
        Ks = np.ascontiguousarray(np.tile(np.asarray(KITTI_K, np.float32), (n, 1)))
        o = o or o_with()
        opts = opts or capi.PoseRefineOpts(2, 0.8, 0.0, 1)
        return L.vdo_pose_refine_batch_dev(refiner.h_, C.c_int(P), pa.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(qs), C.byref(ts),
                                           C.c_void_p(m["idx"].data_ptr() if idx is None else idx), C.c_void_p(m["dist"].data_ptr() if dist is None else dist),
                                           planes, whs.ctypes.data_as(C.POINTER(C.c_int32)), Ks.ctypes.data_as(C.POINTER(C.c_float)), None,
                                           C.c_void_p(T0.data_ptr() if Ti is None else Ti), C.c_void_p(mk.data_ptr() if mask is None else mask),
                                           C.byref(opts), C.byref(o), C.c_uint64(0))

    def o_with(**kw):
        ptr = {k: out[v].data_ptr() for k, v in (("T_dev", "T"), ("flow_dev", "flow"), ("inlier_dev", "inlier"), ("n_points_dev", "n_points"),
                                                  ("stats_dev", "stats"), ("status_dev", "status"))}
        ptr.update(kw)
        return capi.PoseRefineOut(**ptr)

    bad = {
        "P = 0": dict(P=0), "P = 3 > max_pairs": dict(P=3), "frame out of range": dict(pr=((0, nf),)), "negative frame": dict(pr=((-1, 0),)),
        "query cap above the refiner's": dict(qs=capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), nf, cap + 1)),
        "train n_frames 0": dict(ts=capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), 0, cap)),
        "k = 3": dict(opts=capi.PoseRefineOpts(3, 0.0, 0.0, 1)), "ratio with k = 1": dict(opts=capi.PoseRefineOpts(1, 0.8, 0.0, 1)),
        "ratio NaN": dict(opts=capi.PoseRefineOpts(2, float("nan"), 0.0, 1)), "max_depth NaN": dict(opts=capi.PoseRefineOpts(2, 0.8, float("nan"), 1)),
        "quirk 2": dict(opts=capi.PoseRefineOpts(2, 0.8, 0.0, 2)), "quirk -1": dict(opts=capi.PoseRefineOpts(2, 0.8, 0.0, -1)),
        "depth u8": dict(plane=capi.DevPlane(dp.data_dev, capi.VDO_DT_U8, 1, dp.stride_y, dp.stride_x, 0, 1)),
        "depth host memory": dict(plane=capi.DevPlane(host_buf.ctypes.data, capi.VDO_DT_F32, 1, W, 1, 0, 1)),
        "depth misaligned": dict(plane=capi.DevPlane(dp.data_dev + 2, capi.VDO_DT_F32, 1, dp.stride_y, dp.stride_x, 0, 1)),
        "depth width 0": dict(wh=(0, H)),
        "idx NULL": dict(idx=0), "idx host memory": dict(idx=host_buf.ctypes.data), "dist misaligned": dict(dist=m["dist"].data_ptr() + 1),
        "query.y NULL": dict(qs=capi.OrbDescSet(None, S["x"].data_ptr(), None, S["count"].data_ptr(), nf, cap)),
        "T_init NULL": dict(Ti=0), "T_init host memory": dict(Ti=host_buf.ctypes.data), "T_init misaligned": dict(Ti=T0.data_ptr() + 2),
        "mask host memory": dict(mask=host_buf.ctypes.data),
        "out.T NULL": dict(o=o_with(T_dev=None)), "out.flow misaligned": dict(o=o_with(flow_dev=out["flow"].data_ptr() + 4)),
        "out.stats host memory": dict(o=o_with(stats_dev=host_buf.ctypes.data)), "out.status NULL": dict(o=o_with(status_dev=None)),
        "out.inlier NULL": dict(o=o_with(inlier_dev=None)), "out.n_points NULL": dict(o=o_with(n_points_dev=None)),
    }
    torch.cuda.synchronize()
    for what, kw in bad.items():
        assert call(**kw) == ERR_ARG, what
        assert L.vdo_last_error(ctx.h).decode().startswith("vdo_pose_refine_batch_dev"), what
    torch.cuda.synchronize()
    for k, t in out.items():
        assert (t == FILL).all(), k                       # nothing was written
    assert call() == 0                                   # the same arguments otherwise run
    torch.cuda.synchronize()
    assert (out["n_points"][:1] > 0).all() and (out["n_points"][1:] == FILL).all()
    for mp, c in ((65, cap), (0, cap), (1, 0)):
        with pytest.raises(capi.VdoError):
            capi.PoseRefiner(ctx, mp, c)
    info = refiner.info()
    assert info["max_pairs"] == 2 and info["cap"] == cap and info["device_bytes"] > 0
    big = capi.PoseRefiner(ctx, 1, CL_MAX_N + 1)        # the single-CTA scratch is held only above the cluster limit
    assert big.info()["device_bytes"] - capi.PoseRefiner(ctx, 1, CL_MAX_N).info()["device_bytes"] >= (CL_MAX_N + 1) * 18 * 8
