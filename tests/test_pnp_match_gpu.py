"""Poses of matched ORB frame pairs on the device (capi.PnpSolver / vdo_pnp_match_batch_dev).

The correspondences the device gathers from the matches are gathered again on the host (tests/pnp_match_reference.py) and given to
capi.init_model_batch with no motion model: pose, refit, inlier set and RANSAC counters must be identical.  Inputs: synth.make_view_pair
views (KITTI-shaped, 3 000 ORB features, matched with orb_match), and planted matches with known outliers (cross-checked against
cv2.solvePnPRansac).  Also: accuracy against the synthetic truth, batch independence at 64 pairs, the edge cases, CUDA-graph replay and the
refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import pnp_match_reference as R
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_K, make_view_pair

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
W, H = 1242, 375
FILL = 7                                  # fill of the output tensors: slots the call must not write keep it
VIEWS = [dict(t=0, seed=0, dt=1), dict(t=4, seed=1, dt=2, yaw_extra=0.02), dict(t=9, seed=2, dt=1, shift=(0.3, 0.05, 0.0)),
         dict(t=2, seed=3, dt=3, yaw_extra=-0.015, shift=(-0.2, 0.0, 0.1))]


@pytest.fixture(scope="module")
def ctx():
    return capi.Context(0)


@pytest.fixture(scope="module")
def views(ctx):
    """frames a0, b0, a1, b1, ... of the view pairs: ORB keypoints and descriptors (host copies too), depths of every frame"""
    vs = [make_view_pair(width=W, height=H, **kw) for kw in VIEWS]
    grays = [g for v in vs for g in (v["gray_a"], v["gray_b"])]
    ex = capi.OrbExtractor(ctx, W, H, len(grays), n_features=3000)
    r = ex.extract(torch.from_numpy(np.stack(grays)).to(DEV))
    S = {k: r[k].clone() for k in ("descriptors", "x", "y", "count")}
    torch.cuda.synchronize()
    assert (r["status"] == 0).all() and (S["count"] > 1000).all()
    depths = [torch.from_numpy(d).to(DEV) for v in vs for d in (v["depth_a"], v["depth_b"])]
    return dict(vs=vs, S=S, Sh={k: S[k].cpu().numpy() for k in S}, depths=depths, cap=ex.capacity)


def match(ctx, S, pairs, k):
    return capi.orb_match(ctx, S, S, pairs, k=k, cross_check=k == 1)


def filled(solver, P, qcap):
    o = solver.empty_outputs(P, qcap)
    for t in o.values():
        t.fill_(FILL)
    return o


def host_of(o):
    return {k: v.cpu().numpy() for k, v in o.items()}


def reference(ctx, Sh, pairs, m, depths_h, K, Tcw, ratio, max_depth, iters, thr, conf=0.98, K_train=None):
    """per pair: (sel, init_model_batch result or None when the gather is empty)"""
    idx, dist = m["idx"].cpu().numpy(), m["dist"].cpu().numpy()
    out = []
    for p, (q, t) in enumerate(pairs):
        sel, obj, img = R.gather(Sh["x"][q], Sh["y"][q], Sh["count"][q], Sh["x"][t], Sh["y"][t], Sh["count"][t], idx[p], dist[p], depths_h[p],
                                 K, None if Tcw is None else Tcw[p], ratio, max_depth)
        r = capi.init_model_batch(ctx, [dict(obj=obj, img=img)], np.asarray(K if K_train is None else K_train, np.float32), iters=iters, thr=thr, conf=conf)[0]
        out.append((sel, r))
    return out


def assert_equal_to_host(g, ref, counts):
    for p, (sel, r) in enumerate(ref):
        nq = int(counts[p])
        info = g["info"][p]
        assert g["n_corr"][p] == len(sel), p
        assert info[0] == r["iters_run"] and info[1] == r["best_it"] and info[2] == r["n_valid"], (p, info, r)
        assert np.array_equal(g["T"][p].reshape(16), r["T"].reshape(16)), p
        model = len(sel) >= 4 and r["best_it"] >= 0
        assert bool(info[3] & capi.PNP_STATUS_FEW_POINTS) == (len(sel) < 4) and bool(info[3] & capi.PNP_STATUS_NO_MODEL) == (len(sel) >= 4 and not model)
        if model:
            assert np.array_equal(g["Rt"][p], r["Rt"]), p
            assert np.array_equal(np.nonzero(g["inlier"][p, :nq])[0], sel[r["sub"]]), p
            assert g["n_inlier"][p] == len(r["sub"])
        else:
            assert g["n_inlier"][p] == 0 and not g["inlier"][p, :nq].any()
        assert (g["inlier"][p, nq:] == FILL).all()


# (k, ratio, max_depth, Tcw_query, iters, thr): every value of every setting, both match modes
SETTINGS = [(2, None, None, False, 500, 0.4), (2, 0.8, None, False, 500, 0.4), (2, 0.8, 40.0, True, 500, 0.4), (2, None, 40.0, True, 200, 2.0),
            (1, None, None, False, 500, 2.0), (1, None, 40.0, True, 200, 0.4), (2, 0.8, 40.0, False, 200, 2.0), (1, None, None, True, 500, 0.4)]


@pytest.mark.parametrize("k,ratio,max_depth,use_tcw,iters,thr", SETTINGS)
def test_equal_to_host_path(ctx, views, k, ratio, max_depth, use_tcw, iters, thr):
    nv = len(views["vs"])
    pairs = [(2 * i, 2 * i + 1) for i in range(nv)]
    m = match(ctx, views["S"], pairs, k)
    Tcw = np.stack([v["Tcw_a"] for v in views["vs"]]).astype(np.float32) if use_tcw else None
    solver = capi.PnpSolver(ctx, 8, views["cap"], 500)
    out = filled(solver, nv, views["cap"])
    solver.solve(views["S"], views["S"], pairs, m, [views["depths"][q] for q, _ in pairs], KITTI_K, Tcw_query=Tcw, ratio=ratio, max_depth=max_depth,
                 iters=iters, thr=thr, out=out)
    g = host_of(out)
    depths_h = [views["vs"][i]["depth_a"] for i in range(nv)]
    ref = reference(ctx, views["Sh"], pairs, m, depths_h, KITTI_K, Tcw, ratio, max_depth, iters, thr)
    assert all(len(sel) > 100 for sel, _ in ref)
    assert_equal_to_host(g, ref, [views["Sh"]["count"][q] for q, _ in pairs])


def _rot_err_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))))


def test_pose_accuracy_on_view_pairs(ctx, views):
    nv = len(views["vs"])
    pairs = [(2 * i, 2 * i + 1) for i in range(nv)]
    m = match(ctx, views["S"], pairs, 2)
    solver = capi.PnpSolver(ctx, 8, views["cap"], 500)
    Tcw = np.stack([v["Tcw_a"] for v in views["vs"]]).astype(np.float32)
    for tcw in (None, Tcw):
        g = host_of(solver.solve(views["S"], views["S"], pairs, m, [views["depths"][q] for q, _ in pairs], KITTI_K, Tcw_query=tcw, ratio=0.8, thr=2.0))
        for p, v in enumerate(views["vs"]):
            truth = v["T_ba"] if tcw is None else v["Tcw_b"]
            T = g["T"][p].astype(np.float64)
            assert g["info"][p, 3] == 0 and g["n_inlier"][p] > 200, (p, g["info"][p], g["n_inlier"][p])
            assert _rot_err_deg(T[:3, :3], truth[:3, :3]) < 0.2, p
            assert np.linalg.norm(T[:3, 3] - truth[:3, 3]) < 0.05, p


def planted(seed, n=1000, out_frac=0.3, noise=0.1):
    """one query frame of n keypoints at distinct pixels over a random depth plane, one train frame holding their projections under a
    known pose (noise in px, out_frac of them moved by up to 15 px); idx[i] = i"""
    rng = np.random.default_rng(seed)
    K = KITTI_K.astype(np.float64)
    pix = rng.choice(W * H, n, replace=False)
    u = (pix % W + rng.uniform(0, 0.99, n)).astype(np.float32); v = (pix // W + rng.uniform(0, 0.99, n)).astype(np.float32)
    depth = rng.uniform(4, 40, (H, W)).astype(np.float32)
    z = depth[v.astype(int), u.astype(int)].astype(np.float64)
    X = np.stack([(u - K[2]) * z / K[0], (v - K[3]) * z / K[1], z], 1)
    ang = rng.normal(0, 0.02, 3); th = np.linalg.norm(ang); a = ang / th
    Ax = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    Rm = np.eye(3) + np.sin(th) * Ax + (1 - np.cos(th)) * Ax @ Ax
    t = np.array([0.05, 0.01, -0.9]) + rng.normal(0, 0.05, 3)
    Xc = X @ Rm.T + t
    uv = np.stack([K[0] * Xc[:, 0] / Xc[:, 2] + K[2], K[1] * Xc[:, 1] / Xc[:, 2] + K[3]], 1) + rng.normal(0, noise, (n, 2))
    bad = rng.random(n) < out_frac
    uv[bad] += rng.uniform(-15, 15, (int(bad.sum()), 2))
    T = np.eye(4); T[:3, :3] = Rm; T[:3, 3] = t
    q = {"x": torch.from_numpy(u[None]).to(DEV), "y": torch.from_numpy(v[None]).to(DEV), "count": torch.tensor([n], dtype=torch.int32, device=DEV)}
    tr = {"x": torch.from_numpy(uv[None, :, 0].astype(np.float32).copy()).to(DEV), "y": torch.from_numpy(uv[None, :, 1].astype(np.float32).copy()).to(DEV),
          "count": torch.tensor([n], dtype=torch.int32, device=DEV)}
    ar = torch.arange(n, dtype=torch.int32, device=DEV).reshape(1, n, 1)
    m = {"idx": ar.clone(), "dist": torch.zeros_like(ar)}
    return dict(q=q, t=tr, m=m, depth=depth, depth_t=torch.from_numpy(depth).to(DEV), T=T, n=n)


@pytest.mark.parametrize("seed,out_frac", [(11, 0.2), (12, 0.3), (13, 0.4)])
def test_planted_against_cv2(ctx, seed, out_frac):
    cv2 = pytest.importorskip("cv2")
    d = planted(seed, out_frac=out_frac)
    solver = capi.PnpSolver(ctx, 1, d["n"], 500)
    g = host_of(solver.solve(d["q"], d["t"], [(0, 0)], d["m"], [d["depth_t"]], KITTI_K))
    qh, th = host_of(d["q"]), host_of(d["t"])
    sel, obj, img = R.gather(qh["x"][0], qh["y"][0], d["n"], th["x"][0], th["y"][0], d["n"], np.arange(d["n"])[:, None], np.zeros((d["n"], 1)), d["depth"], KITTI_K)
    assert len(sel) == d["n"] == g["n_corr"][0]
    Kc = np.array([[KITTI_K[0], 0, KITTI_K[2]], [0, KITTI_K[1], KITTI_K[3]], [0, 0, 1]], np.float64)
    ok, rv, tv, inl = cv2.solvePnPRansac(obj, img, Kc, np.zeros(4), iterationsCount=500, reprojectionError=0.4, confidence=0.98, flags=cv2.SOLVEPNP_AP3P)
    assert ok
    a, b = set(np.nonzero(g["inlier"][0])[0].tolist()), set(sel[inl.ravel()].tolist())
    assert len(a & b) / len(a | b) >= 0.95
    Rc, _ = cv2.Rodrigues(rv)
    Rt = g["Rt"][0]
    assert np.abs(Rt[:9].reshape(3, 3) - Rc).max() < 2e-3 and np.abs(Rt[9:] - tv.ravel()).max() < 2e-2
    assert np.abs(Rt[9:] - d["T"][:3, 3]).max() < 2e-2


def test_batch_of_64_equals_each_pair_alone(ctx, views):
    F = 2 * len(views["vs"])
    pairs = [(q, t) for q in range(F) for t in range(F)]
    assert len(pairs) == 64
    m = match(ctx, views["S"], pairs, 2)
    solver = capi.PnpSolver(ctx, 64, views["cap"], 500)
    Tcw = np.stack([views["vs"][q // 2]["Tcw_a" if q % 2 == 0 else "Tcw_b"] for q, _ in pairs]).astype(np.float32)
    kw = dict(ratio=0.8, max_depth=40.0, thr=2.0)
    depths = [views["depths"][q] for q, _ in pairs]
    gb = host_of(solver.solve(views["S"], views["S"], pairs, m, depths, KITTI_K, Tcw_query=Tcw, out=filled(solver, 64, views["cap"]), **kw))
    assert (gb["n_inlier"] > 200).any() and (gb["n_inlier"] < 50).any()      # pairs of one view pair and pairs of unrelated frames
    for p, pr in enumerate(pairs):
        ms = {k: m[k][p:p + 1] for k in ("idx", "dist")}
        g1 = host_of(solver.solve(views["S"], views["S"], [pr], ms, [depths[p]], KITTI_K, Tcw_query=Tcw[p:p + 1], out=filled(solver, 1, views["cap"]), **kw))
        for k in g1:
            assert np.array_equal(g1[k][0], gb[k][p]), (p, k)


def _solve_planted(ctx, d, solver, **kw):
    out = filled(solver, 1, d["n"])
    solver.solve(d["q"], d["t"], [(0, 0)], d["m"], [kw.pop("depth", d["depth_t"])], KITTI_K, out=out, **kw)
    return host_of(out)


def _assert_no_model(g, nq, bits):
    assert g["info"][0, 3] == bits and g["n_inlier"][0] == 0
    assert np.array_equal(g["T"][0], np.eye(4, dtype=np.float32)) and np.array_equal(g["Rt"][0], [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0])
    assert (g["inlier"][0, :nq] == 0).all() and (g["inlier"][0, nq:] == FILL).all()


def test_edge_cases(ctx):
    d = planted(21, n=300)
    solver = capi.PnpSolver(ctx, 1, d["n"], 500)
    for nc in range(4):                                  # 0..3 correspondences: FEW_POINTS, identity, no RANSAC iteration
        idx = torch.full_like(d["m"]["idx"], -1)
        idx[0, :nc, 0] = torch.arange(nc, dtype=torch.int32, device=DEV)
        g = _solve_planted(ctx, dict(d, m={"idx": idx, "dist": d["m"]["dist"]}), solver)
        assert g["n_corr"][0] == nc and list(g["info"][0, :3]) == [0, -1, 0]
        _assert_no_model(g, d["n"], capi.PNP_STATUS_FEW_POINTS)
    g = _solve_planted(ctx, d, solver, depth=torch.zeros_like(d["depth_t"]))          # all depths zero
    assert g["n_corr"][0] == 0
    _assert_no_model(g, d["n"], capi.PNP_STATUS_FEW_POINTS)
    for bad in (-1, d["n"] + 1):                         # counts outside 0 .. cap
        g = _solve_planted(ctx, dict(d, q=dict(d["q"], count=torch.tensor([bad], dtype=torch.int32, device=DEV))), solver)
        assert g["info"][0, 3] == capi.PNP_STATUS_QUERY_COUNT | capi.PNP_STATUS_FEW_POINTS and g["n_corr"][0] == 0
        assert (g["inlier"][0] == FILL).all()            # the query row is not written
        g = _solve_planted(ctx, dict(d, t=dict(d["t"], count=torch.tensor([bad], dtype=torch.int32, device=DEV))), solver)
        _assert_no_model(g, d["n"], capi.PNP_STATUS_TRAIN_COUNT | capi.PNP_STATUS_FEW_POINTS)
    # a depth plane given as a crop of a larger tensor or as a transposed view equals the contiguous plane
    ref = _solve_planted(ctx, d, solver, max_depth=30.0)
    assert ref["info"][0, 3] == 0 and ref["n_inlier"][0] > 100
    big = torch.zeros((H + 10, W + 20), dtype=torch.float32, device=DEV)
    big[5:5 + H, 7:7 + W] = d["depth_t"]
    tr = d["depth_t"].t().contiguous().t()
    for view in (big[5:5 + H, 7:7 + W], tr):
        g = _solve_planted(ctx, d, solver, max_depth=30.0, depth=view)
        for k in g:
            assert np.array_equal(g[k], ref[k]), k


def test_cuda_graph_replay_equals_eager(ctx, views):
    nv = len(views["vs"])
    pairs = [(2 * i, 2 * i + 1) for i in range(nv)]
    m = match(ctx, views["S"], pairs, 2)
    m2 = match(ctx, views["S"], [(2 * i + 1, 2 * i) for i in range(nv)], 2)
    solver = capi.PnpSolver(ctx, 8, views["cap"], 500)
    Tcw = np.stack([v["Tcw_a"] for v in views["vs"]]).astype(np.float32)
    kw = dict(Tcw_query=Tcw, ratio=0.8, thr=2.0)
    depths = [views["depths"][q].clone() for q, _ in pairs]
    idx, dist = m["idx"].clone(), m["dist"].clone()
    eager = host_of(solver.solve(views["S"], views["S"], pairs, m, depths, KITTI_K, out=filled(solver, nv, views["cap"]), **kw))
    out = filled(solver, nv, views["cap"])
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        solver.solve(views["S"], views["S"], pairs, {"idx": idx, "dist": dist}, depths, KITTI_K, out=out, **kw)     # warm-up on the side stream
        with torch.cuda.graph(g, stream=s):
            solver.solve(views["S"], views["S"], pairs, {"idx": idx, "dist": dist}, depths, KITTI_K, out=out, **kw)
    torch.cuda.current_stream(DEV).wait_stream(s)
    for t in out.values():
        t.fill_(FILL)
    g.replay()
    torch.cuda.synchronize()
    got = host_of(out)
    for k in eager:
        assert np.array_equal(got[k], eager[k]), k
    # a replay reads the device inputs as they are at replay time (here: every depth doubled), with the captured call's host parameters
    # (not those of a later eager call with other pairs and settings)
    solver.solve(views["S"], views["S"], [(q + 1, q) for q, _ in pairs], m2, [views["depths"][q + 1] for q, _ in pairs], KITTI_K, ratio=0.7, thr=0.4)
    for d in depths:
        d.mul_(2.0)
    eager2 = host_of(solver.solve(views["S"], views["S"], pairs, {"idx": idx, "dist": dist}, depths, KITTI_K, out=filled(solver, nv, views["cap"]), **kw))
    for t in out.values():
        t.fill_(FILL)
    g.replay()
    torch.cuda.synchronize()
    got = host_of(out)
    for k in eager2:
        assert np.array_equal(got[k], eager2[k]), k
    assert not np.array_equal(eager2["T"], eager["T"])


def test_python_refusals(ctx, views):
    S, cap = views["S"], views["cap"]
    pairs = [(0, 1)]
    m = match(ctx, S, pairs, 2)
    m1 = match(ctx, S, pairs, 1)
    solver = capi.PnpSolver(ctx, 2, cap, 500)
    d = [views["depths"][0]]
    ok = dict(query=S, train=S, pairs=pairs, matches=m, depths=d, K=KITTI_K)
    bad = [dict(pairs=[]), dict(pairs=[(0, 1)] * 3), dict(pairs=[(0, 99)]), dict(depths=[d[0].double()]), dict(depths=[d[0].cpu()]),
           dict(depths=[d[0], d[0]]), dict(depths=[d[0][None]]), dict(matches={"idx": m["idx"].long(), "dist": m["dist"]}),
           dict(matches={"idx": m["idx"][:, :100], "dist": m["dist"]}), dict(matches=m1, ratio=0.8), dict(ratio=float("nan")),
           dict(max_depth=float("nan")), dict(iters=0), dict(iters=501), dict(thr=0.0), dict(thr=float("nan")), dict(conf=1.0), dict(conf=0.0),
           dict(K=np.zeros(3)), dict(Tcw_query=np.eye(3)), dict(query=dict(S, x=S["x"].cpu())), dict(train=dict(S, count=S["count"].long())),
           dict(out=dict(solver.empty_outputs(1), T=torch.empty((1, 4, 4), dtype=torch.float64, device=DEV)))]
    for b in bad:
        with pytest.raises(ValueError):
            solver.solve(**dict(ok, **b))
    small = capi.PnpSolver(ctx, 1, 100, 10)
    with pytest.raises(ValueError):
        small.solve(**ok)                                 # query capacity above the solver's cap


def test_c_refusals_write_nothing(ctx, views):
    S, cap = views["S"], views["cap"]
    pairs = [(0, 1)]
    m = match(ctx, S, pairs, 2)
    solver = capi.PnpSolver(ctx, 2, cap, 500)
    out = filled(solver, 2, cap)
    L = ctx.L
    host_buf = np.zeros(1 << 20, np.int32)

    def call(P=1, pr=((0, 1),), qs=None, ts=None, idx=None, dist=None, plane=None, wh=(W, H), opts=None, o=None, K=KITTI_K):
        qs = qs or capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), S["x"].shape[0], cap)
        ts = ts or capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), S["x"].shape[0], cap)
        plane = plane or capi._dev_plane(ctx, "depth", views["depths"][0], W, H)
        planes = (capi.DevPlane * max(P, 1))(*([plane] * max(P, 1)))
        pa = np.ascontiguousarray(np.array(list(pr) * max(P, 1), np.int32)[:max(P, 1)])
        whs = np.ascontiguousarray(np.tile(np.array(wh, np.int32), (max(P, 1), 1)))
        Ks = np.ascontiguousarray(np.tile(np.asarray(K, np.float32), (max(P, 1), 1)))
        o = o or capi.PnpOut(*[out[k].data_ptr() for k in ("T", "Rt", "inlier", "n_corr", "n_inlier", "info")])
        opts = opts or capi.PnpMatchOpts(2, 0.8, 0.0, 500, 0.4, 0.98)
        return L.vdo_pnp_match_batch_dev(solver.h_, C.c_int(P), pa.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(qs), C.byref(ts),
                                         C.c_void_p(m["idx"].data_ptr() if idx is None else idx), C.c_void_p(m["dist"].data_ptr() if dist is None else dist),
                                         planes, whs.ctypes.data_as(C.POINTER(C.c_int32)), Ks.ctypes.data_as(C.POINTER(C.c_float)), None, None,
                                         C.byref(opts), C.byref(o), C.c_uint64(0))

    def opt(**kw):
        base = dict(k=2, ratio=0.8, max_depth=0.0, iters=500, thr=0.4, conf=0.98)
        base.update(kw)
        return capi.PnpMatchOpts(base["k"], base["ratio"], base["max_depth"], base["iters"], base["thr"], base["conf"])

    def o_with(**kw):
        ptr = {k: out[v].data_ptr() for k, v in (("T_dev", "T"), ("Rt_dev", "Rt"), ("inlier_dev", "inlier"), ("n_corr_dev", "n_corr"),
                                                  ("n_inlier_dev", "n_inlier"), ("info_dev", "info"))}
        ptr.update(kw)
        return capi.PnpOut(**ptr)

    nf = S["x"].shape[0]
    dp = capi._dev_plane(ctx, "depth", views["depths"][0], W, H)
    bad = {
        "P = 0": dict(P=0), "P = 3 > max_pairs": dict(P=3), "frame out of range": dict(pr=((0, nf),)), "negative frame": dict(pr=((-1, 0),)),
        "query cap above the solver's": dict(qs=capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), S["count"].data_ptr(), nf, cap + 1)),
        "iters 0": dict(opts=opt(iters=0)), "iters above max_iters": dict(opts=opt(iters=501)), "k = 3": dict(opts=opt(k=3)),
        "ratio with k = 1": dict(opts=opt(k=1)), "thr NaN": dict(opts=opt(thr=float("nan"))), "thr 0": dict(opts=opt(thr=0.0)),
        "conf 0": dict(opts=opt(conf=0.0)), "conf 1": dict(opts=opt(conf=1.0)), "ratio NaN": dict(opts=opt(ratio=float("nan"))),
        "max_depth NaN": dict(opts=opt(max_depth=float("nan"))),
        "depth u8": dict(plane=capi.DevPlane(dp.data_dev, capi.VDO_DT_U8, 1, dp.stride_y, dp.stride_x, 0, 1)),
        "depth 2 channels": dict(plane=capi.DevPlane(dp.data_dev, capi.VDO_DT_F32, 2, dp.stride_y, dp.stride_x, 0, 1)),
        "depth NULL": dict(plane=capi.DevPlane(None, capi.VDO_DT_F32, 1, dp.stride_y, dp.stride_x, 0, 1)),
        "depth host memory": dict(plane=capi.DevPlane(host_buf.ctypes.data, capi.VDO_DT_F32, 1, W, 1, 0, 1)),
        "depth misaligned": dict(plane=capi.DevPlane(dp.data_dev + 2, capi.VDO_DT_F32, 1, dp.stride_y, dp.stride_x, 0, 1)),
        "depth width 0": dict(wh=(0, H)),
        "idx NULL": dict(idx=0), "idx host memory": dict(idx=host_buf.ctypes.data), "idx misaligned": dict(idx=m["idx"].data_ptr() + 1),
        "dist NULL": dict(dist=0),
        "query.x NULL": dict(qs=capi.OrbDescSet(None, None, S["y"].data_ptr(), S["count"].data_ptr(), nf, cap)),
        "train.count host memory": dict(ts=capi.OrbDescSet(None, S["x"].data_ptr(), S["y"].data_ptr(), host_buf.ctypes.data, nf, cap)),
        "out.T NULL": dict(o=o_with(T_dev=None)), "out.info host memory": dict(o=o_with(info_dev=host_buf.ctypes.data)),
        "out.Rt misaligned": dict(o=o_with(Rt_dev=out["Rt"].data_ptr() + 4)), "out.inlier NULL": dict(o=o_with(inlier_dev=None)),
    }
    torch.cuda.synchronize()
    for what, kw in bad.items():
        assert call(**kw) == ERR_ARG, what
        assert L.vdo_last_error(ctx.h).decode().startswith("vdo_pnp_match_batch_dev"), what
    torch.cuda.synchronize()
    for k, t in out.items():
        assert (t == FILL).all(), k                       # nothing was written
    assert call() == 0                                   # the same arguments otherwise run
    torch.cuda.synchronize()
    assert (out["n_corr"][:1] > 0).all() and (out["n_corr"][1:] == FILL).all()
    with pytest.raises(capi.VdoError):
        capi.PnpSolver(ctx, 65, cap, 500)
    with pytest.raises(capi.VdoError):
        capi.PnpSolver(ctx, 1, cap, 4097)
    assert solver.info()["max_pairs"] == 2 and solver.info()["device_bytes"] > 0
