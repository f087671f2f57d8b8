"""The camera across frame pairs on the device (capi.CameraMotion: vdo_stat_build_batch_dev, vdo_cam_track_batch_dev,
vdo_stat_renew_batch_dev, and capi.sample_keys_dev).

Two references, both compared bit for bit:
  * the tracker: capi.Tracker.track over whole sequences, fed nothing but the frames.  The device chain extract -> build -> cam track ->
    update_mask -> track -> static renew -> object renew runs on the tracker's written-back metric depth and the original masks, with no
    tracker pose fed in, and must reproduce its camera, background and object state frame after frame;
  * the host route per call: Frame.filter_static + get3d_camera, init_model_batch + pose_opt_flow2, and renew_frame_info's static part."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from tests.object_motion_reference import inv4
from tests.test_object_renew_gpu import assert_set_equals_tracker as assert_obj_set_equals_tracker
from tests.test_object_renew_gpu import assert_track_equals_tracker
from vdo_slam_b200 import capi
from vdo_slam_b200.synth import KITTI_K, make_sequence_frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ERR_ARG = -2
FILL = 7
M = 8
OMD_K = np.array([618.3587036132812, 618.5924072265625, 328.9866333007812, 237.7507629394531], np.float32)
OMD = dict(width=640, height=480, fx=float(OMD_K[0]), fy=float(OMD_K[1]), cx=float(OMD_K[2]), cy=float(OMD_K[3]), depth_factor=256.0, th_depth_bg=40.0,
           th_depth_obj=25.0, max_track_bg=1200, max_track_obj=800, sf_mg_thres=0.02, sf_ds_thres=0.99, n_features=3000, is_kitti=0, dataset=1)
CONFIGS = {"kitti_I": dict(W=1242, H=375, K=KITTI_K, kw={}, shrink=(25, 50), sf=(0.12, 0.3), nf=2500),
           "omd_II": dict(W=640, H=480, K=OMD_K, kw=dict(OMD, use_sample_feature=1, sample_seed=7), shrink=(0, 0), sf=(0.02, 0.99), nf=3000)}
STAT_COLS = ("x", "y", "depth", "cx", "cy", "flow", "inlier_id", "point")


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


@functools.lru_cache(maxsize=None)
def frames(name, seed, n=12, n_obj=4):
    """test_object_renew_gpu's events at the configuration's size: object 2 parked, a one-frame dropout at frame 5, object 4 entering at
    frame 6, object 1 failing the gate at frame 8"""
    c = CONFIGS[name]
    mk = lambda t: make_sequence_frame(t, seed=seed, width=c["W"], height=c["H"], n_obj=n_obj, parked=(2,), K=c["K"])
    m5 = mk(5)["mask"]
    drop = 1 if (m5 == 1).sum() > (m5 == 3).sum() else 3
    rng = np.random.default_rng(seed + 77)
    out = []
    for t in range(n):
        f = mk(t)
        mask, flow = f["mask"].copy(), f["flow"].copy()
        if t == 5:
            mask[mask == drop] = 0
        if t < 6:
            mask[mask == 4] = 0
        if t == 8:
            sel = f["mask"] == 1
            flow[sel] += rng.normal(0.0, 6.0, (int(sel.sum()), 2)).astype(np.float32)
        out.append(dict(gray=f["gray"], depth_raw=f["depth_raw"], flow=flow, mask=mask.astype(np.int32), ids=list(range(1, n_obj + 1))))
    return out


STAT_F = ("Tcw", "mVelocity", "mvStatKeysTmp", "mvCorres", "mvFlowNext", "mvStatDepthTmp", "mvStat3DPointTmp")
OBJ_F = ("mvObjKeys", "mvObjDepth", "mvObjCorres", "mvObjFlowNext", "mvObj3DPoint", "vObjMod", "vObjCentre3D")
OBJ_I = ("vSemObjLabel", "vObjLabel", "nDynInlierID", "nModLabel", "nSemPosition", "bObjStat", "max_id")


@functools.lru_cache(maxsize=None)
def tracked(ctx, name, seed):
    c = CONFIGS[name]
    tr = capi.Tracker(ctx, local_batch=0, **c["kw"])
    res = []
    for f in frames(name, seed):
        d, m = f["depth_raw"].copy(), f["mask"].copy()
        tr.track(f["gray"], d, f["flow"], m, f["ids"], writeback=True)
        res.append(dict(depth=d, mask=m, **{k: tr.get(k) for k in STAT_F + OBJ_F + OBJ_I + ("nStaInlierID", "TemperalMatch_subset")}))
    return res


def set_rows(S, p=0):
    n = int(S["count"][p])
    return {k: S[k][p, :n] for k in STAT_COLS}


def assert_stat_equals_tracker(S, ref, what):
    r = set_rows(S)
    assert np.array_equal(np.stack([r["x"], r["y"]], 1).reshape(-1), ref["mvStatKeysTmp"]), what
    assert np.array_equal(np.stack([r["cx"], r["cy"]], 1).reshape(-1), ref["mvCorres"]), what
    assert np.array_equal(r["flow"].reshape(-1), ref["mvFlowNext"]), what
    assert np.array_equal(r["depth"], ref["mvStatDepthTmp"]), what
    assert np.array_equal(r["point"].reshape(-1), ref["mvStat3DPointTmp"]), what
    if len(ref["nStaInlierID"]) or len(r["inlier_id"]) == 0:
        assert np.array_equal(r["inlier_id"], ref["nStaInlierID"]), what
    else:                                                     # the first frame: the tracker keeps no IDs, the build marks every row new
        assert (r["inlier_id"] == -1).all(), what
    assert np.array_equal(S["Tcw"][0].reshape(-1), ref["Tcw"]), what


def chain(ctx, name, seq, check):
    """the whole device step over the sequence (P = 1); check(t, set after frame t, cam of pair t - 1 or None, obj track, obj set)"""
    c = CONFIGS[name]
    W, H, K = c["W"], c["H"], c["K"]
    II = bool(c["kw"].get("use_sample_feature", 0))
    ex = capi.OrbExtractor(ctx, W, H, 1, n_features=c["nf"])
    cap = max(ex.info()["capacity"], capi.SAMPLE_KEYS, 1201)
    cam_est = capi.CameraMotion(ctx, 1, cap)
    obj_est = capi.ObjectMotion(ctx, 1, M, ((W + 3) // 4) * ((H + 3) // 4))
    depth = [tens(r["depth"]) for r in seq["ref"]]
    flow = [tens(f["flow"]) for f in seq["frames"]]
    mask = [tens(f["mask"]) for f in seq["frames"]]
    seeds = tens(np.array([7 + t for t in range(len(depth))], np.uint32).view(np.int32))

    def keys(t):
        orb = ex.extract([tens(seq["frames"][t]["gray"])], describe=False)
        return (capi.sample_keys_dev(ctx, seeds[t:t + 1], W, H) if II else orb), orb["count"]

    sets = [cam_est.empty_outputs(1) for _ in range(2)]
    S = sets[1]
    kset, oc = keys(0)
    cam_est.build(kset, [depth[0]], [flow[0]], [mask[0]], K, S, use_sample_feature=int(II), orb_count=oc)
    torch.cuda.synchronize()
    check(0, host_of(S), None, None, None)
    OS, prev = None, None
    for t in range(len(depth) - 1):
        cam = cam_est.track(S, K)
        obj_est.update_mask([depth[t]], [flow[t]], [mask[t]], [mask[t + 1]], samples=OS)
        o = obj_est.track([depth[t]], [flow[t]], [mask[t]], [depth[t + 1]], [mask[t + 1]], K, Tcw_last=S["Tcw"], Tcw_cur=cam["T"], prev=prev, samples=OS,
                          shrink=c["shrink"], sf_mg_thres=c["sf"][0], sf_ds_thres=c["sf"][1])
        kset, oc = keys(t + 1)
        S = cam_est.renew(S, cam, kset, [depth[t + 1]], [flow[t + 1]], [mask[t + 1]], K, use_sample_feature=int(II), orb_count=oc, out=sets[t % 2])
        OS = obj_est.renew(o, [depth[t + 1]], [flow[t + 1]], [mask[t + 1]], K, Tcw_cur=cam["T"])
        prev = o
        torch.cuda.synchronize()
        check(t + 1, host_of(S), host_of(cam), host_of(o), host_of(OS))


# ------------------------------------------------------------------------------------------------ 1. the whole step equals the tracker
@pytest.mark.parametrize("name,seed", [("kitti_I", 0), ("omd_II", 3)])
def test_sequence_equals_the_tracker(ctx, name, seed):
    seq = dict(frames=frames(name, seed), ref=tracked(ctx, name, seed))
    seen = dict(mm=0, carried=0, topped=0, rejected=0)

    def check(t, S, cam, o, OS):
        ref = seq["ref"][t]
        what = f"{name} seed {seed} frame {t}"
        assert_stat_equals_tracker(S, ref, what)
        assert S["status"][0] == 0, what
        if cam is None:
            return
        assert np.array_equal(cam["T"][0].reshape(-1), ref["Tcw"]), what
        assert np.array_equal(cam["velocity"][0].reshape(-1), ref["mVelocity"]), what
        assert np.array_equal(S["velocity"][0].reshape(-1), ref["mVelocity"]), what
        n = int(cam["info"][0, 0])
        chosen = np.nonzero(cam["flags"][0, :n] & 1)[0]
        sub = np.where(cam["flags"][0, chosen] & 4, chosen, -1)
        assert np.array_equal(sub, ref["TemperalMatch_subset"]), what
        assert_track_equals_tracker(o, ref, what)
        assert_obj_set_equals_tracker(OS, ref, what)
        seen["mm"] += int(cam["status"][0] & capi.CAM_USED_MM != 0)
        seen["carried"] += int((set_rows(S)["inlier_id"] >= 0).any())
        seen["topped"] += int((set_rows(S)["inlier_id"] == -1).any())
        seen["rejected"] += int((sub == -1).any())

    chain(ctx, name, seq, check)
    assert seen["carried"] >= 10 and seen["topped"] >= 10 and seen["mm"] >= 1, seen


# ------------------------------------------------------------------------------------------------ 2. per call against the host route
def pair(name, seed, t):
    c = CONFIGS[name]
    fs = [make_sequence_frame(t + k, seed=seed, width=c["W"], height=c["H"], n_obj=3, K=c["K"]) for k in (0, 1)]
    dep = lambda f: np.where(f["depth_raw"] < 0, np.float32(0), np.float32(387.5744) / (f["depth_raw"] / np.float32(256.0))).astype(np.float32)
    return [dict(d=dep(f), f=f["flow"], m=f["mask"].astype(np.int32), gray=f["gray"]) for f in fs]


def layout(a, kind, how):
    if kind == "flow" and how == "chw":
        return tens(np.ascontiguousarray(a.transpose(2, 0, 1)))
    if how == "strided":
        big = np.zeros((a.shape[0] + 3, a.shape[1] + 5) + a.shape[2:], a.dtype)
        big[1:1 + a.shape[0], 2:2 + a.shape[1]] = a
        return tens(big)[1:1 + a.shape[0], 2:2 + a.shape[1]]
    return tens(a)


def host_build(ctx, c, fr0, kx, ky, th=40.0):
    fr = capi.Frame(ctx, c["W"], c["H"])
    fr.upload(depth=fr0["d"], flow=fr0["f"], mask=fr0["m"])
    idx, cx, cy, fu, fv, d = fr.filter_static(kx, ky, th)
    fr.close()
    fx, fy, ccx, ccy = (float(v) for v in c["K"])
    X = np.stack([(kx[idx] - np.float32(ccx)) * d * (np.float32(1) / np.float32(fx)), (ky[idx] - np.float32(ccy)) * d * (np.float32(1) / np.float32(fy)), d], 1)
    return dict(x=kx[idx], y=ky[idx], cx=cx, cy=cy, flow=np.stack([fu, fv], 1), depth=d, point=X.astype(np.float32))


@pytest.mark.parametrize("max_bg", [0, 50, 1200, 100000])
@pytest.mark.parametrize("how", ["plain", "i64_chw", "strided"])
def test_calls_equal_the_host_route(ctx, max_bg, how):
    """build (option I, against Frame.filter_static + get3d_camera), cam track (against init_model_batch with the motion model +
    pose_opt_flow2 mode 0) and renew (against renew_frame_info's static part) on three KITTI pairs"""
    c = CONFIGS["kitti_I"]
    W, H, K = c["W"], c["H"], c["K"]
    ins = [pair("kitti_I", s, t) for s, t in [(0, 2), (1, 4), (3, 1)]]
    P = len(ins)
    ex = capi.OrbExtractor(ctx, W, H, P)
    cap = max(ex.info()["capacity"], 1201) if max_bg < 100000 else 100001
    est = capi.CameraMotion(ctx, P, cap)
    mdt = np.int64 if how == "i64_chw" else np.int32
    fl = "chw" if how == "i64_chw" else how
    pl = lambda k, kind, i: [layout(x[i][k].astype(mdt) if kind == "mask" else x[i][k], kind, fl if kind == "flow" else ("strided" if how == "strided" else "plain"))
                             for x in ins]
    k0 = ex.extract([tens(x[0]["gray"]) for x in ins], describe=False)
    k0h = host_of({k: k0[k] for k in ("x", "y", "count")})
    S = filled(est.empty_outputs(P))
    S["count"].fill_(-1)
    est.build(k0, pl("d", "depth", 0), pl("f", "flow", 0), pl("m", "mask", 0), K, S)
    # a velocity for the motion model
    vel = np.eye(4, dtype=np.float32); vel[0, 3], vel[2, 3] = 0.01, -0.8
    S["velocity"].copy_(tens(np.stack([vel] * P))); S["has_velocity"].fill_(1)
    cam = est.track(S, K)
    k1 = ex.extract([tens(x[1]["gray"]) for x in ins], describe=False)
    k1h = host_of({k: k1[k] for k in ("x", "y", "count")})
    S2 = filled(est.empty_outputs(P))
    est.renew(S, cam, k1, pl("d", "depth", 1), pl("f", "flow", 1), pl("m", "mask", 1), K, max_track_bg=max_bg, out=S2)
    torch.cuda.synchronize()
    Sh, ch, S2h = host_of(S), host_of(cam), host_of(S2)
    for p, x in enumerate(ins):
        n0 = int(k0h["count"][p])
        b = host_build(ctx, c, x[0], k0h["x"][p, :n0], k0h["y"][p, :n0])
        r = set_rows(Sh, p)
        assert len(r["x"]) == len(b["x"]) > 100
        for k in ("x", "y", "cx", "cy", "flow", "depth", "point"):
            assert np.array_equal(r[k], b[k]), (p, k)
        assert (r["inlier_id"] == -1).all() and Sh["status"][p] == 0
        # cam track against the host route on the same rows
        n = len(r["x"])
        T0 = np.eye(4, dtype=np.float32)
        obj = np.zeros((n, 3), np.float32)
        fxk, fyk, cxk, cyk = (np.float32(v) for v in K)
        xc, yc = (r["x"] - cxk) * r["depth"] * (np.float32(1) / fxk), (r["y"] - cyk) * r["depth"] * (np.float32(1) / fyk)
        obj[:, 0], obj[:, 1], obj[:, 2] = xc, yc, r["depth"]                         # Tcw = I: the world point is the camera point
        im = capi.init_model_batch(ctx, [dict(obj=obj, img=np.stack([r["cx"], r["cy"]], 1), T_mm=vel @ T0)], K)[0]
        assert np.array_equal(ch["T_init"][p], im["T"]) and ch["info"][p, 4] == len(im["sub"])
        sub = im["sub"]
        lm = capi.pose_opt_flow2(ctx, [dict(pts=np.stack([r["x"], r["y"]], 1)[sub], depth=r["depth"][sub], flow=r["flow"][sub], K=K, Tcw_last=T0,
                                            T_init=im["T"])], quirk=1, modes=[0])[0]
        assert np.array_equal(ch["T"][p], lm["T"]), p
        flags = ch["flags"][p, :n]
        assert np.array_equal(np.nonzero(flags & 1)[0], sub) and np.array_equal(np.nonzero(flags & 2)[0], sub[lm["inlier"]])
        key = np.stack([r["cx"], r["cy"]], 1).copy()
        key[sub[lm["inlier"]]] = (np.stack([r["x"], r["y"]], 1)[sub[lm["inlier"]]].astype(np.float64) + lm["flow"][lm["inlier"]]).astype(np.float32)
        assert np.array_equal(ch["key"][p, :n], key)
        # renew against renew_frame_info's static part
        fr = capi.Frame(ctx, W, H)
        fr.upload(depth=x[1]["d"], flow=x[1]["f"], mask=x[1]["m"])
        tm = np.where(flags[sub] & 4, sub, -1)
        n1 = int(k1h["count"][p])
        st, _ = capi.renew_frame_info(fr, tm, key, np.stack([k1h["x"][p, :n1], k1h["y"][p, :n1]], 1), max_bg, [], [], [], [], np.zeros((0, 2)), [],
                                      np.zeros((0, 2)), [], [], np.zeros((0, 2)), np.zeros((0, 2)), 0, np.asarray(K, np.float32), inv4(ch["T"][p]))
        fr.close()
        r2 = set_rows(S2h, p)
        assert S2h["count"][p] == len(st["keys"]) <= max_bg + 1, (p, S2h["count"][p], len(st["keys"]))
        for got, want in ((np.stack([r2["x"], r2["y"]], 1), st["keys"]), (np.stack([r2["cx"], r2["cy"]], 1), st["corres"]), (r2["flow"], st["flow"]),
                          (r2["inlier_id"], st["inlier_id"]), (r2["depth"], st["depth"]), (r2["point"], st["p3d"])):
            assert np.array_equal(got, want), (p, max_bg)
        assert (S2h["x"][p, S2h["count"][p]:] == FILL).all()
        assert np.array_equal(S2h["Tcw"][p], ch["T"][p]) and np.array_equal(S2h["velocity"][p], ch["velocity"][p]) and S2h["has_velocity"][p] == 1
        if max_bg == 0:
            assert S2h["count"][p] == 1                                               # the push comes before the '>' test
        if max_bg == 100000:
            assert (r2["inlier_id"] == -1).sum() > 0


# ------------------------------------------------------------------------------------------------ 3. boundaries
def test_few_rows_and_the_first_pair(ctx):
    """a set of 3 rows (no RANSAC: the motion model, which is Tcw itself on the first pair, is chosen and the LM runs on 3 rows) and of 2
    rows (no LM: T = T_init), against the host route; the observations are the keys, so every row is a motion-model inlier"""
    K = KITTI_K
    est = capi.CameraMotion(ctx, 2, 64)
    S = est.empty_outputs(2)
    rng = np.random.default_rng(4)
    for p, n in enumerate((3, 2)):
        x, y = rng.uniform(100, 900, n).astype(np.float32), rng.uniform(50, 300, n).astype(np.float32)
        d = rng.uniform(5, 30, n).astype(np.float32)
        f = rng.uniform(-3, 3, (n, 2)).astype(np.float32)
        S["x"][p, :n] = tens(x); S["y"][p, :n] = tens(y); S["depth"][p, :n] = tens(d); S["flow"][p, :n] = tens(f)
        S["cx"][p, :n] = tens(x); S["cy"][p, :n] = tens(y); S["count"][p] = n
    S["Tcw"].copy_(torch.eye(4, device=DEV).expand(2, 4, 4)); S["has_velocity"].fill_(0)
    cam = host_of(est.track(S, K))
    Sh = host_of(S)
    for p, n in enumerate((3, 2)):
        r = set_rows(Sh, p)
        obj = np.stack([(r["x"] - K[2]) * r["depth"] * (np.float32(1) / K[0]), (r["y"] - K[3]) * r["depth"] * (np.float32(1) / K[1]), r["depth"]], 1)
        im = capi.init_model_batch(ctx, [dict(obj=obj, img=np.stack([r["cx"], r["cy"]], 1), T_mm=np.eye(4, dtype=np.float32))], K)[0]
        assert cam["status"][p] & capi.CAM_FEW_POINTS and cam["status"][p] & capi.CAM_USED_MM
        assert np.array_equal(cam["T_init"][p], im["T"]) and len(im["sub"]) == n
        if n == 3:
            lm = capi.pose_opt_flow2(ctx, [dict(pts=np.stack([r["x"], r["y"]], 1), depth=r["depth"], flow=r["flow"], K=K, Tcw_last=np.eye(4, dtype=np.float32),
                                                T_init=im["T"])], quirk=1, modes=[0])[0]
            assert np.array_equal(cam["T"][p], lm["T"]) and cam["stats"][p, 0] >= 0
        else:
            assert np.array_equal(cam["T"][p], im["T"]) and cam["stats"][p, 0] == -1 and (cam["flags"][p, :n] & 4).all()


def test_top_up_distance_boundary_and_edges(ctx):
    """one carried key at (100.5, 100.5); top-up keys at float distances just under, at and just over 1 px, and keys on the x <= 0 and
    x >= W edges: the renewal against renew_frame_info"""
    W, H = 256, 128
    K = np.array([200.0, 200.0, 128.0, 64.0], np.float32)
    d = np.full((H, W), 10.0, np.float32)
    f = np.empty((H, W, 2), np.float32); f[..., 0], f[..., 1] = 0.5, 0.25
    m = np.zeros((H, W), np.int32)
    est = capi.CameraMotion(ctx, 1, 64)
    last = est.empty_outputs(1)
    last["count"].fill_(1); last["Tcw"].copy_(torch.eye(4, device=DEV)[None])
    cam = filled(est.empty_outputs(1, set=False))
    cam["status"].fill_(0); cam["flags"].fill_(5); cam["T"].copy_(torch.eye(4, device=DEV)[None]); cam["velocity"].copy_(torch.eye(4, device=DEV)[None])
    cam["key"][0, 0] = tens(np.array([100.5, 100.5], np.float32))
    under = np.nextafter(np.float32(101.5), np.float32(0))
    kx = np.array([under, 101.5, np.nextafter(np.float32(101.5), np.float32(200)), 0.0, 0.5, W - 0.5, W - 1.0, 50.0], np.float32)
    ky = np.array([100.5, 100.5, 100.5, 20.0, 20.0, 20.0, 20.0, 30.0], np.float32)
    keys = dict(x=tens(kx[None]), y=tens(ky[None]), count=tens(np.array([len(kx)], np.int32)))
    out = est.renew(last, cam, keys, [tens(d)], [tens(f)], [tens(m)], K, max_track_bg=20)
    torch.cuda.synchronize()
    fr = capi.Frame(ctx, W, H)
    fr.upload(depth=d, flow=f, mask=m)
    st, _ = capi.renew_frame_info(fr, [0], np.array([[100.5, 100.5]], np.float32), np.stack([kx, ky], 1), 20, [], [], [], [], np.zeros((0, 2)), [],
                                  np.zeros((0, 2)), [], [], np.zeros((0, 2)), np.zeros((0, 2)), 0, K, np.eye(4, dtype=np.float32))
    fr.close()
    o = host_of(out)
    r = set_rows(o)
    assert np.array_equal(np.stack([r["x"], r["y"]], 1), st["keys"]) and np.array_equal(r["inlier_id"], st["inlier_id"])
    top = r["x"][1:].tolist()
    assert 101.5 in top and under not in top and 0.0 not in top and 0.5 not in top and W - 0.5 not in top and W - 1.0 in top


def test_option_II_zero_orb_keypoints_gives_an_empty_set(ctx):
    W, H = 640, 480
    fr0 = make_sequence_frame(0, seed=1, width=W, height=H, n_obj=2, K=OMD_K)
    est = capi.CameraMotion(ctx, 1, 3000)
    keys = capi.sample_keys_dev(ctx, tens(np.array([5], np.int32)), W, H)
    d = np.full((H, W), 10.0, np.float32)
    for oc, want_rows in ((0, False), (1, True)):
        S = est.empty_outputs(1)
        est.build(keys, [tens(d)], [tens(fr0["flow"])], [tens(fr0["mask"].astype(np.int32))], OMD_K, S, use_sample_feature=1,
                  orb_count=tens(np.array([oc], np.int32)))
        torch.cuda.synchronize()
        assert (int(S["count"][0]) > 0) == want_rows


def test_sample_keys_dev_equals_the_host_entry(ctx):
    seeds = np.array([0, 7, 2 ** 32 - 1], np.uint32)
    got = host_of(capi.sample_keys_dev(ctx, tens(seeds.view(np.int32)), 640, 480))
    kx, ky = capi.sample_keys(ctx, seeds.tolist(), 640, 480)[:2]
    assert np.array_equal(got["x"], np.asarray(kx).reshape(3, -1)) and np.array_equal(got["y"], np.asarray(ky).reshape(3, -1))
    assert (got["count"] == capi.SAMPLE_KEYS).all()


# ------------------------------------------------------------------------------------------------ 4. batches and graphs
def test_cuda_graph_of_the_step_equals_eager(ctx):
    """option II at OMD size: sample (device seeds) -> build -> cam track -> renew captured once per parity and replayed, equal to eager"""
    name, seed, n = "omd_II", 3, 7
    c = CONFIGS[name]
    W, H, K = c["W"], c["H"], c["K"]
    seq = frames(name, seed)[:n]
    ex = capi.OrbExtractor(ctx, W, H, 1, n_features=3000)
    est = capi.CameraMotion(ctx, 1, max(ex.info()["capacity"], 3000))
    dep = lambda f: tens(np.where(f["depth_raw"] < 0, 0, 387.5744 / (f["depth_raw"] / 256.0)).astype(np.float32))
    depth, flow, mask, gray = [dep(f) for f in seq], [tens(f["flow"]) for f in seq], [tens(f["mask"]) for f in seq], [tens(f["gray"]) for f in seq]
    seeds = [tens(np.array([7 + t], np.int32)) for t in range(n)]
    eager = []
    S = est.empty_outputs(1)
    est.build(capi.sample_keys_dev(ctx, seeds[0], W, H), [depth[0]], [flow[0]], [mask[0]], K, S, use_sample_feature=1,
              orb_count=ex.extract([gray[0]], describe=False)["count"])
    for t in range(n - 1):
        cam = est.track(S, K)
        kk = capi.sample_keys_dev(ctx, seeds[t + 1], W, H)
        S = est.renew(S, cam, kk, [depth[t + 1]], [flow[t + 1]], [mask[t + 1]], K, use_sample_feature=1,
                      orb_count=ex.extract([gray[t + 1]], describe=False)["count"])
        eager.append(({k: v.clone() for k, v in cam.items()}, {k: v.clone() for k, v in S.items()}))
    torch.cuda.synchronize()
    # static inputs, double-buffered sets
    dl, fl, ml, gl, dc, fc, mc, gc, sl, sc = (x.clone() for x in (depth[0], flow[0], mask[0], gray[0], depth[1], flow[1], mask[1], gray[1], seeds[0], seeds[1]))
    sets = [est.empty_outputs(1) for _ in range(2)]
    cams = [est.empty_outputs(1, set=False) for _ in range(2)]
    korb = [ex.empty_outputs(1, describe=False) for _ in range(2)]
    ks = [dict(x=torch.empty(1, 3000, device=DEV), y=torch.empty(1, 3000, device=DEV), count=torch.empty(1, dtype=torch.int32, device=DEV)) for _ in range(2)]
    graphs = []
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        for k in range(2):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                o0 = ex.extract([gl], describe=False, out=korb[0])
                capi.sample_keys_dev(ctx, sl, W, H, out=ks[0])
                est.build(ks[0], [dl], [fl], [ml], K, sets[1 - k], use_sample_feature=1, orb_count=o0["count"])
                cm = est.track(sets[1 - k], K, out=cams[k])
                o1 = ex.extract([gc], describe=False, out=korb[1])
                capi.sample_keys_dev(ctx, sc, W, H, out=ks[1])
                est.renew(sets[1 - k], cm, ks[1], [dc], [fc], [mc], K, use_sample_feature=1, orb_count=o1["count"], out=sets[k])
            graphs.append(g)
    torch.cuda.current_stream(DEV).wait_stream(side)
    sets[1]["count"].fill_(-1)
    for t in range(n - 1):
        dl.copy_(depth[t]); fl.copy_(flow[t]); ml.copy_(mask[t]); gl.copy_(gray[t]); sl.copy_(seeds[t])
        dc.copy_(depth[t + 1]); fc.copy_(flow[t + 1]); mc.copy_(mask[t + 1]); gc.copy_(gray[t + 1]); sc.copy_(seeds[t + 1])
        graphs[t % 2].replay()
        torch.cuda.synchronize()
        ec, es = eager[t]
        for k in ("T", "velocity", "T_init", "info", "status"):
            assert torch.equal(cams[t % 2][k], ec[k]), (t, k)
        cnt = int(es["count"][0])
        assert int(sets[t % 2]["count"][0]) == cnt
        for k in STAT_COLS:
            assert torch.equal(sets[t % 2][k][0, :cnt], es[k][0, :cnt]), (t, k)


def test_64_pairs_with_staggered_restarts(ctx):
    """64 pairs of mixed KITTI and OMD sizes; pair p restarts (count -1) at step p % 3: every step of every pair equals the pair alone"""
    P, steps = 64, 3
    sizes = [("kitti_I", 1242, 375, KITTI_K), ("omd", 640, 480, OMD_K)]
    est = capi.CameraMotion(ctx, P, 8192)
    solo = capi.CameraMotion(ctx, 1, 8192)
    dep = lambda f: tens(np.where(f["depth_raw"] < 0, 0, 387.5744 / (f["depth_raw"] / 256.0)).astype(np.float32))
    seqs, Ks, exs = [], [], {}
    for p in range(P):
        _, w, h, K = sizes[p % 2]
        fs = [make_sequence_frame(t + p % 3, seed=p % 5, width=w, height=h, n_obj=1 + p % 3, K=K) for t in range(steps + 1)]
        if (w, h) not in exs:
            exs[(w, h)] = capi.OrbExtractor(ctx, w, h, 1)
        kk = [exs[(w, h)].extract([tens(f["gray"])], describe=False) for f in fs]
        kk = [dict(x=torch.zeros(1, 8192, device=DEV).index_copy_(1, torch.arange(k["x"].shape[1], device=DEV), k["x"]),
                   y=torch.zeros(1, 8192, device=DEV).index_copy_(1, torch.arange(k["y"].shape[1], device=DEV), k["y"]), count=k["count"].clone()) for k in kk]
        seqs.append([dict(d=dep(f), f=tens(f["flow"]), m=tens(f["mask"].astype(np.int32)), k=k) for f, k in zip(fs, kk)])
        Ks.append(K)
    Kp = np.stack(Ks)
    cat = lambda t, key: dict(x=torch.cat([seqs[p][t]["k"]["x"] for p in range(P)]), y=torch.cat([seqs[p][t]["k"]["y"] for p in range(P)]),
                              count=torch.cat([seqs[p][t]["k"]["count"] for p in range(P)]))
    sets = [est.empty_outputs(P) for _ in range(2)]
    S = sets[1]
    solo_S = [None] * P
    for t in range(steps):
        for p in range(P):
            if p % 3 == t:
                S["count"][p] = -1
        pl = lambda k, i: [seqs[p][t + i][k] for p in range(P)]
        est.build(cat(t, "k"), pl("d", 0), pl("f", 0), pl("m", 0), Kp, S)
        cam = est.track(S, Kp)
        S = est.renew(S, cam, cat(t + 1, "k"), pl("d", 1), pl("f", 1), pl("m", 1), Kp, out=sets[t % 2])
        torch.cuda.synchronize()
        Sh, ch = host_of(S), host_of(cam)
        for p in range(P):
            q = seqs[p]
            if solo_S[p] is None or p % 3 == t:
                solo_S[p] = solo.empty_outputs(1)
            solo.build(q[t]["k"], [q[t]["d"]], [q[t]["f"]], [q[t]["m"]], Ks[p], solo_S[p])
            sc = solo.track(solo_S[p], Ks[p])
            ss = solo.renew(solo_S[p], sc, q[t + 1]["k"], [q[t + 1]["d"]], [q[t + 1]["f"]], [q[t + 1]["m"]], Ks[p])
            torch.cuda.synchronize()
            solo_S[p] = {k: v.clone() for k, v in ss.items()}
            sh, sch = host_of(ss), host_of(sc)
            for k in ("T", "velocity", "info", "status"):
                assert np.array_equal(ch[k][p], sch[k][0]), (t, p, k)
            assert Sh["count"][p] == sh["count"][0], (t, p)
            n = int(sh["count"][0])
            for k in STAT_COLS:
                assert np.array_equal(Sh[k][p, :n], sh[k][0, :n]), (t, p, k)


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_refusals_write_nothing(ctx):
    x = pair("kitti_I", 0, 0)
    c = CONFIGS["kitti_I"]
    ex = capi.OrbExtractor(ctx, c["W"], c["H"], 1)
    est = capi.CameraMotion(ctx, 2, 8192)
    k0 = ex.extract([tens(x[0]["gray"])], describe=False)
    d, f, m = tens(x[0]["d"]), tens(x[0]["f"]), tens(x[0]["m"])
    S = filled(est.empty_outputs(1))
    ok = dict(keys=k0, depths=[d], flows=[f], masks=[m], K=KITTI_K, set=S)
    bad = [dict(th_depth_bg=float("nan")), dict(use_sample_feature=2), dict(use_sample_feature=1), dict(masks=[m.float()]), dict(flows=[d]),
           dict(depths=[d, d], flows=[f, f], masks=[m, m]), dict(depths=[d, d, d], flows=[f, f, f], masks=[m, m, m]), dict(K=np.zeros(3)),
           dict(set=dict(S, point=S["point"][:, :, :2])), dict(keys=dict(k0, x=k0["x"].cpu()))]
    for b in bad:
        with pytest.raises(ValueError):
            est.build(**dict(ok, **b))
    S["count"].fill_(FILL)
    cam = filled(est.empty_outputs(1, set=False))
    for b in (dict(iters=0), dict(iters=501), dict(thr=0.0), dict(conf=1.0), dict(quirk=2), dict(out=dict(cam, key=cam["key"][:, :, :1]))):
        with pytest.raises(ValueError):
            est.track(S, KITTI_K, **dict(dict(out=cam), **b))
    out = filled(est.empty_outputs(1))
    for b in (dict(max_track_bg=-1), dict(max_track_bg=8192), dict(use_sample_feature=1), dict(cam=dict(cam, flags=cam["flags"].int()))):
        with pytest.raises(ValueError):
            est.renew(**dict(dict(last=S, cam=cam, keys=k0, depths_cur=[d], flows_cur=[f], masks_cur=[m], K=KITTI_K, out=out), **b))
    torch.cuda.synchronize()
    for dct in (S, cam, out):
        for k, t in dct.items():
            assert (t == FILL).all(), k
    # the C entries refuse what Python cannot pass, with their name in the error
    st = capi.StatFeatSet(*[S[k].data_ptr() for k in capi._SS_SET])
    ks = capi.OrbDescSet(None, k0["x"].data_ptr(), k0["y"].data_ptr(), k0["count"].data_ptr(), 1, int(k0["x"].shape[1]))
    one = lambda t, kind: (capi.DevPlane * 1)(capi._dev_plane(ctx, kind, t, c["W"], c["H"]))
    wh = np.array([[c["W"], c["H"]]], np.int32)
    Kp = np.ascontiguousarray(KITTI_K[None])
    opts = capi.StatOpts(40.0, 1200, 0, 0)
    host_buf = np.zeros(1 << 16, np.int32)
    st_bad = capi.StatFeatSet(*[host_buf.ctypes.data if k == "count" else S[k].data_ptr() for k in capi._SS_SET])
    for s_ in (None, st_bad):
        rc = ctx.L.vdo_stat_build_batch_dev(est.h_, C.c_int(1), C.byref(ks), one(d, "depth"), one(f, "flow"), one(m, "mask"), wh.ctypes.data_as(C.POINTER(C.c_int32)),
                                            Kp.ctypes.data_as(C.POINTER(C.c_float)), None, C.byref(opts), None if s_ is None else C.byref(s_), C.c_uint64(0))
        assert rc == ERR_ARG and ctx.L.vdo_last_error(ctx.h).decode().startswith("vdo_stat_build_batch_dev")
    torch.cuda.synchronize()
    for k, t in S.items():
        assert (t == FILL).all(), k
