#!/usr/bin/env python
"""bench_camera_track.py -- the camera step and the static half of RenewFrameInfo on the device (capi.CameraMotion) against the host route
they replace, and the whole per-frame step in one CUDA graph against the tracker.

Workload: config-3-shaped pairs (synth.make_sequence_frame, KITTI-shaped 1242x375, 3-5 moving objects, ORB 2500 features, option I,
MaxTrackPointBG 1200, ThDepthBG 40).  Pair p is frames (1, 2) of sequence p % V, entered with the set that building frame 0 and renewing
pair (0, 1) left.  For P in {1, 8, 32, 64} it prints one JSON line:
  build_ms, track_ms, renew_ms   one eager call each (median of CUDA events over --reps calls; build on sets whose count is reset to -1)
  host_ms        the host route, host clock: D2H of the set and the current keys, then per pair capi.init_model_batch (with the motion
                 model), capi.pose_opt_flow2 (mode 0), Frame.upload and capi.renew_frame_info (empty object part)
  equal_host     every pair's T and renewed set equal the host route's
  step_graph_ms  ORB extraction of the current frames, build, cam track, update_mask, object track, static and object renewal, captured
                 once and replayed (median over --reps replays)
  tracker_ms     capi.track_tensors_batch of P trackers (local_batch=0) on the same frames, host clock.  The tracker also keeps its map and
                 tracklets, which the graph does not, so the comparison is of the per-frame estimation only.
The GPU name and power limit are read in the same run.

  python bench_camera_track.py [--pairs 1,8,32,64] [--views 8] [--reps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_pnp_match import gpu_info  # noqa: E402
from tests.object_motion_reference import inv4  # noqa: E402

W, H, M = 1242, 375, 8


def mul4(A, B):
    """cv::Mat A * B of two 4x4 float32 matrices, summed left to right in float"""
    C = np.zeros((4, 4), np.float32)
    for i in range(4):
        for j in range(4):
            s = np.float32(A[i, 0] * B[0, j])
            for k in range(1, 4):
                s = np.float32(s + np.float32(A[i, k] * B[k, j]))
            C[i, j] = s
    return C


OBJ_CAP = ((W + 3) // 4) * ((H + 3) // 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    info = gpu_info()
    t_ = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    depth = lambda raw: np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
    V = a.views
    views = [[make_sequence_frame(t, seed=v, width=W, height=H, n_obj=3 + v % 3) for t in range(3)] for v in range(V)]
    K = KITTI_K

    def events(fn, reps):
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    for P in [int(s) for s in a.pairs.split(",")]:
        fr = [[views[p % V][t] for p in range(P)] for t in range(3)]
        gray = [t_(np.stack([f["gray"] for f in fr[t]])) for t in range(3)]
        dep = [[t_(depth(f["depth_raw"])) for f in fr[t]] for t in range(3)]
        flo = [[t_(f["flow"]) for f in fr[t]] for t in range(3)]
        msk = [[t_(f["mask"].astype(np.int32)) for f in fr[t]] for t in range(3)]
        ex = capi.OrbExtractor(ctx, W, H, P)
        cap = max(ex.info()["capacity"], 1201)
        est = capi.CameraMotion(ctx, P, cap)
        oest = capi.ObjectMotion(ctx, P, M, OBJ_CAP)
        keys = [ex.extract(gray[t], describe=False) for t in range(3)]
        S0 = est.empty_outputs(P)
        est.build(keys[0], dep[0], flo[0], msk[0], K, S0)
        S1 = est.renew(S0, est.track(S0, K), keys[1], dep[1], flo[1], msk[1], K)
        cam = est.track(S1, K)
        S2 = est.renew(S1, cam, keys[2], dep[2], flo[2], msk[2], K)
        torch.cuda.synchronize()
        Sb = est.empty_outputs(P)

        def build():
            Sb["count"].fill_(-1)
            est.build(keys[1], dep[1], flo[1], msk[1], K, Sb)
        for _ in range(a.warmup):
            build(); est.track(S1, K, out=cam); est.renew(S1, cam, keys[2], dep[2], flo[2], msk[2], K, out=S2)
        torch.cuda.synchronize()
        build_ms = events(build, a.reps)
        track_ms = events(lambda: est.track(S1, K, out=cam), a.reps)
        renew_ms = events(lambda: est.renew(S1, cam, keys[2], dep[2], flo[2], msk[2], K, out=S2), a.reps)

        # the host route on the same set
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        Sh = {k: v.cpu().numpy() for k, v in S1.items()}
        kh = {k: keys[2][k].cpu().numpy() for k in ("x", "y", "count")}
        planes = [(d.cpu().numpy(), f.cpu().numpy(), m.cpu().numpy()) for d, f, m in zip(dep[2], flo[2], msk[2])]
        host = []
        for p in range(P):
            n = int(Sh["count"][p])
            x, y, d, fl = Sh["x"][p, :n], Sh["y"][p, :n], Sh["depth"][p, :n], Sh["flow"][p, :n]
            Tl, vel = Sh["Tcw"][p], Sh["velocity"][p]
            xc, yc = (x - K[2]) * d * (np.float32(1) / K[0]), (y - K[3]) * d * (np.float32(1) / K[1])
            Td = Tl.astype(np.float64)
            obj = np.zeros((n, 3), np.float32)
            for r in range(3):                                     # Frame::UnprojectStereoStat as the tracker rounds it
                twl = np.float64(np.float32(-(Td[0, r] * Td[0, 3] + Td[1, r] * Td[1, 3] + Td[2, r] * Td[2, 3])))
                obj[:, r] = (Td[0, r] * xc.astype(np.float64) + Td[1, r] * yc.astype(np.float64) + Td[2, r] * d.astype(np.float64) + twl).astype(np.float32)
            im = capi.init_model_batch(ctx, [dict(obj=obj, img=np.stack([Sh["cx"][p, :n], Sh["cy"][p, :n]], 1),
                                                  T_mm=mul4(vel, Tl) if Sh["has_velocity"][p] else Tl)], K)[0]
            sub = im["sub"]
            T, keyc, tm = im["T"], np.stack([Sh["cx"][p, :n], Sh["cy"][p, :n]], 1).copy(), sub.copy()
            if len(sub) >= 3:
                lm = capi.pose_opt_flow2(ctx, [dict(pts=np.stack([x, y], 1)[sub], depth=d[sub], flow=fl[sub], K=K, Tcw_last=Tl, T_init=im["T"])],
                                         quirk=1, modes=[0])[0]
                T = lm["T"]
                keyc[sub[lm["inlier"]]] = (np.stack([x, y], 1)[sub[lm["inlier"]]].astype(np.float64) + lm["flow"][lm["inlier"]]).astype(np.float32)
                tm[~lm["inlier"]] = -1
            f = capi.Frame(ctx, W, H)
            f.upload(depth=planes[p][0], flow=planes[p][1], mask=planes[p][2])
            nk = int(kh["count"][p])
            st, _ = capi.renew_frame_info(f, tm, keyc, np.stack([kh["x"][p, :nk], kh["y"][p, :nk]], 1), 1200, [], [], [], [], np.zeros((0, 2)), [],
                                          np.zeros((0, 2)), [], [], np.zeros((0, 2)), np.zeros((0, 2)), 0, K, inv4(T))
            f.close()
            host.append((T, st))
        host_ms = (time.perf_counter() - h0) * 1e3
        ch, S2h = {k: v.cpu().numpy() for k, v in cam.items()}, {k: v.cpu().numpy() for k, v in S2.items()}
        equal = all(np.array_equal(ch["T"][p], host[p][0]) and int(S2h["count"][p]) == len(host[p][1]["keys"]) and
                    np.array_equal(np.stack([S2h["x"][p], S2h["y"][p]], 1)[:len(host[p][1]["keys"])], host[p][1]["keys"]) and
                    np.array_equal(S2h["point"][p, :len(host[p][1]["keys"])], host[p][1]["p3d"]) for p in range(P))

        # the whole step in one graph: static inputs for frames (1, 2), double-buffered sets
        g_gray, g_dl, g_fl, g_ml, g_dc, g_fc, g_mc = gray[2].clone(), [x.clone() for x in dep[1]], [x.clone() for x in flo[1]], \
            [x.clone() for x in msk[1]], [x.clone() for x in dep[2]], [x.clone() for x in flo[2]], [x.clone() for x in msk[2]]
        pristine = [x.clone() for x in msk[2]]
        kout = ex.empty_outputs(P, describe=False)
        sets = [est.empty_outputs(P) for _ in range(2)]
        cams = [est.empty_outputs(P, set=False) for _ in range(2)]
        osets = [oest.empty_outputs(P, renew=True) for _ in range(2)]
        touts = [oest.empty_outputs(P, track=True) for _ in range(2)]
        um = oest.empty_outputs(P, update_mask=True)
        for k in range(2):
            sets[k].update({kk: v.clone() for kk, v in S1.items()})
            osets[k]["count"].fill_(-1)
            touts[k]["label"].fill_(-1); touts[k]["id"].fill_(-1); touts[k]["stat"].fill_(0); touts[k]["max_id"].fill_(1)
            touts[k]["H"].copy_(torch.eye(4, device=dev).expand_as(touts[k]["H"]))
        graphs = []
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for k in range(2):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    for mc, pm in zip(g_mc, pristine):
                        mc.copy_(pm)
                    kc = ex.extract(g_gray, describe=False, out=kout)
                    est.build(kc, g_dl, g_fl, g_ml, K, sets[1 - k])
                    cm = est.track(sets[1 - k], K, out=cams[k])
                    oest.update_mask(g_dl, g_fl, g_ml, g_mc, samples=osets[1 - k], out=um)
                    o = oest.track(g_dl, g_fl, g_ml, g_dc, g_mc, K, Tcw_last=sets[1 - k]["Tcw"], Tcw_cur=cm["T"], prev=touts[1 - k], samples=osets[1 - k],
                                   out=touts[k])
                    est.renew(sets[1 - k], cm, kc, g_dc, g_fc, g_mc, K, out=sets[k])
                    oest.renew(o, g_dc, g_fc, g_mc, K, Tcw_cur=cm["T"], out=osets[k])
                graphs.append(g)
        torch.cuda.current_stream(dev).wait_stream(side)
        for r in range(a.warmup):
            graphs[r % 2].replay()
        torch.cuda.synchronize()
        step_ms = events(lambda: (graphs[0].replay(), graphs[1].replay()), a.reps) / 2

        # the tracker on the same frames
        trs = [capi.Tracker(ctx, local_batch=0) for _ in range(P)]
        gt = [list(range(1, 6))] * P
        run = lambda t: capi.track_tensors_batch(trs, gray[t], [x.clone() for x in dep[t]], flo[t], [x.clone() for x in msk[t]], gt, writeback=False)
        for t in range(3):
            run(t)
        ts = []
        for r in range(a.reps):
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            run(1 + r % 2)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - h0) * 1e3)
        tracker_ms = float(np.median(ts))
        rows = S2h["count"][:P].astype(np.float64)
        print(json.dumps(dict(P=P, build_ms=round(build_ms, 4), track_ms=round(track_ms, 4), renew_ms=round(renew_ms, 4), host_ms=round(host_ms, 2),
                              equal_host=bool(equal), step_graph_ms=round(step_ms, 3), tracker_ms=round(tracker_ms, 2), rows_mean=float(rows.mean()),
                              **info)), flush=True)


if __name__ == "__main__":
    main()
