#!/usr/bin/env python
"""bench_object_track.py -- tracked objects on the device (capi.ObjectMotion.track: scene flow, DynObjTracking, then the object step
for the dynamic objects) against the host route it replaces, and against ObjectMotion.estimate on the same pairs.

Workload: config-3-shaped frame pairs (synth.make_sequence_frame (t, t + 1), KITTI-shaped 1242x375, 3-5 moving objects, step 4,
ThDepthObj 25, true camera poses), the reference's settings (500 iterations, thr 0.4, conf 0.98, min_inliers 50, quirk 1, SFMgThres 0.12,
SFDsThres 0.3, the KITTI border band 25 / 50), each pair the start of its sequence (prev = None).  A batch of P pairs takes frame pair p % V
for pair p.  For P in {1, 8, 32, 64} and max_objects M in {8, 32} it prints one JSON line with
  graph_ms           device time of one ObjectMotion.track call captured in a CUDA graph: median of CUDA events around --reps replays
  estimate_graph_ms  the same for ObjectMotion.estimate on the same last frames: the difference is what tracking adds
  host_ms            the host route on the same inputs, host clock: D2H of the planes, then tests/object_track_reference.host_track per pair
  chain_graph_ms     extract -> match -> PnP -> refine -> track captured in one CUDA graph (the camera chain on V view pairs of
                     synth.make_view_pair, 2 V frames extracted), median of CUDA events
  equal_host         the device result equals the host route bit for bit (every output)
and, from a separate torch.profiler run of --prof-reps eager calls, the device time per call of each kernel (k_ot_group holds the
sequential per-slot sums of the classification).  The GPU name and power limit are read in the same run.

  python bench_object_track.py [--pairs 1,8,32,64] [--objects 8,32] [--views 8] [--reps 30] [--warmup 5] [--prof-reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_pnp_match import gpu_info  # noqa: E402

W, H, STEP = 1242, 375, 4
CAP = ((W + STEP - 1) // STEP) * ((H + STEP - 1) // STEP)
KERNEL_RE = r"(k_om_\w+|k_ot_\w+|k_pnp_\w+|k_refine_lm\w*)\("


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--objects", default="8,32")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from tests import object_track_reference as R
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame, make_view_pair

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    V = a.views
    fr = []
    for i in range(V):
        f0, f1 = make_sequence_frame(i % 4, seed=i, width=W, height=H, n_obj=3 + i % 3), make_sequence_frame(i % 4 + 1, seed=i, width=W, height=H, n_obj=3 + i % 3)
        raw = f0["depth_raw"]
        depth = np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
        raw1 = f1["depth_raw"]
        depth1 = np.where(raw1 < 0, np.float32(0), KITTI_BF / (raw1 / KITTI_DEPTH_FACTOR)).astype(np.float32)
        fr.append(dict(depth=depth, flow=f0["flow"], mask=f0["mask"], depth1=depth1, mask1=f1["mask"], Tl=np.linalg.inv(f0["Twc"]).astype(np.float32),
                       Tc=np.linalg.inv(f1["Twc"]).astype(np.float32)))
    vs = [make_view_pair(t=i % 4, seed=i, width=W, height=H) for i in range(V)]
    images = torch.from_numpy(np.stack([g for v in vs for g in (v["gray_a"], v["gray_b"])])).to(dev)
    ex = capi.OrbExtractor(ctx, W, H, 2 * V, n_features=3000)
    cap = ex.capacity
    eo = ex.empty_outputs(2 * V)
    info = gpu_info()
    st = torch.cuda.current_stream(dev)
    D = [torch.from_numpy(f["depth"]).to(dev) for f in fr]
    F = [torch.from_numpy(f["flow"]).to(dev) for f in fr]
    Mk = [torch.from_numpy(f["mask"]).to(dev) for f in fr]
    D1 = [torch.from_numpy(f["depth1"]).to(dev) for f in fr]
    Mk1 = [torch.from_numpy(f["mask1"]).to(dev) for f in fr]
    cam_depths = [torch.from_numpy(v["depth_a"]).to(dev) for v in vs]

    def capture(fn):
        side = torch.cuda.Stream(dev)
        side.wait_stream(st)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            fn()
            with torch.cuda.graph(g, stream=side):
                fn()
        st.wait_stream(side)
        return g

    def time_graph(g):
        for _ in range(a.warmup):
            g.replay()
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            g.replay()
            e1.record(st)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms

    for M in [int(v) for v in a.objects.split(",")]:
        for P in [int(v) for v in a.pairs.split(",")]:
            est = capi.ObjectMotion(ctx, P, M, CAP)
            sel = [p % V for p in range(P)]
            d, f, m, d1, m1 = [D[i] for i in sel], [F[i] for i in sel], [Mk[i] for i in sel], [D1[i] for i in sel], [Mk1[i] for i in sel]
            Tl = torch.from_numpy(np.stack([fr[i]["Tl"] for i in sel])).to(dev)
            Tc = torch.from_numpy(np.stack([fr[i]["Tc"] for i in sel])).to(dev)
            oo, eo_ = est.empty_outputs(P, track=True), est.empty_outputs(P)

            def objects(Tcur=Tc):
                est.track(d, f, m, d1, m1, KITTI_K, Tcw_last=Tl, Tcw_cur=Tcur, out=oo)

            ems = time_graph(capture(lambda: est.estimate(d, f, m, KITTI_K, Tcw_last=Tl, Tcw_cur=Tc, out=eo_)))
            gms = time_graph(capture(objects))
            g = {k: v.cpu().numpy() for k, v in oo.items()}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref = []
            for p in range(P):
                dh, fh, mh, d1h, m1h = (x[p].cpu().numpy() for x in (d, f, m, d1, m1))
                ref.append(R.host_track(ctx, dh, fh, mh, d1h, m1h, KITTI_K, M, Tl[p].cpu().numpy(), Tc[p].cpu().numpy()))
            host_ms = (time.perf_counter() - t0) * 1e3
            equal = True
            for p, r in enumerate(ref):
                n = int(r["n_samples"])
                equal &= int(g["n_samples"][p]) == n and int(g["pair_status"][p]) == int(r["pair_status"]) and int(g["max_id"][p]) == int(r["max_id"])
                equal &= all(np.array_equal(g[k][p, :n], r[k]) for k in r if k.startswith("sample_") or k in ("label_cur", "depth_cur", "flow3d", "obj_label"))
                equal &= all(np.array_equal(g[k][p], r[k]) for k in ("label", "H", "X", "T_init", "centre", "velocity", "info", "stats", "status", "id", "cls",
                                                                      "vote", "stat"))
            # the whole chain in one graph: the camera pose of the current frame from the ORB chain feeds the object step
            pairs = [(2 * (p % V), 2 * (p % V) + 1) for p in range(P)]
            dq = [cam_depths[p % V] for p in range(P)]
            Tq = np.stack([vs[p % V]["Tcw_a"] for p in range(P)]).astype(np.float32)
            solver, refiner = capi.PnpSolver(ctx, P, cap, 500), capi.PoseRefiner(ctx, P, cap)
            mo, po_, ro = capi.orb_match_empty_outputs(ctx, P, cap, cap, 2), solver.empty_outputs(P, cap), refiner.empty_outputs(P, cap)

            def chain():
                r = ex.extract(images, out=eo)
                mt = capi.orb_match(ctx, r, r, pairs, k=2, out=mo)
                s = solver.solve(r, r, pairs, mt, dq, KITTI_K, Tcw_query=Tq, ratio=0.8, out=po_)
                t = refiner.refine(r, r, pairs, mt, dq, KITTI_K, T_init=s["T"], mask=s["inlier"], Tcw_query=Tq, ratio=0.8, out=ro)
                objects(t["T"])

            cms = time_graph(capture(chain))
            med = float(np.median(gms))
            print(json.dumps({"P": P, "max_objects": M, "graph_ms": round(med, 4), "graph_ms_min": round(min(gms), 4), "graph_ms_max": round(max(gms), 4),
                              "graph_us_per_pair": round(med * 1e3 / P, 2), "estimate_graph_ms": round(float(np.median(ems)), 4), "host_ms": round(host_ms, 2),
                              "chain_graph_ms": round(float(np.median(cms)), 4), "equal_host": bool(equal), "objects": int((g["label"] != -1).sum()),
                              "dynamic": int((g["cls"] == capi.OT_DYNAMIC).sum()), "stat": int(g["stat"].sum()),
                              "mean_samples": round(float(g["n_samples"].mean()), 1), "device_mb": round(est.info()["device_bytes"] / 2 ** 20, 1),
                              **info}), flush=True)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.prof_reps):
                    objects()
                torch.cuda.synchronize()
            split = {}
            for e in prof.key_averages():
                hit = re.search(KERNEL_RE, e.key)
                if hit:
                    split[hit.group(1)] = split.get(hit.group(1), 0.0) + e.device_time_total / 1e3 / a.prof_reps     # us -> ms per call
            print(json.dumps({"P": P, "max_objects": M, "kernel_ms_per_call": {k: round(v, 4) for k, v in sorted(split.items())},
                              "kernel_ms_sum": round(sum(split.values()), 4), **info}), flush=True)
            est.close(); solver.close(); refiner.close()


if __name__ == "__main__":
    main()
