#!/usr/bin/env python
"""bench_object_renew.py -- the object half of RenewFrameInfo on the device (capi.ObjectMotion.renew) against the host route it replaces,
and what carrying the sets costs the per-frame object step.

Workload: config-3-shaped sequences (synth.make_sequence_frame, KITTI-shaped 1242x375, 3-5 moving objects with stable labels, step 4,
ThDepthObj 25, MaxTrackPointOBJ 800).  View i is the pair (t, t + 1) of sequence i, t = 1 + i % 4, entered with the set that renewing pair
(t - 1, t) left; a batch of P pairs takes view p % V; max_objects 8.  One pair step per call.  update_mask writes the current masks in place,
so every step graph first restores them from a pristine copy (a device copy inside the graph).  The graphs of one size are replayed
alternately.  For P in {1, 8, 32, 64} it prints one JSON line:
  renew_ms          one replay of renew() alone (median of CUDA events around --reps replays)
  step_set_ms       restore + update_mask(samples=S) -> track(samples=S) -> renew in one graph
  step_raster_ms    restore + update_mask -> track with samples=None (the step before this change) in one graph
  host_ms           the host route, host clock: D2H of the track result and the current planes, then per pair Frame.upload,
                    Frame.sample_objects and capi.renew_frame_info (vdo_renew_frame_info, empty static part)
  equal_host        every pair's set equals the host route's
  rows_mean, carried_mean, topped_mean, new_mean   rows per pair, and its split into carried LM inliers, top-ups and new labels
and, from a separate torch.profiler run of --prof-reps eager renew() calls, the device time per call of each kernel.  The GPU name and
power limit are read in the same run.

  python bench_object_renew.py [--pairs 1,8,32,64] [--views 8] [--reps 30] [--warmup 5] [--prof-reps 5]
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
from tests.object_motion_reference import inv4  # noqa: E402

W, H, STEP, M = 1242, 375, 4, 8
CAP = ((W + STEP - 1) // STEP) * ((H + STEP - 1) // STEP)
KERNEL_RE = r"(k_om_sample|k_rn_select)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    V = a.views
    t_ = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    depth = lambda raw: np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
    views = []
    for i in range(V):
        t = 1 + i % 4
        fs = [make_sequence_frame(t + k, seed=i, width=W, height=H, n_obj=3 + i % 3) for k in (-1, 0, 1)]
        views.append([dict(d=t_(depth(f["depth_raw"])), f=t_(f["flow"]), m=t_(f["mask"]), T=t_(np.linalg.inv(f["Twc"]).astype(np.float32)[None])) for f in fs])
    info = gpu_info()
    st = torch.cuda.current_stream(dev)

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

    def time_alternating(graphs):
        for _ in range(a.warmup):
            for g in graphs:
                g.replay()
        ms = [[] for _ in graphs]
        for _ in range(a.reps):
            for g, out in zip(graphs, ms):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                g.replay()
                e1.record(st)
                e1.synchronize()
                out.append(e0.elapsed_time(e1))
        return [float(np.median(m)) for m in ms]

    for P in [int(v) for v in a.pairs.split(",")]:
        est = capi.ObjectMotion(ctx, P, M, CAP)
        fr = [[views[p % V][k] for p in range(P)] for k in range(3)]            # frame t - 1, t, t + 1 of every pair
        col = lambda k, key: [x[key] for x in fr[k]]
        T = [torch.cat(col(k, "T")) for k in range(3)]
        # the carried set of pair (t - 1, t): the state a sequence is in when pair (t, t + 1) comes
        o0 = est.track(col(0, "d"), col(0, "f"), col(0, "m"), col(1, "d"), col(1, "m"), KITTI_K, Tcw_last=T[0], Tcw_cur=T[1])
        S0 = est.renew(o0, col(1, "d"), col(1, "f"), col(1, "m"), KITTI_K, Tcw_cur=T[1])
        pristine = torch.stack(col(2, "m"))
        work = pristine.clone()
        mc = list(work.unbind(0))
        um, to_, S1 = est.empty_outputs(P, update_mask=True), est.empty_outputs(P, track=True), est.empty_outputs(P, renew=True)
        obj = est.track(col(1, "d"), col(1, "f"), col(1, "m"), col(2, "d"), mc, KITTI_K, Tcw_last=T[1], Tcw_cur=T[2], prev=o0, samples=S0, out=to_)

        def renew():
            est.renew(obj, col(2, "d"), col(2, "f"), mc, KITTI_K, Tcw_cur=T[2], out=S1)

        def step(with_set):
            def run():
                work.copy_(pristine)
                est.update_mask(col(1, "d"), col(1, "f"), col(1, "m"), mc, samples=S0 if with_set else None, out=um)
                o = est.track(col(1, "d"), col(1, "f"), col(1, "m"), col(2, "d"), mc, KITTI_K, Tcw_last=T[1], Tcw_cur=T[2], prev=o0,
                              samples=S0 if with_set else None, out=to_)
                if with_set:
                    est.renew(o, col(2, "d"), col(2, "f"), mc, KITTI_K, Tcw_cur=T[2], out=S1)
            return run

        g_renew, g_set, g_raster = capture(renew), capture(step(True)), capture(step(False))
        renew_ms, set_ms, raster_ms = time_alternating([g_renew, g_set, g_raster])
        g_set.replay()
        torch.cuda.synchronize()
        got = {k: v.cpu().numpy() for k, v in S1.items()}
        # the host route: D2H of the track result and the current planes, then per pair the resident frame, its samples and the renewal
        t0 = time.perf_counter()
        g = {k: v.cpu().numpy() for k, v in to_.items()}
        equal = True
        for p in range(P):
            dh, fh, mh = (x.cpu().numpy() for x in (fr[2][p]["d"], fr[2][p]["f"], mc[p]))
            cur = capi.Frame(ctx, W, H)
            cur.upload(depth=dh, flow=fh, mask=mh)
            s = cur.sample_objects(25.0, STEP)
            n = int(g["n_samples"][p])
            keys = np.stack([(g["sample_x"][p, :n] + g["sample_flow_ref"][p, :n, 0]).astype(np.float32),
                             (g["sample_y"][p, :n] + g["sample_flow_ref"][p, :n, 1]).astype(np.float32)], 1)
            slots = [j for j in range(M) if g["label"][p, j] != -1]
            inl = [[k for k in np.nonzero((g["sample_slot"][p, :n] == j) & (g["sample_flags"][p, :n] & 2 > 0))[0]] for j in slots]
            Tc = fr[2][p]["T"][0].cpu().numpy()
            _, o = capi.renew_frame_info(cur, [], np.zeros((0, 2)), np.zeros((0, 2)), 0, inl, g["stat"][p, slots], g["label"][p, slots], g["id"][p, slots],
                                         keys, g["obj_label"][p, :n], np.stack([s["x"], s["y"]], 1).astype(np.float32), s["depth"], s["label"],
                                         np.stack([s["fx"], s["fy"]], 1), np.stack([s["cx"], s["cy"]], 1), 800, np.asarray(KITTI_K, np.float32), inv4(Tc))
            cur.close()
            c = int(got["count"][p])
            equal &= c == len(o["keys"])
            equal &= bool(np.array_equal(np.stack([got["x"][p, :c], got["y"][p, :c]], 1).astype(np.float32), o["keys"]))
            for k, ok in (("label", "sem"), ("inlier_id", "inlier_id"), ("obj_label", "label"), ("depth", "depth"), ("point", "p3d")):
                equal &= bool(np.array_equal(got[k][p, :c], o[ok]))
        host_ms = (time.perf_counter() - t0) * 1e3
        rows = [got["inlier_id"][p, :got["count"][p]] for p in range(P)]
        labs = [got["obj_label"][p, :got["count"][p]] for p in range(P)]
        print(json.dumps({"P": P, "max_objects": M, "renew_ms": round(renew_ms, 4), "step_set_ms": round(set_ms, 4), "step_raster_ms": round(raster_ms, 4),
                          "host_ms": round(host_ms, 2), "equal_host": bool(equal), "rows_mean": round(float(got["count"].mean()), 1),
                          "carried_mean": round(float(np.mean([(r >= 0).sum() for r in rows])), 1),
                          "topped_mean": round(float(np.mean([((r < 0) & (lb >= 1)).sum() for r, lb in zip(rows, labs)])), 1),
                          "new_mean": round(float(np.mean([(lb == -2).sum() for lb in labs])), 1),
                          "status_bits": int(np.bitwise_or.reduce(got["status"])), **info}), flush=True)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.prof_reps):
                renew()
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            hit = re.search(KERNEL_RE, e.key)
            if hit:
                split[hit.group(1)] = split.get(hit.group(1), 0.0) + e.device_time_total / 1e3 / a.prof_reps     # us -> ms per call
        print(json.dumps({"P": P, "kernel_ms_per_call": {k: round(v, 4) for k, v in sorted(split.items())}, "kernel_ms_sum": round(sum(split.values()), 4),
                          **info}), flush=True)
        est.close()


if __name__ == "__main__":
    main()
