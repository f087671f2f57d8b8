#!/usr/bin/env python
"""bench_object_update_mask.py -- UpdateMask on the device (capi.ObjectMotion.update_mask) against the host route it replaces, and the
cost it adds to the device pair chain.

Workload: config-3-shaped frame pairs (synth.make_sequence_frame (t, t + 1), KITTI-shaped 1242x375, 3-5 moving objects with stable labels,
step 4, ThDepthObj 25), where the current mask of view i misses its one (even i) or two (odd i) largest objects, as a segmentation network
that drops objects for a frame.  A batch of P pairs takes view p % V for pair p; max_objects 8.  update_mask writes the current masks in
place, so every timed variant first restores them from a pristine copy (a device copy inside the graph); the copy is timed alone too and
the update's cost is the difference.  The variants of one size are replayed alternately.  For P in {1, 8, 32, 64} it prints one JSON line:
  restore_ms         one replay of the restore copy alone (median of CUDA events around --reps replays)
  update_graph_ms    restore + update_mask in one graph; update_ms = update_graph_ms - restore_ms
  host_ms            the host route, host clock: D2H of the planes, then per pair Frame.upload of the last and current frames,
                     Frame.sample_objects and capi.update_mask (vdo_update_mask)
  chain_ms           restore + extract -> match -> PnP -> refine -> update_mask -> track in one graph (V view pairs of
                     synth.make_view_pair, 2 V frames extracted); chain_no_update_ms the same without update_mask
  equal_host         the device masks and recovered slots equal the host route's
and, from a separate torch.profiler run of --prof-reps eager calls, the device time per call of each kernel (k_um_vote is the sequential
per-slot vote).  The GPU name and power limit are read in the same run.

  python bench_object_update_mask.py [--pairs 1,8,32,64] [--views 8] [--reps 30] [--warmup 5] [--prof-reps 5]
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

W, H, STEP, M = 1242, 375, 4, 8
CAP = ((W + STEP - 1) // STEP) * ((H + STEP - 1) // STEP)
KERNEL_RE = r"(k_om_sample|k_um_\w+(?:<\d>)?)"


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
    from vdo_slam_b200.synth import KITTI_BF, KITTI_DEPTH_FACTOR, KITTI_K, make_sequence_frame, make_view_pair

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    V = a.views
    fr = []
    for i in range(V):
        f0, f1 = (make_sequence_frame(i % 4 + k, seed=i, width=W, height=H, n_obj=3 + i % 3) for k in (0, 1))
        depth = lambda raw: np.where(raw < 0, np.float32(0), KITTI_BF / (raw / KITTI_DEPTH_FACTOR)).astype(np.float32)
        labs, cnt = np.unique(f1["mask"][f1["mask"] != 0], return_counts=True)
        mask1 = f1["mask"].copy()
        mask1[np.isin(mask1, labs[np.argsort(-cnt)][:1 + i % 2])] = 0
        fr.append(dict(depth=depth(f0["depth_raw"]), flow=f0["flow"], mask=f0["mask"], depth1=depth(f1["depth_raw"]), mask1=mask1))
    vs = [make_view_pair(t=i % 4, seed=i, width=W, height=H) for i in range(V)]
    images = torch.from_numpy(np.stack([g for v in vs for g in (v["gray_a"], v["gray_b"])])).to(dev)
    ex = capi.OrbExtractor(ctx, W, H, 2 * V, n_features=3000)
    cap = ex.capacity
    eo = ex.empty_outputs(2 * V)
    info = gpu_info()
    st = torch.cuda.current_stream(dev)
    t_ = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    D, F, Mk, D1 = ([t_(f[k]) for f in fr] for k in ("depth", "flow", "mask", "depth1"))
    cam_depths = [t_(v["depth_a"]) for v in vs]

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
        sel = [p % V for p in range(P)]
        d, f, m, d1 = [D[i] for i in sel], [F[i] for i in sel], [Mk[i] for i in sel], [D1[i] for i in sel]
        pristine = t_(np.stack([fr[i]["mask1"] for i in sel]))
        work = pristine.clone()
        mc = list(work.unbind(0))
        uo, to_ = est.empty_outputs(P, update_mask=True), est.empty_outputs(P, track=True)

        def restore():
            work.copy_(pristine)

        def update():
            restore()
            est.update_mask(d, f, m, mc, out=uo)

        pairs = [(2 * (p % V), 2 * (p % V) + 1) for p in range(P)]
        dq = [cam_depths[p % V] for p in range(P)]
        Tq = np.stack([vs[p % V]["Tcw_a"] for p in range(P)]).astype(np.float32)
        solver, refiner = capi.PnpSolver(ctx, P, cap, 500), capi.PoseRefiner(ctx, P, cap)
        mo, po_, ro = capi.orb_match_empty_outputs(ctx, P, cap, cap, 2), solver.empty_outputs(P, cap), refiner.empty_outputs(P, cap)

        def chain(with_update):
            def run():
                restore()
                r = ex.extract(images, out=eo)
                mt = capi.orb_match(ctx, r, r, pairs, k=2, out=mo)
                s = solver.solve(r, r, pairs, mt, dq, KITTI_K, Tcw_query=Tq, ratio=0.8, out=po_)
                t = refiner.refine(r, r, pairs, mt, dq, KITTI_K, T_init=s["T"], mask=s["inlier"], Tcw_query=Tq, ratio=0.8, out=ro)
                if with_update:
                    est.update_mask(d, f, m, mc, out=uo)
                est.track(d, f, m, d1, mc, KITTI_K, Tcw_cur=t["T"], out=to_)
            return run

        g_restore, g_update, g_chain, g_chain0 = capture(restore), capture(update), capture(chain(True)), capture(chain(False))
        restore_ms, update_ms, chain_ms, chain0_ms = time_alternating([g_restore, g_update, g_chain, g_chain0])
        g_update.replay()
        torch.cuda.synchronize()
        got, got_mask = {k: v.cpu().numpy() for k, v in uo.items()}, work.cpu().numpy()
        # the host route: D2H of the planes, then per pair the resident frames, the samples and vdo_update_mask
        t0 = time.perf_counter()
        equal = True
        for p in range(P):
            dh, fh, mh, ch = (x.cpu().numpy() for x in (d[p], f[p], m[p], pristine[p]))
            last, cur = capi.Frame(ctx, W, H), capi.Frame(ctx, W, H)
            last.upload(depth=dh, flow=fh, mask=mh)
            cur.upload(mask=ch)
            s = last.sample_objects(25.0, STEP)
            slots = sorted(set(s["label"].tolist()))[:M]
            keep = np.isin(s["label"], slots)
            hm, warped = capi.update_mask(cur, last, s["label"][keep], np.stack([s["cx"][keep], s["cy"][keep]], 1))
            last.close(); cur.close()
            equal &= bool(np.array_equal(hm, got_mask[p]))
            equal &= sorted(warped) == sorted(int(L) for L, r in zip(got["label"][p], got["recovered"][p]) if r)
        host_ms = (time.perf_counter() - t0) * 1e3
        print(json.dumps({"P": P, "max_objects": M, "restore_ms": round(restore_ms, 4), "update_graph_ms": round(update_ms, 4),
                          "update_ms": round(update_ms - restore_ms, 4), "host_ms": round(host_ms, 2), "chain_ms": round(chain_ms, 4),
                          "chain_no_update_ms": round(chain0_ms, 4), "equal_host": bool(equal), "recovered": int(got["recovered"].sum()),
                          "dropped": int(sum(1 + i % 2 for i in sel)), "mean_samples": round(float(got["n_samples"].mean()), 1), **info}), flush=True)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.prof_reps):
                update()
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            hit = re.search(KERNEL_RE, e.key)
            if hit:
                split[hit.group(1)] = split.get(hit.group(1), 0.0) + e.device_time_total / 1e3 / a.prof_reps     # us -> ms per call
        print(json.dumps({"P": P, "kernel_ms_per_call": {k: round(v, 4) for k, v in sorted(split.items())}, "kernel_ms_sum": round(sum(split.values()), 4),
                          **info}), flush=True)
        est.close(); solver.close(); refiner.close()


if __name__ == "__main__":
    main()
