#!/usr/bin/env python
"""bench_pnp_refine.py -- refined poses of matched ORB frame pairs on the device (capi.PoseRefiner) against the host route it replaces.

Workload: the view pairs of bench_pnp_match.py (synth.make_view_pair, KITTI-shaped 1242x375, 3 000 ORB features, orb_match k = 2), PnP with
ratio 0.8, 500 iterations, thr 0.4 px (the reference's) or 2 px; then PoseOptimizationFlow2Cam (quirk 1) from PnP's pose on PnP's inliers.
A batch of P pairs takes view pair p % V for pair p.  For P in {1, 8, 32, 64} and each thr it prints one JSON line with
  graph_ms        device time of one PoseRefiner.refine call captured in a CUDA graph: median of CUDA events around --reps replays
  host_ms         the host route on the same inputs, host clock: D2H of matches, keypoints, counts, PnP pose and inlier flags, the numpy
                  gather of tests/pnp_match_reference.py restricted to the inliers, and capi.pose_opt_flow2 of all P problems
  chain_graph_ms  extract -> match -> PnP -> refine captured in one CUDA graph (2 V frames extracted), median of CUDA events
  chain_host_ms   extract -> match -> PnP in one CUDA graph, then the host route for the refinement, host clock around both
  equal_host      the device result equals the host route bit for bit (T, stats, flows and inlier flags)
  rot_err_deg / t_err_m   median and max over the pairs of the PnP pose's and the refined pose's error against the synthetic truth T_ba
and, from a separate torch.profiler run of --prof-reps eager calls, the device time per call of each kernel (gather, cluster LM,
single-CTA LM, scatter).  The GPU name and power limit are read in the same run.

  python bench_pnp_refine.py [--pairs 1,8,32,64] [--views 8] [--reps 50] [--warmup 5] [--prof-reps 10]
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

from bench_pnp_match import gpu_info, rot_err_deg  # noqa: E402

W, H = 1242, 375
KERNELS = ("k_refine_gather", "k_refine_lm_cl", "k_refine_lm", "k_refine_scatter")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    from tests import pnp_match_reference as R
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import KITTI_K, make_view_pair

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    V = a.views
    vs = [make_view_pair(t=3 * i, seed=i, dt=1 + i % 3, yaw_extra=0.01 * ((i % 5) - 2), shift=(0.1 * ((i % 3) - 1), 0.0, 0.0), width=W, height=H)
          for i in range(V)]
    images = torch.from_numpy(np.stack([g for v in vs for g in (v["gray_a"], v["gray_b"])])).to(dev)
    ex = capi.OrbExtractor(ctx, W, H, 2 * V, n_features=3000)
    cap = ex.capacity
    eo = ex.empty_outputs(2 * V)
    S = ex.extract(images, out=eo)
    torch.cuda.synchronize()
    assert int(S["status"].abs().sum()) == 0
    depths = [torch.from_numpy(v["depth_a"]).to(dev) for v in vs]
    depths_h = [v["depth_a"] for v in vs]
    solver, refiner = capi.PnpSolver(ctx, 64, cap, 500), capi.PoseRefiner(ctx, 64, cap)
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

    def host_route(P, pairs, m, po):
        """D2H, numpy gather restricted to the PnP inliers, capi.pose_opt_flow2: (per pair the query indices, the host results)"""
        idx, dist = m["idx"].cpu().numpy(), m["dist"].cpu().numpy()
        Sh = {k: S[k].cpu().numpy() for k in ("x", "y", "count")}
        T0, inl = po["T"].cpu().numpy(), po["inlier"].cpu().numpy()
        probs, sels = [], []
        for p, (q, t) in enumerate(pairs):
            sel, obj, img = R.gather(Sh["x"][q], Sh["y"][q], Sh["count"][q], Sh["x"][t], Sh["y"][t], Sh["count"][t], idx[p], dist[p], depths_h[p % V],
                                     KITTI_K, None, 0.8, None)
            keep = inl[p][sel] != 0
            sel, z, img = sel[keep], obj[keep, 2], img[keep]
            pts = np.stack([Sh["x"][q][sel], Sh["y"][q][sel]], 1)
            probs.append(dict(pts=pts, depth=z, flow=(img - pts).astype(np.float32), K=KITTI_K, Tcw_last=np.eye(4, dtype=np.float32), T_init=T0[p]))
            sels.append(sel)
        return sels, capi.pose_opt_flow2(ctx, probs, quirk=1, modes=[0] * P)

    for P in [int(v) for v in a.pairs.split(",")]:
        pairs = [(2 * (p % V), 2 * (p % V) + 1) for p in range(P)]
        dp = [depths[p % V] for p in range(P)]
        mo = capi.orb_match_empty_outputs(ctx, P, cap, cap, 2)
        for thr in (0.4, 2.0):
            po, ro = solver.empty_outputs(P, cap), refiner.empty_outputs(P, cap)

            def front():
                m = capi.orb_match(ctx, S, S, pairs, k=2, out=mo)
                solver.solve(S, S, pairs, m, dp, KITTI_K, ratio=0.8, thr=thr, out=po)

            def refine():
                refiner.refine(S, S, pairs, mo, dp, KITTI_K, T_init=po["T"], mask=po["inlier"], ratio=0.8, out=ro)

            front()
            torch.cuda.synchronize()
            gms = time_graph(capture(refine))
            gd = {k: v.cpu().numpy() for k, v in ro.items()}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sels, ref = host_route(P, pairs, mo, po)
            host_ms = (time.perf_counter() - t0) * 1e3
            equal = all(np.array_equal(gd["T"][p], ref[p]["T"]) and np.array_equal(gd["stats"][p], ref[p]["stats"])
                        and np.array_equal(gd["flow"][p, sels[p]], ref[p]["flow"]) and np.array_equal(gd["inlier"][p, sels[p]], ref[p]["inlier"].astype(np.uint8))
                        and int(gd["n_points"][p]) == len(sels[p]) for p in range(P))
            # the whole chain in one graph, and the chain with the host route for the last step
            def chain():
                ex.extract(images, out=eo)
                front()
                refine()

            cms = time_graph(capture(chain))
            g_front = capture(lambda: (ex.extract(images, out=eo), front()))
            hms = []
            for _ in range(max(3, a.reps // 10)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                g_front.replay()
                host_route(P, pairs, mo, po)
                hms.append((time.perf_counter() - t0) * 1e3)
            Tp = po["T"].cpu().numpy()
            err = lambda T: ([rot_err_deg(T[p][:3, :3].astype(np.float64), vs[p % V]["T_ba"][:3, :3]) for p in range(P)],
                             [float(np.linalg.norm(T[p][:3, 3] - vs[p % V]["T_ba"][:3, 3])) for p in range(P)])
            (rp, tp), (rr, tr) = err(Tp), err(gd["T"])
            stat = lambda v: [round(float(np.median(v)), 4), round(float(max(v)), 4)]
            med = float(np.median(gms))
            print(json.dumps({"P": P, "thr": thr, "graph_ms": round(med, 4), "graph_ms_min": round(min(gms), 4), "graph_ms_max": round(max(gms), 4),
                              "graph_us_per_pair": round(med * 1e3 / P, 2), "host_ms": round(host_ms, 2),
                              "chain_graph_ms": round(float(np.median(cms)), 4), "chain_host_ms": round(float(np.median(hms)), 2),
                              "equal_host": bool(equal), "mean_points": round(float(gd["n_points"].mean()), 1),
                              "min_points": int(gd["n_points"].min()), "max_points": int(gd["n_points"].max()),
                              "mean_lm_iters": round(float(gd["stats"][:, 0].mean()), 1), "mean_inliers": round(float(gd["stats"][:, 4].mean()), 1),
                              "pnp_rot_err_deg_med_max": stat(rp), "refined_rot_err_deg_med_max": stat(rr),
                              "pnp_t_err_m_med_max": stat(tp), "refined_t_err_m_med_max": stat(tr), **info}), flush=True)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.prof_reps):
                    refine()
                torch.cuda.synchronize()
            split = {k: 0.0 for k in KERNELS}
            for e in prof.key_averages():
                hit = re.search(r"(k_refine_\w+)\(", e.key)
                if hit and hit.group(1) in split:
                    split[hit.group(1)] += e.device_time_total / 1e3 / a.prof_reps      # us -> ms per call
            print(json.dumps({"P": P, "thr": thr, "kernel_ms_per_call": {k.replace("k_refine_", ""): round(v, 4) for k, v in split.items()},
                              "kernel_ms_sum": round(sum(split.values()), 4), **info}), flush=True)


if __name__ == "__main__":
    main()
