#!/usr/bin/env python
"""bench_pnp_match.py -- poses of matched ORB frame pairs on the device (capi.PnpSolver) against the host paths it replaces.

Workload: V synthetic view pairs (synth.make_view_pair, KITTI-shaped 1242x375, static corridor, B's image warped from A's through the
geometry), ORB from one OrbExtractor (3 000 features, scale 1.2, 8 levels, FAST 20 / 7), matched query A -> train B with orb_match (k = 2).
A batch of P pairs takes view pair p % V for pair p (P > V repeats view pairs; every pair is still solved on its own).  Settings:
ratio 0.8, no depth cap, 500 iterations, confidence 0.98, and thr = 0.4 px (the reference's solvePnPRansac call) or 2 px.
For P in {1, 8, 32, 64} and each thr it prints one JSON line with
  graph_ms        device time of one PnpSolver.solve call captured in a CUDA graph: median of CUDA events around --reps replays
  host_init_ms    (a) the host path on the same matches: D2H of idx / dist / keypoints / counts, the numpy gather of
                  tests/pnp_match_reference.py (depth read from host copies) and capi.init_model_batch of all P problems, host clock
  cv2_ms          (b) cv2.solvePnPRansac(AP3P) on each pair's gathered correspondences, summed over the P pairs, host clock
  equal_host      the device result equals (a) bit for bit (T, inlier sets, iteration counters)
  rot_err_deg / t_err_m   median and max over the pairs of the device pose's error against the synthetic truth T_ba
and, from a separate torch.profiler run of --prof-reps eager calls, the device time per call of each kernel (gather, samples, hyp, score,
finish, scatter).  The GPU name and power limit are read in the same run.

  python bench_pnp_match.py [--pairs 1,8,32,64] [--views 8] [--reps 50] [--warmup 5] [--prof-reps 10] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H = 1242, 375
KERNELS = ("k_pnp_gather", "k_pnp_samples", "k_pnp_hyp", "k_pnp_score", "k_pnp_finish", "k_pnp_scatter")


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers are still device times; say that the card could not be read
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def rot_err_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the profiler's per-kernel table (nothing is written without it)")
    a = ap.parse_args()
    import cv2
    import torch
    from tests import pnp_match_reference as R
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import KITTI_K, make_view_pair

    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    V = a.views
    vs = [make_view_pair(t=3 * i, seed=i, dt=1 + i % 3, yaw_extra=0.01 * ((i % 5) - 2), shift=(0.1 * ((i % 3) - 1), 0.0, 0.0), width=W, height=H)
          for i in range(V)]
    grays = [g for v in vs for g in (v["gray_a"], v["gray_b"])]
    ex = capi.OrbExtractor(ctx, W, H, len(grays), n_features=3000)
    r = ex.extract(torch.from_numpy(np.stack(grays)).to(dev))
    S = {k: r[k].clone() for k in ("descriptors", "x", "y", "count")}
    torch.cuda.synchronize()
    assert int(r["status"].abs().sum()) == 0
    depths = [torch.from_numpy(v["depth_a"]).to(dev) for v in vs]
    depths_h = [v["depth_a"] for v in vs]
    cap = ex.capacity
    solver = capi.PnpSolver(ctx, 64, cap, 500)
    info = gpu_info()
    Kc = np.array([[KITTI_K[0], 0, KITTI_K[2]], [0, KITTI_K[1], KITTI_K[3]], [0, 0, 1]], np.float64)
    st = torch.cuda.current_stream(dev)
    prof_rows = []

    for P in [int(v) for v in a.pairs.split(",")]:
        pairs = [(2 * (p % V), 2 * (p % V) + 1) for p in range(P)]
        m = capi.orb_match(ctx, S, S, pairs, k=2)
        dp = [depths[p % V] for p in range(P)]
        for thr in (0.4, 2.0):
            kw = dict(ratio=0.8, iters=500, thr=thr, conf=0.98)
            out = solver.empty_outputs(P, cap)
            side = torch.cuda.Stream(dev)
            side.wait_stream(st)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(side):
                solver.solve(S, S, pairs, m, dp, KITTI_K, out=out, **kw)
                with torch.cuda.graph(g, stream=side):
                    solver.solve(S, S, pairs, m, dp, KITTI_K, out=out, **kw)
            st.wait_stream(side)
            for _ in range(a.warmup):
                g.replay()
            gms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                g.replay()
                e1.record(st)
                e1.synchronize()
                gms.append(e0.elapsed_time(e1))
            gd = {k: v.cpu().numpy() for k, v in out.items()}
            # (a) the host path on the same matches
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            idx, dist = m["idx"].cpu().numpy(), m["dist"].cpu().numpy()
            Sh = {k: S[k].cpu().numpy() for k in ("x", "y", "count")}
            probs, sels = [], []
            for p, (q, t) in enumerate(pairs):
                sel, obj, img = R.gather(Sh["x"][q], Sh["y"][q], Sh["count"][q], Sh["x"][t], Sh["y"][t], Sh["count"][t], idx[p], dist[p], depths_h[p % V],
                                         KITTI_K, None, 0.8, None)
                probs.append(dict(obj=obj, img=img)); sels.append(sel)
            ref = capi.init_model_batch(ctx, probs, KITTI_K, iters=500, thr=thr, conf=0.98)
            host_ms = (time.perf_counter() - t0) * 1e3
            equal = all(np.array_equal(gd["T"][p], ref[p]["T"]) and gd["info"][p, 0] == ref[p]["iters_run"] and gd["info"][p, 1] == ref[p]["best_it"]
                        and gd["info"][p, 2] == ref[p]["n_valid"] and np.array_equal(np.nonzero(gd["inlier"][p, :Sh["count"][pairs[p][0]]])[0],
                                                                                      sels[p][ref[p]["sub"]] if ref[p]["best_it"] >= 0 else sels[p][:0])
                        for p in range(P))
            # (b) cv2 per pair on the same correspondences
            t0 = time.perf_counter()
            for pr in probs:
                cv2.solvePnPRansac(pr["obj"], pr["img"], Kc, np.zeros(4), iterationsCount=500, reprojectionError=thr, confidence=0.98, flags=cv2.SOLVEPNP_AP3P)
            cv2_ms = (time.perf_counter() - t0) * 1e3
            re = [rot_err_deg(gd["T"][p][:3, :3].astype(np.float64), vs[p % V]["T_ba"][:3, :3]) for p in range(P)]
            te = [float(np.linalg.norm(gd["T"][p][:3, 3] - vs[p % V]["T_ba"][:3, 3])) for p in range(P)]
            med = float(np.median(gms))
            print(json.dumps({"P": P, "thr": thr, "graph_ms": round(med, 4), "graph_ms_min": round(min(gms), 4), "graph_ms_max": round(max(gms), 4),
                              "graph_us_per_pair": round(med * 1e3 / P, 2), "host_init_ms": round(host_ms, 2), "cv2_ms": round(cv2_ms, 2),
                              "cv2_threads": cv2.getNumThreads(), "equal_host": bool(equal), "mean_corr": round(float(gd["n_corr"].mean()), 1),
                              "mean_inliers": round(float(gd["n_inlier"].mean()), 1), "mean_iters_run": round(float(gd["info"][:, 0].mean()), 1),
                              "rot_err_deg_med": round(float(np.median(re)), 4), "rot_err_deg_max": round(max(re), 4),
                              "t_err_m_med": round(float(np.median(te)), 4), "t_err_m_max": round(max(te), 4), **info}), flush=True)
            # per-kernel device time, in a run of its own
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.prof_reps):
                    solver.solve(S, S, pairs, m, dp, KITTI_K, out=out, **kw)
                torch.cuda.synchronize()
            split = {k: 0.0 for k in KERNELS}
            for e in prof.key_averages():
                for k in KERNELS:
                    if k in e.key:
                        split[k] += e.device_time_total / 1e3 / a.prof_reps      # us -> ms per call
            row = {"P": P, "thr": thr, "kernel_ms_per_call": {k.replace("k_pnp_", ""): round(v, 4) for k, v in split.items()},
                   "kernel_ms_sum": round(sum(split.values()), 4), **info}
            prof_rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pnp_match_kernels.json"), "w") as f:
            json.dump(prof_rows, f, indent=1)


if __name__ == "__main__":
    main()
