#!/usr/bin/env python
"""bench_full_batch.py -- full-batch optimisations (FullBatchOptimization) of several graphs / sequences, one by one or in one call.

Graph level, two workloads:
  * config 3: the full-batch graphs of B config-3 sequences (1242x375, 3 000 ORB features, seeds 0..B-1, --frames frames each), taken
    with graph_export(1) at the end of the sequence -- the graphs the trackers' batch_optimize(1) solves;
  * config 4: config-4-shaped synthetic graphs (synth.make_batch_graph, 200 frames, 5 objects, 40 000 static and 10 000 dynamic points),
    seeds 4..4+B-1.
For B in {1, 2, 4, 8} they are solved (a) one by one with BatchGraph.optimize and (b) with one capi.optimize_batch, the arms alternated rep
by rep from the same initial estimates (BatchGraph.reset).  Reported per B: ms per graph of each arm (host clock around calls that end in a
device synchronise), kernel launches per call, host synchronises per call (cudaStreamSynchronize / cudaEventSynchronize records of one
torch.profiler pass per arm), and the largest estimate difference between the arms.

Tracker level: the B config-3 trackers, twice: Tracker.batch_optimize(1) one tracker after another against one
capi.batch_optimize_trackers(trackers, 1), alternated, and the largest map difference.  With VDO_PROFILE=1 the library prints the build /
ingest + finalize / optimise split of every call to stderr.  The GPU name and power limit are read in the same run.

  python bench_full_batch.py [--batches 1,2,4,8] [--frames 154] [--reps 3] [--reps4 2] [--skip-config4]
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

KW = dict(max_iterations=300, gain_threshold=1e-4)      # FullBatchOptimization's cap and gain threshold (src/Optimizer.cc:1330-1335)
CONFIG4 = dict(n_frames=200, n_objects=5, n_static=40000, n_dynamic=10000)


def track_sequences(ctx, B, frames):
    """B config-3 sequences (seeds 0..B-1) tracked to their end, twice (two identical tracker sets)"""
    import torch
    from bench import sequence_frames
    from vdo_slam_b200 import capi
    dev = torch.device("cuda", 0)
    sets = [[capi.Tracker(ctx, n_features=3000) for _ in range(B)] for _ in range(2)]
    for s in range(B):
        seq = sequence_frames(frames, s)
        for f in seq:
            ins = [torch.from_numpy(f[k]).to(dev) for k in ("gray", "depth_raw", "flow", "mask")]
            for trs in sets:
                trs[s].track_tensors(*ins, f["obj_ids"], writeback=False)
    return sets


def _syncs(fn):
    """host synchronises of one call of fn, from the CUDA runtime records of torch.profiler"""
    import torch
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
    names = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize")
    return sum(1 for e in prof.events() if e.name in names)


def graph_level(ctx, graphs, batches, reps):
    from vdo_slam_b200 import capi
    res = []
    for B in batches:
        Ga = [capi.BatchGraph(ctx, g) for g in graphs[:B]]
        Gb = [capi.BatchGraph(ctx, g) for g in graphs[:B]]
        t_a = t_b = 0.0
        dmax = 0.0
        for rep in range(reps + 1):                      # rep 0 warms up
            ms = {}
            for arm in (("a", "b") if rep % 2 == 0 else ("b", "a")):
                for G in (Ga if arm == "a" else Gb):
                    G.reset()
                t0 = time.perf_counter()
                if arm == "a":
                    ra = [G.optimize(**KW) for G in Ga]
                else:
                    rb = capi.optimize_batch(Gb, **KW)
                ms[arm] = time.perf_counter() - t0
            if rep:
                t_a += ms["a"]; t_b += ms["b"]
            for A, Bg in zip(Ga, Gb):
                (sa, pa), (sb, pb) = A.vertices(), Bg.vertices()
                dmax = max(dmax, float(np.abs(sa - sb).max()), float(np.abs(pa - pb).max()))
        for G in Ga + Gb:
            G.reset()
        sync_a = _syncs(lambda: [G.optimize(**KW) for G in Ga])
        sync_b = _syncs(lambda: capi.optimize_batch(Gb, **KW))
        res.append({
            "B": B, "points": [int(len(g["pt"])) for g in graphs[:B]], "pcg_path": [1 - G.solver_info()["dense"] for G in Ga],
            "lm_iterations": [r["iterations"] for r in ra], "pcg_iterations": [r["pcg_iterations"] for r in ra],
            "batched_lm_iterations": [r["iterations"] for r in rb], "batched_pcg_iterations": [r["pcg_iterations"] for r in rb],
            "separate_ms_per_graph": round(1e3 * t_a / reps / B, 3), "batched_ms_per_graph": round(1e3 * t_b / reps / B, 3),
            "separate_launches": sum(r["kernel_launches"] for r in ra), "batched_launches": rb[0]["kernel_launches"],
            "separate_syncs": sync_a, "batched_syncs": sync_b,
            "max_abs_estimate_diff": dmax,
        })
    return res


def tracker_level(ctx, sets, reps):
    from vdo_slam_b200 import capi
    A, Bs = sets
    t_a = t_b = 0.0
    for rep in range(reps):
        for arm in (("a", "b") if rep % 2 == 0 else ("b", "a")):
            t0 = time.perf_counter()
            if arm == "a":
                for t in A:
                    t.batch_optimize(1)
            else:
                capi.batch_optimize_trackers(Bs, 1)
            if arm == "a":
                t_a += time.perf_counter() - t0
            else:
                t_b += time.perf_counter() - t0
    dmax = 0.0
    for x, y in zip(A, Bs):
        for k in ("vmCameraPose_RF", "vmRigidMotion_RF", "vp3DPointSta", "vp3DPointDyn"):
            a, b = x.map_get(k), y.map_get(k)
            dmax = max(dmax, float(np.abs(a - b).max()) if a.size else 0.0)
    B = len(A)
    return {"B": B, "loop_ms_per_tracker": round(1e3 * t_a / reps / B, 3), "batched_ms_per_tracker": round(1e3 * t_b / reps / B, 3),
            "max_abs_map_diff": dmax}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=154)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reps4", type=int, default=2)
    ap.add_argument("--skip-config4", action="store_true")
    a = ap.parse_args()
    import torch
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_batch_graph
    if not torch.cuda.is_available():
        raise SystemExit("bench_full_batch.py needs a CUDA device (there is no CPU path)")
    batches = [int(b) for b in a.batches.split(",")]
    ctx = capi.Context(0)
    out = {"gpu": gpu_info(0)}
    sets = track_sequences(ctx, max(batches), a.frames)
    graphs3 = [t.graph_export(1) for t in sets[0]]
    out["config3_workload"] = f"full-batch graphs of config-3 sequences after {a.frames} frames, seeds 0..B-1; {a.reps} reps per arm after one warm-up"
    out["config3"] = graph_level(ctx, graphs3, batches, a.reps)
    if not a.skip_config4:
        graphs4 = [make_batch_graph(seed=4 + s, **CONFIG4) for s in range(max(batches))]
        out["config4_workload"] = f"config-4-shaped graphs {CONFIG4}, seeds 4..; {a.reps4} reps per arm after one warm-up"
        out["config4"] = graph_level(ctx, graphs4, batches, a.reps4)
        del graphs4
    out["tracker_level"] = [tracker_level(ctx, [s[:B] for s in sets], a.reps) for B in batches]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
