#!/usr/bin/env python
"""bench_window_batch.py -- the windowed optimisations (PartialBatchOptimization) of several config-3 sequences, one by one or batched.

Graph level: the window graphs of B config-3 trackers (1242x375, 3 000 ORB features, seeds 0..B-1, WINDOW 20 / OVERLAP 4), taken with
graph_export(0) after the 20 frames that end in the first window (f_id 19) -- the exact graphs the trackers solve there.  For B in
{1, 2, 4, 8, 16} they are solved (a) one by one with BatchGraph.optimize and (b) with one capi.optimize_batch, the two arms alternated
rep by rep from the same initial estimates (BatchGraph.reset).  Reported per B: ms per window of each arm (host clock around calls that
end in a device synchronise), kernel launches per call, and the largest estimate difference between the arms.

Tracker level: B config-3 sequences through capi.track_tensors_batch over --frames frames (windows fire at f_id 19 and 35): the wall
clock of the steps on which the windows fire against the other steps, and the windowed_ba stage (stage_ms[8]).  --tracker-only runs this
part alone.

The GPU name and power limit are read in the same run.

  python bench_window_batch.py [--batches 1,2,4,8,16] [--reps 10] [--frames 40] [--tracker-batch 8] [--tracker-only]
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

KW = dict(max_iterations=100, gain_threshold=1e-3)      # PartialBatchOptimization's cap and gain threshold (src/Optimizer.cc:230)


def _held(frames, dev):
    import torch
    return [(torch.from_numpy(f["gray"]).to(dev), torch.from_numpy(f["depth_raw"]).to(dev), torch.from_numpy(f["flow"]).to(dev),
             torch.from_numpy(f["mask"]).to(dev)) for f in frames]


def window_graphs(ctx, held, ids):
    """the window graph each sequence's tracker solves at f_id 19: tracked with the windowed optimisation off, so graph_export(0) sees the
    map that optimisation would start from"""
    from vdo_slam_b200 import capi
    out = []
    for h, i in zip(held, ids):
        tr = capi.Tracker(ctx, n_features=3000, local_batch=0)
        for t in range(20):
            tr.track_tensors(*h[t], i[t], writeback=False)
        out.append(tr.graph_export(0))
    return out


def graph_level(ctx, graphs, batches, reps):
    from vdo_slam_b200 import capi
    res = []
    for B in batches:
        Ga = [capi.BatchGraph(ctx, g) for g in graphs[:B]]
        Gb = [capi.BatchGraph(ctx, g) for g in graphs[:B]]
        info = [G.solver_info()["dense"] for G in Ga]
        t_a = t_b = 0.0
        la = lb = 0
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
            la, lb = sum(r["kernel_launches"] for r in ra), rb[0]["kernel_launches"]
            for A, Bg in zip(Ga, Gb):
                (sa, pa), (sb, pb) = A.vertices(), Bg.vertices()
                dmax = max(dmax, float(np.abs(sa - sb).max()), float(np.abs(pa - pb).max()))
        res.append({
            "B": B, "dense_path": sum(info),
            "points": [int(len(g["pt"])) for g in graphs[:B]] if B <= 4 else [int(min(len(g["pt"]) for g in graphs[:B])), int(max(len(g["pt"]) for g in graphs[:B]))],
            "lm_iterations": [r["iterations"] for r in ra], "trials": [r["trials"] for r in ra],
            "separate_ms_per_window": round(1e3 * t_a / reps / B, 4), "batched_ms_per_window": round(1e3 * t_b / reps / B, 4),
            "separate_launches": la, "batched_launches": lb,
            "max_abs_estimate_diff": dmax,
        })
    return res


def tracker_level(ctx, held, ids, B, frames, warmup=4):
    """per-step wall clock of every track_tensors_batch call; the steps on which the windows fire (f_id 19 and 35 for WINDOW 20 /
    OVERLAP 4) against the other steps after the warm-up.  stage_ms[8] is reported summed over the trackers and as its largest entry:
    solved tracker by tracker, the step spends the sum; solved as one batched stage, every tracker records the whole stage."""
    from vdo_slam_b200 import capi
    trs = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
    step_ms, fired = [], []
    for t in range(frames):
        runs0 = int(trs[0].get("local_ba")[0])
        t0 = time.perf_counter()
        capi.track_tensors_batch(trs, [held[i][t][0] for i in range(B)], [held[i][t][1] for i in range(B)], [held[i][t][2] for i in range(B)],
                                 [held[i][t][3] for i in range(B)], [ids[i][t] for i in range(B)], writeback=False)
        step_ms.append(1e3 * (time.perf_counter() - t0))
        fired.append(int(trs[0].get("local_ba")[0]) > runs0)
    st = np.array([tr.get("stage_ms")[8] for tr in trs], np.float64)
    win = [m for m, f in zip(step_ms, fired) if f]
    rest = [m for t, (m, f) in enumerate(zip(step_ms, fired)) if not f and t >= warmup]
    return {
        "B": B, "frames": frames, "window_steps": [t for t, f in enumerate(fired) if f],
        "windows_per_tracker": [int(tr.get("local_ba")[0]) for tr in trs],
        "window_step_ms": [round(m, 3) for m in win], "other_step_ms_mean": round(float(np.mean(rest)), 3),
        "windowed_ba_stage_ms_sum": round(float(st.sum()), 3), "windowed_ba_stage_ms_max": round(float(st.max()), 3),
        "final_Tcw": [tr.get("Tcw").tolist() for tr in trs],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,4,8,16")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--tracker-batch", type=int, default=8)
    ap.add_argument("--tracker-only", action="store_true")
    a = ap.parse_args()
    import torch
    from bench import sequence_frames
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_window_batch.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    batches = [int(b) for b in a.batches.split(",")]
    n_seq = max(a.tracker_batch, 0 if a.tracker_only else max(batches))
    n_frames = max(a.frames, 20)
    seqs = [sequence_frames(n_frames, seed) for seed in range(n_seq)]
    held = [_held(s, dev) for s in seqs]
    ids = [[f["obj_ids"] for f in s] for s in seqs]
    del seqs
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    out = {"gpu": gpu_info(0)}
    if not a.tracker_only:
        graphs = window_graphs(ctx, held[:max(batches)], ids)
        out["graph_workload"] = (f"window graphs (WINDOW 20, static points only) of config-3 trackers at f_id 19, seeds 0..B-1; {a.reps} reps per arm "
                                 f"after one warm-up, arms alternated")
        out["graph_level"] = graph_level(ctx, graphs, batches, a.reps)
    out["tracker_workload"] = f"{a.tracker_batch} config-3 sequences (seeds 0..{a.tracker_batch - 1}) through track_tensors_batch, {a.frames} frames"
    out["tracker_level"] = tracker_level(ctx, held, ids, a.tracker_batch, a.frames)
    print(json.dumps(out))
    bad = [r["B"] for r in out.get("graph_level", []) if r["max_abs_estimate_diff"] > 1e-8]
    if bad:
        raise SystemExit(f"the two arms disagree at B = {bad}")


if __name__ == "__main__":
    main()
