#!/usr/bin/env python
"""bench_map_graph.py -- the windowed optimisation (PartialBatchOptimization) of config-3 trackers as their sequences grow.

Windows: B config-3 sequences (1242x375, 3 000 ORB features, seeds 0..B-1, WINDOW 20 / OVERLAP 4) through capi.track_tensors_batch over
--frames frames.  For every step on which the windows fire (f_id 19, 35, 51, ...) the windowed_ba stage of that step (the stage_ms[8]
increment of tracker 0; the stage is batched, so every tracker records the whole stage) and the step's wall clock; the aggregate frames/s
of all steps after --warmup.  A graph built from the whole history gets slower with f_id; one built from the tracklet tables kept per frame
does not.

--split: one sequence with the windowed optimisation off, stopped at the given f_ids: the time of one mode-0 graph build
(vdo_tracker_graph_export of one array, averaged over the 16 arrays) and of vdo_tracker_batch_optimize(0).  With VDO_PROFILE=1 set, the
library prints the build + ingest and finalize phases of the same calls on stderr.

The GPU name and power limit are read in the same run.

  python bench_map_graph.py [--frames 154] [--batches 1,8] [--warmup 4] [--split 19,35,51,99,147]
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
GRAPH_ARRAYS = 16


def _held(frames, dev):
    import torch
    return [(torch.from_numpy(f["gray"]).to(dev), torch.from_numpy(f["depth_raw"]).to(dev), torch.from_numpy(f["flow"]).to(dev),
             torch.from_numpy(f["mask"]).to(dev), f["obj_ids"]) for f in frames]


def windows(ctx, held, B, frames, warmup):
    from vdo_slam_b200 import capi
    trs = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
    per_window, step_ms = {}, []
    for t in range(frames):
        runs0, st0 = int(trs[0].get("local_ba")[0]), float(trs[0].get("stage_ms")[8])
        t0 = time.perf_counter()
        capi.track_tensors_batch(trs, [held[i][t][0] for i in range(B)], [held[i][t][1] for i in range(B)], [held[i][t][2] for i in range(B)],
                                 [held[i][t][3] for i in range(B)], [held[i][t][4] for i in range(B)], writeback=False)
        step_ms.append(1e3 * (time.perf_counter() - t0))
        if int(trs[0].get("local_ba")[0]) > runs0:
            per_window[t] = {"windowed_ba_ms": round(float(trs[0].get("stage_ms")[8]) - st0, 3), "step_ms": round(step_ms[-1], 3)}
    timed = sum(step_ms[warmup:]) / 1e3
    return {"B": B, "frames": frames, "per_window": per_window, "frames_per_s_aggregate": round(B * (frames - warmup) / timed, 3),
            "windowed_ba_stage_ms_total": round(float(trs[0].get("stage_ms")[8]), 3)}


def split(ctx, held, stops):
    from vdo_slam_b200 import capi
    tr = capi.Tracker(ctx, n_features=3000, local_batch=0)
    out = {}
    t = 0
    for stop in stops:
        while t <= stop:
            tr.track_tensors(*held[t][:4], held[t][4], writeback=False)
            t += 1
        tr.graph_export(0)                                                 # warm
        t0 = time.perf_counter()
        g = tr.graph_export(0)
        build = 1e3 * (time.perf_counter() - t0) / GRAPH_ARRAYS
        sys.stderr.write(f"[bench_map_graph] f_id {stop}: batch_optimize(0)\n")
        sys.stderr.flush()
        t0 = time.perf_counter()
        tr.batch_optimize(0)
        out[stop] = {"graph_build_ms": round(build, 3), "batch_optimize_ms": round(1e3 * (time.perf_counter() - t0), 3), "points": int(len(g["pt"])),
                     "observations": int(len(g["obs_w"]))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=154)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--split", default="")
    a = ap.parse_args()
    import torch
    from bench import sequence_frames
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_map_graph.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    stops = [int(s) for s in a.split.split(",") if s]
    batches = [int(b) for b in a.batches.split(",") if b]
    n_seq = max(batches + [1])
    n_frames = max([a.frames] + [s + 1 for s in stops])
    held = []
    for seed in range(n_seq):
        held.append(_held(sequence_frames(n_frames, seed), dev))
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    out = {"gpu": gpu_info(0), "workload": f"config-3 sequences (seeds 0..B-1), {n_frames} frames, WINDOW 20 / OVERLAP 4, track_tensors_batch"}
    if stops:
        out["split"] = split(ctx, held[0], stops)
    out["windows"] = [windows(ctx, held, B, a.frames, a.warmup) for B in batches]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
