#!/usr/bin/env python
"""bench_multi_sequence.py -- several config-3 sequences tracked one after another or as one batch.

For B in {1, 2, 4, 8}: B distinct synthetic config-3 sequences (1242x375, 3 000 ORB features, seeds 0..B-1), held on the GPU as CUDA tensors
(u8 gray, f32 raw depth, (H,W,2) f32 flow, i32 mask), are tracked two ways, alternated step by step in one process:
  (a) separate: B trackers, Tracker.track_tensors called once per tracker per step
  (b) batched:  B trackers, one capi.track_tensors_batch per step
Reported per B: aggregate frames/s of each arm (host wall clock per step; every call ends in a device synchronise), per-stage ms per step
(stage_ms summed over the B trackers), kernel launches per step of each arm (a separate torch.profiler pass), and the largest pose
difference between the arms (must be 0).  The GPU name and power limit are read in the same run.

  python bench_multi_sequence.py [--frames 64] [--warmup 4] [--batches 1,2,4,8] [--profile-steps 2]
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

STAGES = ("ingest+depth", "update_mask", "frame_build", "look_ups", "camera_model", "camera_lm", "objects", "renewal", "windowed_ba")


def _held(frames, dev):
    import torch
    return [(torch.from_numpy(f["gray"]).to(dev), torch.from_numpy(f["depth_raw"]).to(dev), torch.from_numpy(f["flow"]).to(dev),
             torch.from_numpy(f["mask"]).to(dev)) for f in frames]


def _step_a(trs, held, ids, t):
    return np.stack([tr.track_tensors(*held[i][t], ids[i][t], writeback=False) for i, tr in enumerate(trs)])


def _step_b(trs, held, ids, t):
    from vdo_slam_b200 import capi
    B = len(trs)
    return capi.track_tensors_batch(trs, [held[i][t][0] for i in range(B)], [held[i][t][1] for i in range(B)], [held[i][t][2] for i in range(B)],
                                    [held[i][t][3] for i in range(B)], [ids[i][t] for i in range(B)], writeback=False)


def launches_per_step(ctx, held, ids, B, steps):
    """kernel launches per step of each arm, counted from torch.profiler's CUDA kernel records after 3 unprofiled steps"""
    import torch
    from vdo_slam_b200 import capi
    out = {}
    for arm, fn in (("separate", _step_a), ("batched", _step_b)):
        trs = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
        for t in range(3):
            fn(trs, held, ids, t)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for t in range(3, 3 + steps):
                fn(trs, held, ids, t)
            torch.cuda.synchronize()
        n = sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in ev.name.lower()
                and "memset" not in ev.name.lower())
        out[arm] = n / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--profile-steps", type=int, default=2)
    a = ap.parse_args()
    import torch
    from bench import sequence_frames
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_sequence.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    batches = [int(b) for b in a.batches.split(",")]
    Bmax = max(batches)
    seqs = [sequence_frames(a.frames, seed) for seed in range(Bmax)]
    held = [_held(s, dev) for s in seqs]
    ids = [[f["obj_ids"] for f in s] for s in seqs]
    del seqs
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    results = []
    for B in batches:
        tr_a = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
        tr_b = [capi.Tracker(ctx, n_features=3000) for _ in range(B)]
        t_a = t_b = 0.0
        dpose = 0.0
        st_a = st_b = None
        for t in range(a.frames):
            if t == a.warmup:
                st_a = sum(tr.get("stage_ms") for tr in tr_a)
                st_b = sum(tr.get("stage_ms") for tr in tr_b)
                t_a = t_b = 0.0
            T = {}
            for arm in (("a", "b") if t % 2 == 0 else ("b", "a")):
                t0 = time.perf_counter()
                T[arm] = _step_a(tr_a, held[:B], ids, t) if arm == "a" else _step_b(tr_b, held[:B], ids, t)
                dt = time.perf_counter() - t0
                if arm == "a":
                    t_a += dt
                else:
                    t_b += dt
            dpose = max(dpose, float(np.abs(T["a"] - T["b"]).max()))
        steps = a.frames - a.warmup
        sa = (sum(tr.get("stage_ms") for tr in tr_a) - st_a) / steps
        sb = (sum(tr.get("stage_ms") for tr in tr_b) - st_b) / steps
        launches = launches_per_step(ctx, held[:B], ids, B, a.profile_steps)
        results.append({
            "B": B,
            "separate_fps": B * steps / t_a, "batched_fps": B * steps / t_b,
            "separate_ms_per_step": 1e3 * t_a / steps, "batched_ms_per_step": 1e3 * t_b / steps,
            "separate_stage_ms_per_step": {k: round(float(v), 4) for k, v in zip(STAGES, sa)},
            "batched_stage_ms_per_step": {k: round(float(v), 4) for k, v in zip(STAGES, sb)},
            "separate_launches_per_step": launches["separate"], "batched_launches_per_step": launches["batched"],
            "max_abs_pose_diff": dpose,
        })
    out = {
        "workload": f"config3 x B: {a.frames} frames of 1242x375 per sequence ({a.warmup} warm-up), 3000 ORB features, seeds 0..B-1, inputs held as CUDA tensors",
        "gpu": gpu_info(0),
        "results": results,
    }
    print(json.dumps(out))
    bad = [r["B"] for r in results if r["max_abs_pose_diff"] != 0.0]
    if bad:
        raise SystemExit(f"the two arms disagree at B = {bad}")


if __name__ == "__main__":
    main()
