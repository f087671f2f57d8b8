#!/usr/bin/env python
"""bench_mixed_sequences.py -- sequences of two image sizes and ORB settings tracked in one mixed call, per geometry group, or one by one.

For B in {2, 4, 8}: B/2 KITTI-shaped sequences (1242x375, 2 500 ORB features, option I) and B/2 OMD-shaped ones (640x480, 3 000 ORB
features, sampled background features), synthetic and held on the GPU as CUDA tensors (u8 gray, f32 raw depth, (H,W,2) f32 flow, i32
mask), are tracked three ways, the order of the arms rotated step by step in one process:
  (a) mixed:    one capi.track_tensors_mixed call per step over all B trackers
  (b) grouped:  one capi.track_tensors_batch call per geometry per step (two calls)
  (c) separate: B Tracker.track_tensors calls per step
Reported per B: aggregate frames/s of each arm (host wall clock per step; every call ends in a device synchronise), kernel launches per
step of each arm (a separate torch.profiler pass, counted as bench_multi_sequence.py counts them), and the largest pose difference between
the arms (must be 0).  The GPU name and power limit are read in the same run.

  python bench_mixed_sequences.py [--frames 40] [--warmup 4] [--batches 2,4,8] [--profile-steps 2]
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

OMD_K = (618.3587036132812, 618.5924072265625, 328.9866333007812, 237.7507629394531)
KITTI = dict(n_features=2500)
OMD = dict(width=640, height=480, fx=OMD_K[0], fy=OMD_K[1], cx=OMD_K[2], cy=OMD_K[3], n_features=3000, use_sample_feature=1, is_kitti=0, dataset=1,
           sf_mg_thres=0.02, sf_ds_thres=0.99)
ARMS = ("mixed", "grouped", "separate")


def _omd_frame(args):
    from vdo_slam_b200.synth import make_sequence_frame
    return make_sequence_frame(args[0], seed=args[1], width=640, height=480, K=OMD_K)


def omd_frames(n_frames, seed):
    import multiprocessing as mp
    jobs = [(t, seed) for t in range(n_frames)]
    with mp.get_context("fork").Pool(min(32, os.cpu_count() or 1)) as pool:
        return pool.map(_omd_frame, jobs)


def _held(frames, dev):
    import torch
    return [(torch.from_numpy(f["gray"]).to(dev), torch.from_numpy(f["depth_raw"]).to(dev), torch.from_numpy(f["flow"]).to(dev),
             torch.from_numpy(f["mask"]).to(dev)) for f in frames]


def make_trackers(ctx, B):
    """trackers 0 .. B/2 - 1 KITTI-shaped, the rest OMD-shaped"""
    from vdo_slam_b200 import capi
    return [capi.Tracker(ctx, **(KITTI if i < B // 2 else OMD)) for i in range(B)]


def _planes(held, t, idx):
    return [[held[i][t][k] for i in idx] for k in range(4)]


def step(arm, trs, held, ids, t):
    from vdo_slam_b200 import capi
    B = len(trs)
    if arm == "mixed":
        return capi.track_tensors_mixed(trs, *_planes(held, t, range(B)), [ids[i][t] for i in range(B)], writeback=False)
    if arm == "grouped":
        T = np.zeros((B, 4, 4), np.float32)
        for g in (range(B // 2), range(B // 2, B)):
            T[list(g)] = capi.track_tensors_batch([trs[i] for i in g], *_planes(held, t, g), [ids[i][t] for i in g], writeback=False)
        return T
    return np.stack([tr.track_tensors(*held[i][t], ids[i][t], writeback=False) for i, tr in enumerate(trs)])


def launches_per_step(ctx, held, ids, B, steps):
    """kernel launches per step of each arm, counted from torch.profiler's CUDA kernel records after 3 unprofiled steps"""
    import torch
    out = {}
    for arm in ARMS:
        trs = make_trackers(ctx, B)
        for t in range(3):
            step(arm, trs, held, ids, t)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for t in range(3, 3 + steps):
                step(arm, trs, held, ids, t)
            torch.cuda.synchronize()
        n = sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in ev.name.lower()
                and "memset" not in ev.name.lower())
        out[arm] = n / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batches", default="2,4,8")
    ap.add_argument("--profile-steps", type=int, default=2)
    a = ap.parse_args()
    import torch
    from bench import sequence_frames
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_sequences.py needs a CUDA device (there is no CPU path)")
    batches = [int(b) for b in a.batches.split(",")]
    if any(b < 2 or b % 2 for b in batches):
        raise SystemExit("--batches: every B must be even and at least 2 (half KITTI-shaped, half OMD-shaped)")
    dev = torch.device("cuda", 0)
    half = max(batches) // 2
    seqs = [sequence_frames(a.frames, s) for s in range(half)] + [omd_frames(a.frames, s) for s in range(half)]
    held_all = [_held(s, dev) for s in seqs]
    ids_all = [[f["obj_ids"] for f in s] for s in seqs]
    del seqs
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    results = []
    for B in batches:
        pick = list(range(B // 2)) + list(range(half, half + B // 2))      # B/2 KITTI-shaped, then B/2 OMD-shaped
        held, ids = [held_all[i] for i in pick], [ids_all[i] for i in pick]
        trs = {arm: make_trackers(ctx, B) for arm in ARMS}
        secs = dict.fromkeys(ARMS, 0.0)
        dpose = 0.0
        for t in range(a.frames):
            if t == a.warmup:
                secs = dict.fromkeys(ARMS, 0.0)
            T = {}
            order = ARMS[t % 3:] + ARMS[:t % 3]
            for arm in order:
                t0 = time.perf_counter()
                T[arm] = step(arm, trs[arm], held, ids, t)
                secs[arm] += time.perf_counter() - t0
            dpose = max(dpose, float(np.abs(T["mixed"] - T["grouped"]).max()), float(np.abs(T["mixed"] - T["separate"]).max()))
        steps = a.frames - a.warmup
        launches = launches_per_step(ctx, held, ids, B, a.profile_steps)
        r = {"B": B, "max_abs_pose_diff": dpose}
        for arm in ARMS:
            r[f"{arm}_fps"] = B * steps / secs[arm]
            r[f"{arm}_ms_per_step"] = 1e3 * secs[arm] / steps
            r[f"{arm}_launches_per_step"] = launches[arm]
        results.append(r)
    out = {
        "workload": (f"B/2 KITTI-shaped (1242x375, 2500 ORB features) + B/2 OMD-shaped (640x480, 3000 ORB features, UseSampleFeature 1) synthetic "
                     f"sequences, {a.frames} frames each ({a.warmup} warm-up), inputs held as CUDA tensors"),
        "gpu": gpu_info(0),
        "results": results,
    }
    print(json.dumps(out))
    bad = [r["B"] for r in results if r["max_abs_pose_diff"] != 0.0]
    if bad:
        raise SystemExit(f"the arms disagree at B = {bad}")


if __name__ == "__main__":
    main()
