#!/usr/bin/env python
"""bench_omd.py -- the OMD configuration (example/omd.yaml) with detected and with sampled background features.

For B in {1, 8}: B distinct synthetic OMD-shaped sequences (640x480, dataset = 1, the omd.yaml thresholds and windows, 3 000 ORB features;
the synthetic depth is disparity * 256, so DepthMapFactor is 256), held on the GPU as CUDA tensors, are tracked with one
capi.track_tensors_batch per step, once with use_sample_feature = 0 and once with 1 (seeds 1000 + i), the two arms alternated step by
step in one process.  Reported per B and arm: aggregate frames/s (host wall clock per step; every call ends in a device synchronise) and
the per-stage ms per step (stage_ms summed over the B trackers).  Also reported: the device time of the sampler launch (vdo_sample_keys,
CUDA events around the kernel, median of --sampler-reps calls) for 1 and 8 frames of 640x480.  The GPU name and power limit are read in
the same run.

  python bench_omd.py [--frames 40] [--warmup 4] [--batches 1,8] [--sampler-reps 50]
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
W, H = 640, 480
K = (618.3587036132812, 618.5924072265625, 328.9866333007812, 237.7507629394531)
OMD = dict(width=W, height=H, fx=K[0], fy=K[1], cx=K[2], cy=K[3], depth_factor=256.0, th_depth_bg=40.0, th_depth_obj=25.0, max_track_bg=1200,
           max_track_obj=800, sf_mg_thres=0.02, sf_ds_thres=0.99, n_features=3000, is_kitti=0, dataset=1, window_size=20, overlap_size=4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--sampler-reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_sequence_frame
    if not torch.cuda.is_available():
        raise SystemExit("bench_omd.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    batches = [int(b) for b in a.batches.split(",")]
    Bmax = max(batches)
    held, ids = [], []
    for s in range(Bmax):
        fr = [make_sequence_frame(t, seed=s, width=W, height=H, K=np.asarray(K, np.float32)) for t in range(a.frames)]
        held.append([tuple(torch.from_numpy(np.ascontiguousarray(f[k])).to(dev) for k in ("gray", "depth_raw", "flow", "mask")) for f in fr])
        ids.append([f["obj_ids"] for f in fr])
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    results = []
    for B in batches:
        arms = {s: [capi.Tracker(ctx, use_sample_feature=s, sample_seed=1000 + i, **OMD) for i in range(B)] for s in (0, 1)}
        wall = {0: 0.0, 1: 0.0}
        st0 = {}
        for t in range(a.frames):
            if t == a.warmup:
                st0 = {s: sum(tr.get("stage_ms") for tr in arms[s]) for s in (0, 1)}
                wall = {0: 0.0, 1: 0.0}
            for s in ((0, 1) if t % 2 == 0 else (1, 0)):
                t0 = time.perf_counter()
                capi.track_tensors_batch(arms[s], [held[i][t][0] for i in range(B)], [held[i][t][1] for i in range(B)], [held[i][t][2] for i in range(B)],
                                         [held[i][t][3] for i in range(B)], [ids[i][t] for i in range(B)], writeback=False)
                wall[s] += time.perf_counter() - t0
        steps = a.frames - a.warmup
        r = {"B": B}
        for s, name in ((0, "detected"), (1, "sampled")):
            st = (sum(tr.get("stage_ms") for tr in arms[s]) - st0[s]) / steps
            r[f"{name}_fps"] = B * steps / wall[s]
            r[f"{name}_ms_per_step"] = 1e3 * wall[s] / steps
            r[f"{name}_stage_ms_per_step"] = {k: round(float(v), 4) for k, v in zip(STAGES, st)}
            r[f"{name}_local_ba_runs"] = int(arms[s][0].get("local_ba")[0])
        results.append(r)
    sampler = {}
    for n in (1, 8):
        seeds = list(range(n))
        for _ in range(5):
            capi.sample_keys(ctx, seeds, W, H)
        ms = [capi.sample_keys(ctx, seeds, W, H)[2] for _ in range(a.sampler_reps)]
        sampler[f"frames_{n}_ms_median"] = float(np.median(ms))
        sampler[f"frames_{n}_ms_min"] = float(np.min(ms))
    out = {
        "workload": f"OMD-shaped x B: {a.frames} frames of 640x480 per sequence ({a.warmup} warm-up), omd.yaml thresholds, 3000 ORB features, seeds 0..B-1, "
                    "inputs held as CUDA tensors, one track_tensors_batch per step",
        "gpu": gpu_info(0),
        "results": results,
        "sampler_kernel": sampler,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
