#!/usr/bin/env python
"""bench_orb_batch.py -- ORB features of B KITTI-size frames held as CUDA tensors: per-frame calls against one batched call.

For B in {1, 8, 32}: B synthetic 1242x375 gray frames (synth.make_frame, seeds 0..B-1), held on the GPU as u8 CUDA tensors, get their ORB
keypoints and descriptors (3 000 features, scale 1.2, 8 levels, FAST 20 / 7) two ways, alternated step by step in one process:
  (a) per frame: B x (Frame.upload_tensors + Frame.orb_extract + Frame.orb_describe), the same kernels one frame per call, results in host memory
  (b) batched:   one OrbExtractor.extract call, everything on the device, results in CUDA tensors
Reported per B: wall time per frame of each arm (host clock per step; every step ends in a device synchronise), the device time of (b)
from CUDA events, kernel launches, host synchronises and the largest kernels' device time per step of B frames of each arm (torch.profiler,
a separate pass), and whether the two arms return the same keypoints and descriptors (they must).  The GPU name and power limit are read
in the same run.

  python bench_orb_batch.py [--steps 20] [--warmup 3] [--batches 1,8,32] [--profile-steps 2]
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

ORB = dict(n_features=3000, scale_factor=1.2, n_levels=8, ini_th_fast=20, min_th_fast=7)
W, H = 1242, 375


def arm_a(F, frames):
    out = []
    for t in frames:
        F.upload_tensors(image=t)
        r = F.orb_extract(nfeatures=ORB["n_features"], scale=ORB["scale_factor"], nlevels=ORB["n_levels"], ini_th=ORB["ini_th_fast"],
                          min_th=ORB["min_th_fast"])
        r["descriptors"] = F.orb_describe(len(r["x"]))
        out.append(r)
    return out


def arm_b(ex, batch, out):
    return ex.extract(batch, out=out)


def same(ra, rb) -> bool:
    for i, a in enumerate(ra):
        n = int(rb["count"][i])
        if n != len(a["x"]) or int(rb["status"][i]) != 0 or rb["n_candidates"][i].tolist() != a["n_candidates"]:
            return False
        for k in ("x", "y", "octave", "response", "angle", "size", "descriptors"):
            if not np.array_equal(rb[k][i, :n].cpu().numpy(), a[k]):
                return False
    return True


def _profile(fn, calls: int):
    """(kernel records, host synchronise count) of `calls` calls of fn in one torch.profiler window closed by torch.cuda.synchronize"""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    ev = list(prof.events())
    kern = [e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    syncs = sum(1 for e in ev if e.device_type == torch.autograd.DeviceType.CPU and e.name.startswith("cuda") and "Synchronize" in e.name)
    return kern, syncs


def profile_counts(fn, calls: int) -> dict:
    """kernel launches and host synchronises (runtime calls named *Synchronize) per call, from torch.profiler's records; the synchronises of
    an empty window (the closing torch.cuda.synchronize and the profiler's own) are subtracted.  Device time per kernel name per call."""
    kern, syncs = _profile(fn, calls)
    _, base = _profile(lambda: None, calls)
    per_kernel = {}
    for e in kern:
        name = e.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0].split("::")[-1]
        per_kernel[name] = per_kernel.get(name, 0.0) + e.device_time_total / 1e3 / calls
    top = {k: round(v, 4) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1])[:8]}
    return {"kernel_launches_per_call": len(kern) / calls, "host_synchronises_per_call": (syncs - base) / calls, "kernel_ms_per_call": top}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--profile-steps", type=int, default=2)
    a = ap.parse_args()
    import torch
    from bench_device_input import gpu_info
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_frame
    if not torch.cuda.is_available():
        raise SystemExit("bench_orb_batch.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    batches = [int(b) for b in a.batches.split(",")]
    held = torch.from_numpy(np.stack([make_frame(s)["gray"] for s in range(max(batches))])).to(dev)
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    F = capi.Frame(ctx, W, H)
    results = []
    for B in batches:
        frames, batch = list(held[:B].unbind(0)), held[:B]
        ex = capi.OrbExtractor(ctx, W, H, B, **ORB)
        out = ex.empty_outputs(B)
        t_a = t_b = 0.0
        ok = True
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dev_ms = []
        for step in range(a.warmup + a.steps):
            for arm in (("a", "b") if step % 2 == 0 else ("b", "a")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "a":
                    ra = arm_a(F, frames)
                else:
                    ev0.record()
                    rb = arm_b(ex, batch, out)
                    ev1.record()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if step >= a.warmup:
                    if arm == "a":
                        t_a += dt
                    else:
                        t_b += dt
                        dev_ms.append(ev0.elapsed_time(ev1))
            if step == a.warmup:
                ok = ok and same(ra, rb)
        ok = ok and same(ra, rb)
        pa = profile_counts(lambda: arm_a(F, frames), a.profile_steps)
        pb = profile_counts(lambda: arm_b(ex, batch, out), a.profile_steps)
        results.append({
            "B": B,
            "per_frame_ms_per_frame": 1e3 * t_a / (a.steps * B), "batched_ms_per_frame": 1e3 * t_b / (a.steps * B),
            "batched_device_ms_per_call": float(np.median(dev_ms)), "batched_device_ms_per_call_min": float(np.min(dev_ms)),
            "per_frame_launches_per_call": pa["kernel_launches_per_call"], "batched_launches_per_call": pb["kernel_launches_per_call"],
            "per_frame_host_syncs_per_call": pa["host_synchronises_per_call"], "batched_host_syncs_per_call": pb["host_synchronises_per_call"],
            "batched_kernel_ms_per_call": pb["kernel_ms_per_call"],
            "capacity_per_frame": ex.capacity, "device_bytes": ex.info()["device_bytes"],
            "identical_outputs": ok,
        })
        ex.close()
    print(json.dumps({
        "workload": f"ORB of B x 1242x375 u8 CUDA tensors, {ORB}, {a.steps} timed steps after {a.warmup} warm-up, arms alternated",
        "gpu": gpu_info(0),
        "results": results,
    }))
    bad = [r["B"] for r in results if not r["identical_outputs"]]
    if bad:
        raise SystemExit(f"the two arms disagree at B = {bad}")


if __name__ == "__main__":
    main()
