#!/usr/bin/env python
"""bench_device_input.py -- what device-resident frame input saves a PyTorch pipeline on the config-3 sequence.

The frames are held on the GPU in the form flow / segmentation networks hand them over: BGR HWC u8 colour (synth.colour_from_gray of the
sequence's gray), f32 raw depth, (2,H,W) f32 flow, int64 mask.  Two trackers run the same 154 frames of 1242x375 (3 000 ORB features), alternating frame by frame:
  (a) host route:   .cpu() of the four tensors, cv2.cvtColor, Tracker.track with write-back into the host arrays
  (b) device route: Tracker.track_tensors with write-back into the tensors
Reported: frames/s of each (host wall clock per call, every call ends in a device synchronise), their per-frame stage_ms[0] (upload +
depth prep) and stage_ms[1] (UpdateMask + write-back), the device time of k_ingest_frame over repeated Frame.upload_tensors (CUDA
kernel records of torch.profiler), the largest pose difference between the routes (must be 0), and the GPU name and power limit.

  python bench_device_input.py [--frames 154] [--warmup 3] [--ingest-reps 200]
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


def gpu_info(index: int = 0) -> dict:
    import torch
    out = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)], capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:                       # reported as unknown, never guessed
        out["power_limit_error"] = str(e)
    return out


def ingest_kernel_ms(ctx, held, reps: int):
    """k_ingest_frame over `reps` Frame.upload_tensors calls cycling through the held frames (16 frames of inputs, 200 MB, do not fit the 50 MB
    L2): mean kernel time from the CUDA kernel records of torch.profiler (None if it saw no launch), launches seen, and the mean host
    wall-clock time of one upload_tensors call (check + launch + synchronise) measured without the profiler"""
    import torch
    from vdo_slam_b200 import capi
    H, W = held[0][1].shape
    F = capi.Frame(ctx, W, H)
    ring = held[:16]
    for img, d, fl, m in ring:
        F.upload_tensors(image=img, depth=d, flow=fl, mask=m, rgb=False)
    t0 = time.perf_counter()
    for i in range(reps):
        img, d, fl, m = ring[i % len(ring)]
        F.upload_tensors(image=img, depth=d, flow=fl, mask=m, rgb=False)
    wall = (time.perf_counter() - t0) / reps
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(reps):
            img, d, fl, m = ring[i % len(ring)]
            F.upload_tensors(image=img, depth=d, flow=fl, mask=m, rgb=False)
    us, n = 0.0, 0
    for ev in prof.key_averages():
        if "k_ingest_frame" in ev.key:
            us += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            n += ev.count
    F.close()
    return (us / n / 1e3 if n else None), n, wall * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=154)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ingest-reps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import cv2
    import torch
    from bench import sequence_frames
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import colour_from_gray
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_input.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    frames = sequence_frames(a.frames, a.seed)
    bgr = [colour_from_gray(f["gray"], seed=t) for t, f in enumerate(frames)]
    H, W = frames[0]["gray"].shape
    held = []                                    # what a network pipeline would hand over, resident on the GPU
    for f, c in zip(frames, bgr):
        held.append((torch.from_numpy(c).to(dev), torch.from_numpy(f["depth_raw"]).to(dev), torch.from_numpy(f["flow"]).to(dev).permute(2, 0, 1).contiguous(),
                     torch.from_numpy(f["mask"]).to(dev).to(torch.int64)))
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    tr_a, tr_b = capi.Tracker(ctx, n_features=3000), capi.Tracker(ctx, n_features=3000)
    t_a, t_b, dpose = [], [], 0.0
    st_a = st_b = None
    for t, (f, (img, d, fl, m)) in enumerate(zip(frames, held)):
        if t == a.warmup:
            st_a, st_b = tr_a.get("stage_ms").copy(), tr_b.get("stage_ms").copy()
        d_b, m_b = d.clone(), m.clone()          # route (b) writes back into its tensors; (a) must read the untouched ones
        torch.cuda.synchronize()

        def route_a():
            c, dd, ff, mm = img.cpu().numpy(), d.cpu().numpy(), fl.cpu().numpy(), m.cpu().numpy()
            gray = cv2.cvtColor(c, cv2.COLOR_BGR2GRAY)
            return tr_a.track(gray, dd, np.ascontiguousarray(ff.transpose(1, 2, 0)), mm.astype(np.int32), f["obj_ids"], writeback=True)

        def route_b():
            return tr_b.track_tensors(img, d_b, fl, m_b, f["obj_ids"], writeback=True, rgb=False)

        order = (("a", route_a), ("b", route_b)) if t % 2 == 0 else (("b", route_b), ("a", route_a))
        T = {}
        for name, fn in order:
            t0 = time.perf_counter()
            T[name] = fn()
            (t_a if name == "a" else t_b).append(time.perf_counter() - t0)
        dpose = max(dpose, float(np.abs(T["a"] - T["b"]).max()))
    n = a.frames - a.warmup
    sa, sb = (tr_a.get("stage_ms") - st_a) / n, (tr_b.get("stage_ms") - st_b) / n
    k_ms, k_n, call_ms = ingest_kernel_ms(ctx, held, a.ingest_reps)
    npx = H * W
    ingest_bytes = npx * (3 + 4 + 8 + 8) + npx * (1 + 4 + 8 + 4)     # reads (BGR u8, f32, 2 x f32, i64) + resident writes (u8, f32, 2 x f32, i32)
    out = {
        "workload": f"config3: {a.frames} frames of {W}x{H}, 3000 ORB features, inputs held as CUDA tensors (BGR HWC u8, f32 depth, (2,H,W) f32 flow, i64 mask)",
        "gpu": gpu_info(0),
        "host_route_fps": n / sum(t_a[a.warmup:]),
        "device_route_fps": n / sum(t_b[a.warmup:]),
        "host_route_ms_per_frame": 1e3 * sum(t_a[a.warmup:]) / n,
        "device_route_ms_per_frame": 1e3 * sum(t_b[a.warmup:]) / n,
        "host_route_stage_ms": {"upload+depth_prep": float(sa[0]), "update_mask+writeback": float(sa[1])},
        "device_route_stage_ms": {"upload+depth_prep": float(sb[0]), "update_mask+writeback": float(sb[1])},
        "k_ingest_frame_ms": k_ms, "k_ingest_frame_launches_profiled": k_n,
        "k_ingest_frame_GBps": (ingest_bytes / (k_ms * 1e-3) / 1e9) if k_ms else None, "k_ingest_frame_bytes": ingest_bytes,
        "upload_tensors_call_ms": call_ms,
        "max_abs_pose_diff": dpose,
    }
    print(json.dumps(out))
    if dpose != 0.0:
        raise SystemExit(f"the two routes disagree: largest pose difference {dpose}")


if __name__ == "__main__":
    main()
