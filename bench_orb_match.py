#!/usr/bin/env python
"""bench_orb_match.py -- ORB descriptor matching of P pairs of consecutive frames on the device (capi.orb_match) against
cv2.BFMatcher(NORM_HAMMING) on the host.

Frames 0..P of synthetic sequence 0 (synth.make_sequence_frame, 1242x375) get their ORB keypoints and descriptors from one OrbExtractor
(3 000 features, scale 1.2, 8 levels, FAST 20 / 7); pair p is (frame p, frame p + 1).  For P in {1, 8, 32, 64} and three modes:
  knn    k = 2, no window
  window k = 2, r = 15 px around the query position moved by the synthetic flow
  cross  k = 1 with cross-check
the time of one orb_match call (CUDA events around an eager call on torch's stream, after warm-up; median of --reps calls: call_ms, which
includes the host's argument checks while the GPU waits), the device time of the same call captured in a CUDA graph (events around a
replay; median: graph_ms, and per pair), and distance evaluations per second (sum over pairs of nq * nt over graph_ms; the window mode
tests the same pairs, it only skips the popcount of non-candidates).  The host arm is cv2.BFMatcher.knnMatch per pair (knnMatch(mask=) in window mode, crossCheck=True match
in cross mode), timed with a host clock.  Every P asserts that the device result equals cv2's, pair by pair.  The GPU name and power
limit are read in the same run.  Prints one JSON line per (P, mode).

  python bench_orb_match.py [--pairs 1,8,32,64] [--reps 20] [--warmup 3] [--host-pairs 8]
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

W, H, RADIUS = 1242, 375, 15.0


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers are still device times; say that the card could not be read
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,32,64")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-pairs", type=int, default=8, help="pairs timed on the host per P (all pairs are compared)")
    a = ap.parse_args()
    import cv2
    import torch
    from tests import orb_match_reference as R
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_sequence_frame

    Ps = [int(v) for v in a.pairs.split(",")]
    nf = max(Ps) + 1
    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    frames = [make_sequence_frame(t, seed=0, width=W, height=H) for t in range(nf)]
    ex = capi.OrbExtractor(ctx, W, H, 64, n_features=3000)
    parts = []
    for s in range(0, nf, 64):
        r = ex.extract(torch.from_numpy(np.stack([f["gray"] for f in frames[s:s + 64]])).to(dev))
        parts.append({k: r[k].clone() for k in ("descriptors", "x", "y", "count", "status")})
    S = {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
    torch.cuda.synchronize()
    assert int(S["status"].abs().sum()) == 0
    Sh = {k: S[k].cpu().numpy() for k in ("descriptors", "x", "y", "count")}
    cnt = Sh["count"]
    cap = S["x"].shape[1]
    info = gpu_info()

    def pred_for(P):
        out = np.zeros((P, cap, 2), np.float32)
        for p in range(P):
            x, y = Sh["x"][p], Sh["y"][p]
            xi = np.clip(np.nan_to_num(x), 0, W - 1).astype(np.int64)     # rows past the count hold whatever the buffer held
            yi = np.clip(np.nan_to_num(y), 0, H - 1).astype(np.int64)
            out[p, :, 0] = x + frames[p]["flow"][yi, xi, 0].astype(np.float32)
            out[p, :, 1] = y + frames[p]["flow"][yi, xi, 1].astype(np.float32)
        return out

    for P in Ps:
        pairs = [(p, p + 1) for p in range(P)]
        pred = pred_for(P)
        pred_t = torch.from_numpy(pred).to(dev)
        evals = float(sum(int(cnt[q]) * int(cnt[t]) for q, t in pairs))
        for mode in ("knn", "window", "cross"):
            k = 1 if mode == "cross" else 2
            kw = dict(k=k, radius=RADIUS if mode == "window" else None, pred=pred_t if mode == "window" else None, cross_check=mode == "cross")
            out = capi.orb_match_empty_outputs(ctx, P, cap, cap, k, mode == "cross")
            for _ in range(a.warmup):
                capi.orb_match(ctx, S, S, pairs, out=out, **kw)
            st = torch.cuda.current_stream(dev)
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                capi.orb_match(ctx, S, S, pairs, out=out, **kw)
                e1.record(st)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            med = float(np.median(ms))
            # the same call captured in a CUDA graph: device time without the host's argument checks and enqueue
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                capi.orb_match(ctx, S, S, pairs, out=out, **kw)
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
            gmed = float(np.median(gms))
            gi, gd = out["idx"].cpu().numpy(), out["dist"].cpu().numpy()
            host_ms = []
            for p, (q, t) in enumerate(pairs):
                nq, nt = int(cnt[q]), int(cnt[t])
                cand = R.window_mask(Sh["x"][t, :nt], Sh["y"][t, :nt], pred[p, :nq], RADIUS) if mode == "window" else None
                t0 = time.perf_counter()
                ci, cd = R.cv2_knn(cv2, Sh["descriptors"][q, :nq], Sh["descriptors"][t, :nt], k, cand, mode == "cross")
                if p < a.host_pairs:
                    host_ms.append((time.perf_counter() - t0) * 1e3)
                assert np.array_equal(gi[p, :nq], ci) and np.array_equal(gd[p, :nq], cd), f"P={P} {mode}: pair {p} differs from cv2"
            print(json.dumps({"P": P, "mode": mode, "k": k, "call_ms": round(med, 4), "call_ms_min": round(min(ms), 4), "call_ms_max": round(max(ms), 4),
                              "graph_ms": round(gmed, 4), "graph_ms_min": round(min(gms), 4), "graph_ms_max": round(max(gms), 4),
                              "graph_us_per_pair": round(gmed * 1e3 / P, 2), "distance_evals_per_s": float(f"{evals / (gmed * 1e-3):.4g}"), "mean_features": round(float(np.mean(cnt[:P + 1])), 1),
                              "cv2_ms_per_pair": round(float(np.median(host_ms)), 2), "cv2_equal": True, "cv2_threads": cv2.getNumThreads(),
                              **info}), flush=True)


if __name__ == "__main__":
    main()
