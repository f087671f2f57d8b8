"""Where the time of one config-5 LM solve goes outside and inside the PCG (the flagship workload of bench.py), stage by stage.

After one warm-up solve it prints one JSON line with
  * (a) totals with the profiler off: ms per solve (CUDA events around --solves solves), LM iterations, trials and PCG iterations,
    and vdo_graph_time_kernel "pcg_iterate8" (CUDA events around replays of the captured 8-iteration chunk);
  * (b) from torch.profiler's kernel records over one solve (a run of its own: tracing slows the host): device time and launch count of
    every kernel name (template arguments kept) and of the copies and memsets, their totals per phase of the LM trial, and for the
    tile kernels the compulsory HBM bytes per launch (bench.kernel_bytes and the counts below), GB/s and the share of 3.35 TB/s;
  * (c) idle time: solve time (a) minus the time some kernel or copy of the solve ran (the union of the profiled intervals, so that the
    kernels of the second stream beside the chain tiles or the PCR clusters count once). It is the cost of the host synchronisations:
    one per PCG chunk and one per trial;
  * (d) the card name, its power limit and clocks.max.sm, read in the same run.

    python bench_lm_trial.py [--workload config5] [--solves 3] [--no-profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, LM_MAX_ITERS, LM_GAIN, kernel_bytes  # noqa: E402
from bench_pcg_iteration import card  # noqa: E402

HBM_GBS = 3350.0     # H100 SXM data sheet

# phase of a kernel record, by the first matching (substring, phase) pair; names are "k_name<template args>"
PHASES = [
    ("k_pcg_p_hpp", "pcg"), ("k_band_mul", "pcg"), ("k_tile_finalize_ap_dot", "pcg"), ("k_pcg_step_a", "pcg"),
    ("k_tile_schur2<One, false, 1>", "pcg"), ("k_tile_schur2<One, true, 1>", "pcg"),
    ("k_tile_schur2<Many, false, 1>", "pcg"), ("k_tile_schur2<Many, true, 1>", "pcg"),
    ("k_tile_schur2<One, false, 2>", "backsub"), ("k_tile_schur2<One, true, 2>", "backsub"),
    ("k_tile_schur2<Many, false, 2>", "backsub"), ("k_tile_schur2<Many, true, 2>", "backsub"),
    ("k_tile_lin<One, false, true>", "linearise"), ("k_tile_lin<One, true, true>", "linearise"),
    ("k_tile_lin<Many, false, true>", "linearise"), ("k_tile_lin<Many, true, true>", "linearise"),
    ("k_tile_finalize_lin", "linearise"), ("k_lin_se3_edges<One, true>", "linearise"), ("k_lin_se3_edges<Many, true>", "linearise"),
    ("k_max_diagonal", "linearise"),
    ("k_factor_landmarks", "setup"), ("k_precond_begin", "setup"), ("k_tile_precond", "setup"), ("k_tile_finalize_precond", "setup"),
    ("k_pcr_factor", "setup"), ("k_band_form", "setup"), ("k_tile_schur2", "setup"), ("k_tile_finalize_schur2", "setup"),
    ("k_pcg_init", "setup"), ("k_set_scalars", "setup"), ("k_batch_scalars", "setup"), ("k_tile_setup", "setup"),
    ("k_vertex_transform", "backsub"),
    ("k_apply_update", "update_chi2"), ("k_tile_lin", "update_chi2"), ("k_lin_se3_edges", "update_chi2"), ("k_tile_post", "update_chi2"),
    ("k_update_se3", "update_chi2"),
    ("Memcpy DtoD", "push_pop"), ("Memset", "memset"), ("Memcpy DtoH", "read_back"), ("k_gather_scalars", "read_back"),
]


def phase_of(name):
    return next((p for k, p in PHASES if k in name), "other")


def short(name):
    return name.split("(")[0].replace("void ", "").replace("vdo::", "")


def trial_bytes(g):
    """Compulsory HBM bytes per launch of the per-trial and per-iteration landmark-side kernels (tiled layout; every array a kernel
    stages or writes, counted once; per-vertex gathers and segment descriptors not counted): bench.kernel_bytes plus the kernels it does
    not count."""
    kb = kernel_bytes(g)
    P = len(g["pt"])
    dyn = np.zeros(P, bool)
    if len(g["ter_pph"]):
        dyn[g["ter_pph"][:, 0]] = True; dyn[g["ter_pph"][:, 1]] = True
    Pd = int(dyn.sum()); Ps = P - Pd
    Epd = int(dyn[g["obs_cp"][:, 1]].sum()); Eps = len(g["obs_cp"]) - Epd
    C = len(g["se3"])
    kb.update({
        # H_ll + lambda I pivots: static hll 8 read, pivot 8 + g 8 written; chains hll, tk_omega read, pivot, g, gamma written
        "factor_static": 24 * Ps, "factor_chains": 40 * Pd,
        # preconditioner sums: edge omega' 8 + tile-local landmark 1 + permutation 2; landmark p 24 + g 8 (+ gamma 8, tk_omega 8, permutation 2)
        "precond_static": 11 * Eps + 32 * Ps, "precond_chains": 11 * Epd + 50 * Pd,
        # rhs (mode 0): as schur_* less the vertex-side camera and plus b_l 24 per landmark
        "rhs_static": 13 * Eps + 60 * Ps, "rhs_chains": 13 * Epd + 143 * Pd,
        # back-substitution (mode 2): edge omega' 8 + camera slot 1; landmark p 24 + pivot 8 + begin 4 + b_l 24 + x_l 24 written
        # (+ Q_k 72, tk_omega 8, motion slot 1)
        "backsub_static": 9 * Eps + 84 * Ps, "backsub_chains": 9 * Epd + 165 * Pd,
        # linearisation (k_tile_lin reads an 8-bit camera slot, not bench.kernel_bytes' 4-byte camera index, and the permutation with the
        # tile-local landmark as one 4-byte word): edge camera slot 1 + z 24 + class 1 + omega' (written) 8 + permutation | landmark 4
        # (+ tile-local landmark 1, static); landmark p 24 + begin 4 + hll 8 + b_l 24 + tk_omega 8 (+ motion slot 1 + class 1 + permutation 2
        # + Q_k (written) 72)
        "lin_static": 39 * Eps + 68 * Ps, "lin_chains": 38 * Epd + 144 * Pd,
        # chi2 (no write): edge camera slot 1 + z 24 + class 1 (+ tile-local landmark 1, static); landmark p 24 (+ begin 4 + motion slot 1
        # + class 1)
        "chi2_static": 27 * Eps + 24 * Ps, "chi2_chains": 26 * Epd + 30 * Pd,
        # update: se3 96 read + written + x_p 48; points 24 read + written + x_l 24 + b_l 24
        "apply_update": 240 * C + 96 * P,
        # push and pop: one copy of the estimate each way
        "copy_estimate": 2 * (96 * C + 24 * P),
    })
    return kb


# kernel-name substring -> trial_bytes key (the One instantiations of a lone solve)
BYTES_OF = [
    ("k_tile_lin<One, false, true>", "lin_static"), ("k_tile_lin<One, true, true>", "lin_chains"),
    ("k_tile_lin<One, false, false>", "chi2_static"), ("k_tile_lin<One, true, false>", "chi2_chains"),
    ("k_tile_finalize_lin", "lin_finalize"), ("k_factor_landmarks", None), ("k_tile_precond<One, false>", "precond_static"),
    ("k_tile_precond<One, true>", "precond_chains"), ("k_band_form", "band_form"),
    ("k_tile_schur2<One, false, 0>", "rhs_static"), ("k_tile_schur2<One, true, 0>", "rhs_chains"),
    ("k_tile_schur2<One, true, 1>", "schur_chains"),
    ("k_tile_schur2<One, false, 2>", "backsub_static"), ("k_tile_schur2<One, true, 2>", "backsub_chains"),
    ("k_apply_update", "apply_update"),
]


def profile_solve(G, g):
    import torch
    from torch.profiler import profile, ProfilerActivity
    G.reset()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = G.optimize(max_iterations=LM_MAX_ITERS, gain_threshold=LM_GAIN)
        torch.cuda.synchronize()
    us = defaultdict(float); n = defaultdict(int)
    iv = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        key = short(e.name)
        us[key] += t; n[key] += 1
        iv.append((e.time_range.start, e.time_range.end))
    # union of the device intervals: time in which some kernel or copy of the solve ran
    iv.sort()
    busy, cur0, cur1 = 0.0, None, None
    for a, b in iv:
        if cur1 is None or a > cur1:
            if cur1 is not None:
                busy += cur1 - cur0
            cur0, cur1 = a, b
        else:
            cur1 = max(cur1, b)
    if cur1 is not None:
        busy += cur1 - cur0
    span = (iv[-1][1] - iv[0][0]) if iv else 0.0
    kb = trial_bytes(g)
    kernels = {}
    phases = defaultdict(float)
    for k in sorted(us, key=lambda k: -us[k]):
        ph = phase_of(k)
        phases[ph] += us[k] / 1e3
        row = {"ms": us[k] / 1e3, "launches": n[k], "us_per_launch": us[k] / n[k], "phase": ph}
        key = next((b for s, b in BYTES_OF if s in k), None)
        if key is None and k.startswith("k_factor_landmarks"):
            row["bytes_per_launch"] = kb["factor_static"] + kb["factor_chains"]
        elif key is not None:
            row["bytes_per_launch"] = kb[key]
        if "bytes_per_launch" in row:
            gbs = row["bytes_per_launch"] / (row["us_per_launch"] * 1e-6) / 1e9
            row["GBps"] = gbs; row["share_of_hbm_peak"] = gbs / HBM_GBS
        kernels[k] = row
    return r, kernels, dict(phases), busy / 1e3, span / 1e3, kb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config5", choices=[k for k in WORKLOADS if k != "cpu_sample"])
    ap.add_argument("--solves", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_batch_graph

    torch.cuda.set_device(0)
    g = make_batch_graph(**WORKLOADS[args.workload])
    ctx = capi.Context(0)
    G = capi.BatchGraph(ctx, g)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    G.optimize(max_iterations=LM_MAX_ITERS, gain_threshold=LM_GAIN)      # warm-up solve: modules, captures, allocations
    ms = []
    for _ in range(args.solves):
        G.reset()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = G.optimize(max_iterations=LM_MAX_ITERS, gain_threshold=LM_GAIN)
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    solve_ms = float(np.median(ms))
    it8 = G.time_kernel("pcg_iterate8", 50)
    out = {"workload": args.workload, "lm_iterations": r["iterations"], "trials": r["trials"], "pcg_iterations": r["pcg_iterations"],
           "solve_ms": ms, "solve_ms_median": solve_ms, "lm_it_per_s": r["iterations"] / (solve_ms * 1e-3),
           "pcg_iterate8_ms": it8, "pcg_ms_estimate": it8 * r["pcg_iterations"] / 8.0}
    if not args.no_profile:
        rp, kernels, phases, busy_ms, span_ms, kb = profile_solve(G, g)
        out["profile"] = {
            "counts": [rp["iterations"], rp["trials"], rp["pcg_iterations"]],
            "phases_ms": phases, "phases_ms_per_trial": {k: v / max(rp["trials"], 1) for k, v in phases.items()},
            "kernel_ms_sum": sum(v["ms"] for v in kernels.values()), "busy_ms": busy_ms, "profiled_span_ms": span_ms,
            "idle_ms": solve_ms - busy_ms, "kernels": kernels, "bytes": kb,
            "note": "kernel times: torch.profiler over one solve; busy = union of the device intervals (second-stream kernels beside the "
                    "chain tiles / PCR clusters count once); idle_ms = solve_ms_median (profiler off) - busy_ms",
        }
    out["gpu"] = card()
    G.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
