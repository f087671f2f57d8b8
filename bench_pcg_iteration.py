"""Where the time of one fused PCG iteration goes on the config-5 graph (the flagship workload of bench.py).

After one warm-up solve it prints one JSON line with
  * us_per_pcg_iter: CUDA-event timing of replays of the captured 8-iteration chunk (vdo_graph_time_kernel "pcg_iterate8") / 8;
  * chain_tiles_us: the chain-tile Schur product alone, back-to-back launches (vdo_graph_time_kernel "schur_chains", as bench.py);
  * with --profile (a run of its own: tracing slows the host), the per-iteration device time of every kernel that runs inside the
    chunks of one solve, from torch.profiler's kernel records, the sum of those on the critical path besides the chain tiles, and the
    remainder: the idle time between dependent nodes (us_per_pcg_iter - chain tiles - other kernels);
  * the card name, its power limit and clocks.max.sm, read in the same run.

    python bench_pcg_iteration.py [--workload config5] [--reps 50] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import WORKLOADS, LM_MAX_ITERS, LM_GAIN  # noqa: E402

# the kernels of the fused PCG iteration (DESIGN 5b)
CHUNK_KERNELS = ("k_pcg_p_hpp", "k_band_mul", "k_tile_schur2", "k_tile_finalize", "k_pcg_step_a")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clk}
    except Exception as e:  # the numbers stay valid without it, but say so
        return {"error": f"nvidia-smi: {e}"}


def profile_solve(G, pcg_iters):
    """Device time per PCG iteration of each chunk kernel over one solve, from torch.profiler kernel records."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    G.reset()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        G.optimize(max_iterations=LM_MAX_ITERS, gain_threshold=LM_GAIN)
        torch.cuda.synchronize()
    us = defaultdict(float)
    n = defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        base = next((k for k in CHUNK_KERNELS if k in name), None)
        if base is None:
            continue
        key = name.split("(")[0].replace("void ", "").replace("vdo::", "")
        us[key] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        n[key] += 1
    # the chunk kernels launch once per iteration of every chunk (also after convergence, when they return at once); the same kernels
    # with other template arguments (right-hand side, back-substitution) once per LM trial
    return {k: {"us_per_pcg_iter": us[k] / max(pcg_iters, 1), "launches": n[k]} for k in sorted(us) if n[k] >= pcg_iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config5", choices=[k for k in WORKLOADS if k != "cpu_sample"])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--profile", action="store_true", help="also one torch.profiler pass over a solve (take timings from a run without it)")
    args = ap.parse_args()
    import torch
    from vdo_slam_b200 import capi
    from vdo_slam_b200.synth import make_batch_graph

    torch.cuda.set_device(0)
    g = make_batch_graph(**WORKLOADS[args.workload])
    ctx = capi.Context(0)
    G = capi.BatchGraph(ctx, g)
    r = G.optimize(max_iterations=LM_MAX_ITERS, gain_threshold=LM_GAIN)      # warm-up solve: modules, captures, allocations
    pcg = r["pcg_iterations"]
    it_us = G.time_kernel("pcg_iterate8", args.reps) * 1e3 / 8.0
    chain_us = G.time_kernel("schur_chains", args.reps) * 1e3
    out = {"workload": args.workload, "lm_iterations": r["iterations"], "pcg_iterations": pcg,
           "pcg_iters_per_lm_iter": pcg / max(r["iterations"], 1),
           "us_per_pcg_iter": it_us, "chain_tiles_us": chain_us, "chain_share": chain_us / it_us,
           "how": f"CUDA events around {args.reps} replays of the captured 8-iteration chunk / back-to-back chain-tile launches"}
    if args.profile:
        k = profile_solve(G, pcg)
        is_chain = lambda n: n.startswith("k_tile_schur2") and "true" in n
        chains = sum(v["us_per_pcg_iter"] for n, v in k.items() if is_chain(n))
        beside = sum(v["us_per_pcg_iter"] for n, v in k.items() if n.startswith("k_band_mul"))
        others = sum(v["us_per_pcg_iter"] for n, v in k.items() if not is_chain(n) and not n.startswith("k_band_mul"))
        out["profile"] = {"kernels": k, "chain_tiles_us": chains, "band_mul_us_beside_chains": beside, "other_kernels_us": others,
                          "gaps_us": it_us - chains - others, "other_plus_gaps_share": (it_us - chains) / it_us,
                          "note": "kernel times: torch.profiler over one solve / PCG iterations of that solve; k_band_mul runs on a second stream "
                                  "beside the chain tiles and is left out of the sum; gaps = us_per_pcg_iter - chain tiles - other kernels"}
    out["gpu"] = card()
    G.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
