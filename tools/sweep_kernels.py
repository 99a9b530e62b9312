#!/usr/bin/env python
"""Device time per kernel of one configs[1] generation (population 1024 x 10 symbols x 1M bars), as bench.py builds it, for
the random seed-42 population and for the generation-3 population bench.py's `evolved_population_value` times.

    python tools/sweep_kernels.py [--sweeps 3] [--warmup 3] [--json OUT.json]

torch.profiler with CUDA activities (CUPTI) records every kernel, memset and copy of the profiled sweeps; the table lists the
mean device time per sweep of each, the share of the summed device time, and launches per sweep.  The card's name, power
limit and SM clock (nvidia-smi, sampled during the profiled sweeps) are printed beside it: the numbers mean nothing
without them.  `peak chunks` is PopulationSweep.last_peak_chunks (time chunks that set a new equity peak and took the
record-by-record drawdown pass), compared with tools/peak_chunks_model.py's CPU count."""
import argparse
import json
import re
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import harness
from ai_crypto_trader_b200.dist import ShardedFitness
from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population, evaluation_order

POP, S, N = 1024, 10, 1_000_000


def short(name: str) -> str:
    """'void b200bt::chunk_partial_kernel(...)' -> 'chunk_partial_kernel'; template arguments kept."""
    m = re.search(r"(?:b200bt::)?([A-Za-z_][A-Za-z0-9_]*(?:<[^()]*>)?)\(", name)
    return m.group(1) if m else name


def profile_sweeps(sweep, indiv, order, plan, fit, sweeps, warmup):
    for _ in range(warmup):
        sweep.evaluate_device(indiv, order, POP, fit, plan=plan)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof, harness.sampled_clocks() as clocks:
        for _ in range(sweeps):
            sweep.evaluate_device(indiv, order, POP, fit, plan=plan)
        torch.cuda.synchronize()
    total, count = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = short(e.name)
            total[k] += e.time_range.elapsed_us() / 1e3
            count[k] += 1
    rows = sorted(((k, total[k] / sweeps, count[k] / sweeps) for k in total), key=lambda r: -r[1])
    return rows, {**harness.card(), "sm_clock": clocks.sm_clock}


def report(tag, rows, clocks, extra):
    summed = sum(r[1] for r in rows)
    print(f"\n== {tag}: {clocks['card']}, power limit {clocks['power_limit']}, SM clock {clocks['sm_clock']['sm_mhz']} MHz "
          f"(max {clocks['sm_max_mhz']})")
    print("   " + ", ".join(f"{k} {v}" for k, v in extra.items()))
    print(f"   {'kernel':<44}{'ms/sweep':>10}{'share':>8}{'launches':>10}")
    for k, ms, n in rows:
        print(f"   {k[:44]:<44}{ms:10.3f}{100 * ms / summed:7.1f}%{n:10.1f}")
    print(f"   {'sum of device time':<44}{summed:10.3f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", help="also write the tables here")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    market, population = harness.configs1(S, N, POP)
    sweep = PopulationSweep(market)
    fit = torch.empty(POP, dtype=torch.float64, device=dev)
    out = {}

    def leg(tag, pop, order):
        indiv = torch.from_numpy(decode_population(pop, sweep.period_row).view(np.uint8)).to(dev)
        order_dev = torch.from_numpy(order).to(dev) if order is not None else None
        plan = sweep.plan(pop)
        rows, clocks = profile_sweeps(sweep, indiv, order_dev, plan, fit, args.sweeps, args.warmup)
        segs = sum(int(p.n_seg) for p in plan) * S if plan else 0
        peak = getattr(sweep, "last_peak_chunks", None)
        extra = {"path": type(plan[0]).__name__ if plan else "fused", "K": getattr(plan[0], "K", None) if plan else None,
                 "records": float(sweep.lane_stats()["n_records"].sum()), "chunks": segs,
                 "peak chunks": peak if peak is None else f"{peak} ({100 * peak / max(segs, 1):.2f} %)",
                 "fallback lanes": sweep.last_invalid_lanes, "pool blocks planned": [p.pool_blocks for p in plan or []],
                 "pool blocks used": [int(p.overflow[2]) for p in plan or []]}
        report(tag, rows, clocks, extra)
        out[tag] = {"kernels": [{"kernel": k, "ms_per_sweep": ms, "launches_per_sweep": n} for k, ms, n in rows],
                    "card": clocks, **extra}

    leg("random population (seed 42)", population, evaluation_order(population))
    leg("generation-3 population", harness.generation3(ShardedFitness(sweep.evaluate, device=dev), population), None)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
