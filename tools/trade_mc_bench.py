#!/usr/bin/env python
"""Trade-sequence Monte-Carlo throughput on the configs[1] workload.

    python tools/trade_mc_bench.py [--top 64] [--paths 10000] [--reps 10]

The configs[1] synthetic market and population of bench.py (10 symbols x 1M 1-minute bars, population 1024, seed 42) are
swept once; the `--top` individuals by fitness x all symbols are the lanes.  Timed separately:
  * extraction: PopulationSweep.trade_pnl (two sweeps of the top individuals + b200bt_trade_pnl), host clock;
  * the Monte-Carlo kernel (b200bt_trade_mc) for `bootstrap` (block 1) and `shuffle`: CUDA events, warmed up, `--reps`
    repetitions; round-trip steps/s = paths x sum(T) / kernel time;
  * the statistics of every lane (risk_statistics with the drawdown's p95: a few launches and a read-back per lane),
    host clock.
Prints one JSON line with the card's name, power limit and the SM clock sampled during the kernel timing, the trip
counts (min / median / max / sum) and the registers / local memory of the new kernels.  Needs an H100; no fallback.
"""
import argparse
import json
import time

import numpy as np
import torch

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--top", type=int, default=64)
    ap.add_argument("--paths", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--pop", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trade_mc_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from ai_crypto_trader_b200.monte_carlo import risk_statistics
    from ai_crypto_trader_b200.trade_monte_carlo import TradeMonteCarlo
    torch.cuda.set_device(0)
    market, population = harness.configs1(a.symbols, a.bars, a.pop)
    sweep = PopulationSweep(market)
    fitness = sweep.evaluate(population)
    rank = np.argsort(-np.nan_to_num(fitness, nan=-np.inf, posinf=np.finfo(np.float64).max), kind="stable")
    top = [population[i] for i in rank[:a.top]]

    sweep.trade_pnl(top)                                   # warm-up (plans, buffers)
    ext, (trip, n_trips, fee) = harness.wall_ms(lambda: sweep.trade_pnl(top), 3)
    nt = n_trips.cpu().numpy().reshape(-1).astype(np.int32)
    fe = fee.cpu().numpy().reshape(-1)
    rows = trip.view(len(nt), -1)
    sum_t = int(nt.sum())

    mc = TradeMonteCarlo()
    legs = {}
    for method in ("bootstrap", "shuffle"):
        run = lambda: mc.simulate(rows, nt, fe, a.paths, method, 1, 10000.0, 2024)
        with harness.sampled_clocks() as clocks:
            ms = float(np.mean(harness.event_ms(run, a.reps, warmup=2)))
        finals, maxdd = run()
        t0 = time.perf_counter()
        p5 = [risk_statistics(mc.engine, finals[r], maxdd[r], 10000.0, 0.95, mdd_percentiles=(95,))["percentile_values"][1]
              for r in range(len(nt))]
        stats_ms = (time.perf_counter() - t0) * 1e3
        legs[method] = {"kernel_ms": ms, "round_trip_steps_per_s": a.paths * sum_t / (ms * 1e-3),
                        "statistics_ms_all_lanes": stats_ms, "statistics_ms_per_lane": stats_ms / len(nt),
                        "sm_clock": clocks.sm_clock, "p5_final_equity_median": float(np.median(p5))}
    print(json.dumps({
        "workload": f"trade Monte-Carlo: top {a.top} of configs[1] population {a.pop} by fitness x {a.symbols} symbols x "
                    f"{a.bars} bars, {a.paths} paths per lane",
        **harness.card(), "lanes": int(len(nt)),
        "trips": {"min": int(nt.min()), "median": float(np.median(nt)), "max": int(nt.max()), "sum": sum_t},
        "extraction_ms": {"median": float(np.median(ext)), "runs": ext},
        "methods": legs, "kernels": harness.kernel_resources(["trade_mc_kernel", "trade_pnl_kernel"]),
    }))


if __name__ == "__main__":
    main()
