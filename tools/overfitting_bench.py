#!/usr/bin/env python
"""Cost of the backtest-overfitting kernels (csrc/overfitting.cu) on the configs[1] workload.

    python tools/overfitting_bench.py [--reps 5]

* b200bt_daily_pnl on the event buffers of the configs[1] synthetic market (10 symbols x 1M 1-minute bars) for the two
  populations of tools/book_bench.py: the random one (seed 42) and generation 3 of GeneticAlgorithm(seed 42) started
  from it; beside it, the sweep that writes those buffers;
* b200bt_cscv on matrices of as many days as those rows: N = 1024 trials at B = 16 and 20, N = 10 000 at B = 16.
Every leg is timed with CUDA events after a warm-up run.  Prints one JSON line with the card's name, power limit and the
SM clock sampled while timing.  Needs an H100; no fallback.
"""
import argparse
import ctypes as C
import json
import math

import numpy as np
import torch

import harness


def _time(fn, reps):
    ms = harness.event_ms(fn, reps)
    return {"ms_median": float(np.median(ms)), "ms_runs": ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--pop", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("overfitting_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.overfitting import cscv
    from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population
    torch.cuda.set_device(0)
    market, random_pop = harness.configs1(a.symbols, a.bars, a.pop)
    evolved = harness.generation3(PopulationSweep(market).fitness_function, random_pop)
    out = {"workload": f"configs[1]: population {a.pop} x {a.symbols} symbols x {a.bars} 1-minute bars",
           **harness.card(), "daily_pnl": {}, "cscv": {}}
    with harness.sampled_clocks() as clocks:
        st = _lib.current_stream()
        D = 0
        for label, population in (("random", random_pop), ("generation_3", list(evolved))):
            sweep = PopulationSweep(market)
            sweep.daily_pnl(population)                                   # plans, zone map
            pop = len(population)
            indiv = torch.from_numpy(decode_population(population, sweep.period_row).view(np.uint8)).to(market.device)
            cap = sweep._exact_cap(sweep._stats)
            records = float(sweep._stats[:, :, 0].sum().item())
            first, D = sweep.calendar_days()
            plan = sweep.plan(population)
            fit = torch.empty(pop, dtype=torch.float64, device=market.device)
            lanes = torch.empty((pop, market.S, D), dtype=torch.float64, device=market.device)
            book = torch.empty((pop, D), dtype=torch.float64, device=market.device)

            def sweep_events():
                sweep.evaluate_device(indiv, None, pop, fit, plan=plan, event_cap=cap)

            def rows():
                _lib.call("b200bt_daily_pnl", market.close.data_ptr(), _lib.ld(market.close), market.S, market.N,
                          indiv.data_ptr(), pop, C.byref(sweep.cfg), sweep._stats.data_ptr(), sweep._events.data_ptr(), cap,
                          lanes.data_ptr(), D, book.data_ptr(), st)

            t_sweep = _time(sweep_events, a.reps)
            t_rows = _time(rows, a.reps)
            out["daily_pnl"][label] = {"records": records, "days": D, "busiest_lane": cap, "sweep_with_events": t_sweep,
                                       "daily_pnl": t_rows,
                                       "records_per_s": records / (t_rows["ms_median"] * 1e-3)}
        rng = np.random.default_rng(3)
        for N, B in ((1024, 16), (1024, 20), (10_000, 16)):
            x = torch.from_numpy(rng.normal(0.0, 1.0, (N, D))).cuda()
            t = _time(lambda: cscv(x, B), a.reps)
            C_ = math.comb(B, B // 2)
            out["cscv"][f"N={N},B={B}"] = {"days": D, "combinations": C_, "trial_splits": N * C_, "cscv_call": t}
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
