#!/usr/bin/env python
"""Cost of the market-regime kernels (csrc/regime.cu) on the configs[1] workload.

    python tools/regime_bench.py [--reps 5]

* regime.regime_labels on the configs[1] synthetic market (10 symbols x 1M 1-minute bars): the SMA rows, the 5-minute
  resample and alignment, and b200bt_regime_labels (timed as a whole and the labelling kernel alone);
* b200bt_class_stats at R = 5 on the event buffers of the two populations of tools/overfitting_bench.py (the random
  one, seed 42, and generation 3 of GeneticAlgorithm(seed 42) started from it); beside it, the sweep that writes those
  buffers and b200bt_daily_pnl on the same buffers.
Every leg is timed with CUDA events, median of --reps runs after a warm-up run.  Prints one JSON line with the card's
name, power limit and the SM clock sampled while timing.  Needs an H100; no fallback.
"""
import argparse
import ctypes as C
import json

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
        raise SystemExit("regime_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib, regime
    from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population
    torch.cuda.set_device(0)
    market, random_pop = harness.configs1(a.symbols, a.bars, a.pop)
    evolved = harness.generation3(PopulationSweep(market).fitness_function, random_pop)
    out = {"workload": f"configs[1]: population {a.pop} x {a.symbols} symbols x {a.bars} 1-minute bars",
           **harness.card(), "class_stats": {}}
    with harness.sampled_clocks() as clocks:
        st = _lib.current_stream()
        out["regime_labels"] = _time(lambda: regime.regime_labels(market), a.reps)
        rows = regime.trend_rows(market)
        S, N = market.S, market.N
        K = int(_lib.load().b200bt_regime_max_windows(N, 1))
        labels = torch.empty((S, N), dtype=torch.uint8, device=market.device)
        win = torch.empty((S, K, 8), dtype=torch.float64, device=market.device)
        params = regime.regime_params(60)
        base, plane = rows.data_ptr(), S * N

        def label_kernel():
            _lib.call("b200bt_regime_labels", base, base + 4 * plane, base + 8 * plane, base + 12 * plane, S, N, N,
                      market.minute0, 1, C.byref(params), labels.data_ptr(), N, win.data_ptr(), K, st)

        out["regime_labels_kernel"] = _time(label_kernel, a.reps)
        labels, _ = regime.regime_labels(market)
        R = 5
        for label, population in (("random", random_pop), ("generation_3", list(evolved))):
            sweep = PopulationSweep(market)
            sweep.daily_pnl(population)                                   # plans, zone map, exact cap
            pop = len(population)
            indiv = torch.from_numpy(decode_population(population, sweep.period_row).view(np.uint8)).to(market.device)
            cap = sweep._exact_cap(sweep._stats)
            records = float(sweep._stats[:, :, 0].sum().item())
            first, D = sweep.calendar_days()
            plan = sweep.plan(population)
            fit = torch.empty(pop, dtype=torch.float64, device=market.device)
            lanes = torch.empty((pop, S, D), dtype=torch.float64, device=market.device)
            classes = torch.empty((R, pop, S, 20), dtype=torch.float64, device=market.device)

            def sweep_events():
                sweep.evaluate_device(indiv, None, pop, fit, plan=plan, event_cap=cap)

            def rows_pass():
                _lib.call("b200bt_daily_pnl", market.close.data_ptr(), _lib.ld(market.close), S, N, indiv.data_ptr(), pop,
                          C.byref(sweep.cfg), sweep._stats.data_ptr(), sweep._events.data_ptr(), cap, lanes.data_ptr(), D,
                          None, st)

            def class_pass():
                _lib.call("b200bt_class_stats", market.close.data_ptr(), _lib.ld(market.close), S, N, indiv.data_ptr(), pop,
                          C.byref(sweep.cfg), sweep._stats.data_ptr(), sweep._events.data_ptr(), cap, labels.data_ptr(), N,
                          R, classes.data_ptr(), st)

            t_sweep = _time(sweep_events, a.reps)
            t_rows = _time(rows_pass, a.reps)
            t_cls = _time(class_pass, a.reps)
            out["class_stats"][label] = {"records": records, "busiest_lane": cap, "sweep_with_events": t_sweep,
                                         "daily_pnl": t_rows, "class_stats_R5": t_cls,
                                         "records_per_s": records / (t_cls["ms_median"] * 1e-3)}
            del sweep, lanes, classes
            torch.cuda.empty_cache()
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
