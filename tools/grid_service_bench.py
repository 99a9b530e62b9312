"""Time b200bt_grid_service_sweep (one service instance per individual, grid parameters coupled across its symbols) next
to b200bt_grid_sweep on the same population, at BASELINE configs[1]'s shape (1024 random grid_param_ranges() individuals
x 10 symbols x 1M 1-minute bars, start bar 43 200) and on the default config's 3 symbols.

    python tools/grid_service_bench.py [--pop 1024] [--bars 1000000] [--reps 5]

Prints one JSON line: the card and its power limit, and per symbol count the kernel times (CUDA events, median of --reps
launches after a warm-up) with and without per-day rows for both entry points, plus the service's adjust ticks and
regenerations per individual.
"""
from __future__ import annotations

import argparse
import json
import random

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pop", type=int, default=1024)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.grid import GridSweep, grid_param_ranges
    from ai_crypto_trader_b200.sweep import MarketData
    torch.cuda.set_device(0)
    out = {"workload": "grid_service_sweep", "gpu": ", ".join(harness.card().values()), "pop": a.pop, "bars": a.bars, "runs": []}
    ohlcv = synth.synth_ohlcv(10, a.bars)
    rng = random.Random(1)
    pop = [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi))
            for k, (lo, hi) in grid_param_ranges().items()} for _ in range(a.pop)]
    for S in (10, 3):
        market = MarketData(np.ascontiguousarray(ohlcv[:, :S]))
        sweep = GridSweep(market, quantity=0.01, start_bar=43_200, service=True)
        st = sweep.grid_stats(pop)                                  # warm-up; the stats describe the population
        sv = sweep.service_stats()
        packed, bounds = sweep.decode(pop)
        indiv = torch.from_numpy(packed.copy()).to(market.device)
        bnd = torch.from_numpy(bounds).to(market.device)
        stats = torch.empty((a.pop, S, 20), dtype=torch.float64, device=market.device)
        service = torch.empty((a.pop, 12), dtype=torch.float64, device=market.device)
        rows = torch.empty((a.pop, sweep.calendar_days()[1]), dtype=torch.float64, device=market.device)
        res = {"symbols": S}
        for name, sv_out, day in (("service_ms", service, False), ("service_day_ms", service, True),
                                  ("lane_ms", None, False), ("lane_day_ms", None, True)):      # None: b200bt_grid_sweep
            times = harness.event_ms(lambda: sweep.launch(indiv, bnd, stats, sv_out, rows if day else None), a.reps)
            res[name] = round(float(np.median(times)), 3)
        res["adjust_ticks_per_individual"] = float(sv["n_adjustments"].mean())
        res["regenerations_per_individual"] = float(st["n_regenerations"].sum(axis=1).mean())
        res["num_grids_changes_per_individual"] = float(sv["n_num_grids_changes"].mean())
        res["mean_trades_per_lane"] = float(st["total_trades"].mean())
        out["runs"].append(res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
