"""Time b200bt_grid_sweep at BASELINE configs[1]'s shape: 1024 grid parameter sets x 10 symbols x 1M 1-minute bars.

    python tools/grid_bench.py [--pop 1024] [--symbols 10] [--bars 1000000] [--reps 10] [--day-profit]

Prints one JSON line: the card and its power limit, kernel time (CUDA events, median / min / max of --reps launches after
a warm-up), lane-ticks per second, and the DRAM bytes the kernel must move (each CTA of 16 individuals streams its
symbol's closes once: S * ceil(pop / 16) * N * 4 bytes through L2, of which S * N * 4 come from DRAM, plus the stats).
"""
from __future__ import annotations

import argparse
import json
import random

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pop", type=int, default=1024)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--day-profit", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.grid import GridSweep, grid_param_ranges
    from ai_crypto_trader_b200.sweep import MarketData
    torch.cuda.set_device(0)
    market = MarketData(synth.synth_ohlcv(a.symbols, a.bars))
    sweep = GridSweep(market, quantity=0.01)
    rng = random.Random(1)
    pop = [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi))
            for k, (lo, hi) in grid_param_ranges().items()} for _ in range(a.pop)]
    st = sweep.grid_stats(pop)                                      # warm-up; the stats describe the population
    packed, bounds = sweep.decode(pop)                              # the kernel alone is timed from here
    indiv = torch.from_numpy(packed).to(market.device)
    bnd = torch.from_numpy(bounds).to(market.device)
    stats = torch.empty((a.pop, a.symbols, 20), dtype=torch.float64, device=market.device)
    D = sweep.calendar_days()[1]
    rows = torch.empty((a.pop, D), dtype=torch.float64, device=market.device) if a.day_profit else None
    times = harness.event_ms(lambda: sweep.launch(indiv, bnd, stats, rows=rows), a.reps, warmup=0)
    ticks = a.pop * a.symbols * (a.bars - sweep.start_bar)
    ms = float(np.median(times))
    print(json.dumps({
        "workload": "grid_sweep" + ("+day_profit" if a.day_profit else ""), "gpu": ", ".join(harness.card().values()),
        "pop": a.pop, "symbols": a.symbols, "bars": a.bars, "start_bar": sweep.start_bar,
        "ms_median": round(ms, 3), "ms_min": round(min(times), 3), "ms_max": round(max(times), 3),
        "lane_ticks_per_s": ticks / (ms / 1e3),
        "dram_bytes": a.symbols * a.bars * 4 + a.pop * a.symbols * (160 + 16),
        "l2_bytes": a.symbols * -(-a.pop // 16) * a.bars * 4,
        "mean_trades_per_lane": float(st["total_trades"].mean()),
        "mean_regenerations_per_lane": float(st["n_regenerations"].mean()),
        "lanes_with_near_ties": int((st["near_ties"] > 0).sum()),
    }))


if __name__ == "__main__":
    main()
