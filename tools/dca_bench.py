"""Time the DCA kernels at BASELINE configs[1]'s shape: 1024 DCA parameter sets x 10 symbols x 1M 1-minute bars.

    python tools/dca_bench.py [--pop 1024] [--symbols 10] [--bars 1000000] [--reps 5]

Prints one JSON line per workload -- b200bt_dca_dip_pct; the sweep with random genes; the sweep with per-day rows; the
worst case (cooldown 0 and a threshold every checked tick meets: a dip purchase on every tick) -- with the card, its power
limit and max SM clock, kernel time (CUDA events, median / min / max of --reps launches after a warm-up), lane-ticks per
second and purchases per lane.
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
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.dca import DCASweep, dca_param_ranges, dip_pct
    from ai_crypto_trader_b200.sweep import MarketData
    torch.cuda.set_device(0)
    ohlcv = synth.synth_ohlcv(a.symbols, a.bars)
    ohlcv[1] = np.maximum(ohlcv[1], ohlcv[3])
    market = MarketData(ohlcv)
    gpu = ", ".join(harness.card().values())
    sweep = DCASweep(market, start_bar=7 * 1440, usdc_balance=5000.0)
    T = a.bars - sweep.start_bar

    def report(name, times, purchases=None):
        ms = times[len(times) // 2]
        row = {"workload": name, "gpu": gpu, "pop": a.pop, "symbols": a.symbols, "bars": a.bars,
               "ms_median": round(ms, 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3)}
        if purchases is not None:
            row["lane_ticks_per_s"] = a.pop * a.symbols * T / (ms / 1e3)
            row["purchases_per_lane"] = purchases
        print(json.dumps(row), flush=True)

    report("dca_dip_pct", sorted(harness.event_ms(lambda: dip_pct(market), a.reps)))
    rng = random.Random(1)
    random_pop = [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi))
                   for k, (lo, hi) in dca_param_ranges().items()} for _ in range(a.pop)]
    worst = [dict(p, price_dip_detection=1, max_dip_frequency_days=0, dip_threshold_pct=-1e300) for p in random_pop]
    for name, pop, day in (("dca_sweep", random_pop, False), ("dca_sweep+day_rows", random_pop, True),
                           ("dca_sweep worst case", worst, False)):
        st = sweep.dca_stats(pop)
        per_lane = float((st["n_scheduled"] + st["n_dip"] + st["n_rebalance"]).mean())
        packed, first, target, reb = sweep.decode(pop)
        dev = market.device
        indiv = torch.from_numpy(packed.copy()).to(dev)
        first_us = torch.from_numpy(first).to(dev)
        tgt = torch.from_numpy(target).to(dev)
        stats = torch.empty((a.pop, a.symbols, 20), dtype=torch.float64, device=dev)
        service = torch.empty((a.pop, 5), dtype=torch.float64, device=dev)
        rows = torch.empty((a.pop, sweep.calendar_days()[1]), dtype=torch.float64, device=dev) if day else None
        run = lambda: sweep.launch(indiv, first_us, stats, service, rows, target=tgt, rebalance_any=reb)
        report(name, sorted(harness.event_ms(run, a.reps)), per_lane)


if __name__ == "__main__":
    main()
