#!/usr/bin/env python
"""Cost of the market-monitor kernel (csrc/market_monitor.cu) on the configs[1] workload.

    python tools/market_monitor_bench.py [--reps 5]

* b200bt_market_monitor on the configs[1] synthetic market (10 symbols x 1M 1-minute bars), W = 100 klines per frame,
  the 3-, 5- and 15-minute klines resampled once beforehand (not timed): with the 352-byte rows (and labels) written,
  and with the labels alone;
* PopulationSweep.class_stats with the trend labels (3 classes) on a random population of --pop individuals (seed 42).
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
        raise SystemExit("market_monitor_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200 import indicators as ind
    from ai_crypto_trader_b200 import market_monitor as mm
    from ai_crypto_trader_b200.sweep import PopulationSweep
    torch.cuda.set_device(0)
    market, population = harness.configs1(a.symbols, a.bars, a.pop)
    S, N = market.S, market.N
    k3, k5, k15 = (ind.resample(market, k) for k in (3, 5, 15))
    rows = torch.empty((S, N, mm.ROW_DTYPE.itemsize // 8), dtype=torch.float64, device=market.device)
    labels = torch.empty((S, N), dtype=torch.uint8, device=market.device)
    params = mm.monitor_params(100, 0)

    def launch(with_rows):
        _lib.call("b200bt_market_monitor", market.ohlcv.data_ptr(), S, N, market.minute0, 1, k3.ohlcv.data_ptr(), k3.N,
                  k5.ohlcv.data_ptr(), k5.N, k15.ohlcv.data_ptr(), k15.N, C.byref(params),
                  rows.data_ptr() if with_rows else None, labels.data_ptr(), _lib.current_stream())

    out = {"workload": f"configs[1]: {S} symbols x {N} 1-minute bars, W = 100", **harness.card()}
    with harness.sampled_clocks() as clocks:
        for with_rows in (True, False):
            t = _time(lambda: launch(with_rows), a.reps)
            out["rows" if with_rows else "labels_only"] = dict(t, updates=S * N, updates_per_s=S * N / (t["ms_median"] * 1e-3))
        trend, names = mm.monitor_labels(market, "trend")
        sweep = PopulationSweep(market)
        out["class_stats_trend"] = _time(lambda: sweep.class_stats(population, trend, len(names)), a.reps)
        _, views = sweep.class_stats(population, trend, len(names))
        out["records_per_trend"] = [float(v["n_records"].sum()) for v in views]
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
