#!/usr/bin/env python
"""Cost of the volume-profile kernel (csrc/volume_profile.cu) on the configs[1] workload.

    python tools/volume_profile_bench.py [--reps 5]

* volume_profile.volume_profile_history on the configs[1] synthetic market (10 symbols x 1M 1-minute bars), 100-bar
  frames at the 5-minute clock (the monitor's df_5m; the 5-minute resample included) and at the 1-minute clock, with
  the 384-byte rows written and with the labels alone;
* volume_profile_labels (the 5-minute labels brought to the 1-minute clock) and PopulationSweep.class_stats with those
  6 zone labels on a random population of --pop individuals (seed 42).
Every leg is timed with CUDA events, median of --reps runs after a warm-up run.  Prints one JSON line with the card's
name, power limit and the SM clock sampled while timing.  Needs an H100; no fallback.
"""
import argparse
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
        raise SystemExit("volume_profile_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import volume_profile as vp
    from ai_crypto_trader_b200.sweep import PopulationSweep
    torch.cuda.set_device(0)
    market, population = harness.configs1(a.symbols, a.bars, a.pop)
    out = {"workload": f"configs[1]: {a.symbols} symbols x {a.bars} 1-minute bars, 100-bar frames, 20 bins",
           **harness.card()}
    with harness.sampled_clocks() as clocks:
        for tf in (5, 1):
            frames = a.symbols * (a.bars // tf)
            for rows in (True, False):
                key = f"history_{tf}m_{'rows' if rows else 'labels_only'}"
                t = _time(lambda: vp.volume_profile_history(market, tf, rows=rows), a.reps)
                out[key] = dict(t, frames=frames, frames_per_s=frames / (t["ms_median"] * 1e-3))
        out["labels_base_clock"] = _time(lambda: vp.volume_profile_labels(market), a.reps)
        labels = vp.volume_profile_labels(market)
        sweep = PopulationSweep(market)
        out["class_stats_6_zones"] = _time(lambda: sweep.class_stats(population, labels, 6), a.reps)
        _, views = sweep.class_stats(population, labels, 6)
        out["records_per_zone"] = [float(v["n_records"].sum()) for v in views]
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
