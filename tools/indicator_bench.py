#!/usr/bin/env python
"""Family 1 (rolling indicators) on the C2-sized market (10 symbols x 1M bars): time per call with CUDA events
and GB/s against SURVEY 8(d)'s algorithmic bytes (4 B per input row read + 4 B per output row written, per bar).

    python tools/indicator_bench.py [--symbols 10] [--bars 1000000]
"""
import argparse, json, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
from ai_crypto_trader_b200 import indicators as ind, synth
from ai_crypto_trader_b200.sweep import MarketData, rsi_bank

ap = argparse.ArgumentParser()
ap.add_argument("--symbols", type=int, default=10)
ap.add_argument("--bars", type=int, default=1_000_000)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
a = ap.parse_args()
m = MarketData(synth.synth_ohlcv(a.symbols, a.bars))
o, h, l, c, v = m.open, m.high, m.low, m.close, m.volume
peak = json.loads((Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json").read_text()).get("hbm_gbs", 3350.0) \
    if (Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json").exists() else 3350.0     # H100 SXM data sheet

def timed(fn, reps=None):
    reps = reps or a.reps
    for _ in range(a.warmup): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

cases = [  # name, callable, input rows, output rows
    ("rsi_bank x26 (no NaN fill)", lambda: rsi_bank(c, list(range(5, 31)), fill=False), 1, 26),
    ("rsi_bank x26 (filled)", lambda: rsi_bank(c, list(range(5, 31))), 1, 26),
    ("ema_bank x2 (12, 26)", lambda: ind.ema_bank(c, [12, 26]), 1, 2),
    ("sma_bank x3 (20, 50, 200)", lambda: ind.sma_bank(c, [20, 50, 200]), 1, 3),
    ("macd (line, signal, diff)", lambda: ind.macd(c), 1, 3),
    ("bollinger (5 outputs)", lambda: ind.bollinger(c), 1, 5),
    ("stochastic (%K, %D)", lambda: ind.stochastic(h, l, c), 3, 2),
    ("williams_r", lambda: ind.williams_r(h, l, c), 3, 1),
    ("ichimoku (a, b)", lambda: ind.ichimoku(h, l), 2, 2),
    ("atr_bank x1 (14)", lambda: ind.atr_bank(h, l, c, [14]), 3, 1),
    ("vwap", lambda: ind.vwap(h, l, c, v), 4, 1),
]
rows = []
for name, fn, n_in, n_out in cases:
    ms = timed(fn)
    gb = (n_in + n_out) * 4 * a.symbols * a.bars / 1e9
    rows.append({"kernel": name, "ms": round(ms, 4), "algorithmic_GB": round(gb, 3), "GBps": round(gb / (ms * 1e-3), 1),
                 "frac_of_hbm_peak": round(gb / (ms * 1e-3) / peak, 3)})
    print(f"{name:32s} {ms:8.3f} ms  {gb:6.3f} GB  {gb / (ms * 1e-3):8.1f} GB/s  {gb / (ms * 1e-3) / peak:6.1%}")
print(json.dumps({"workload": f"{a.symbols} symbols x {a.bars} bars", "hbm_peak_GBps": peak, "indicators": rows}))
