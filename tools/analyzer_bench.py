#!/usr/bin/env python
"""TechnicalAnalyzer (all 21 indicator columns + NaN policy: b200bt_analyzer) on S symbols x 1M bars: time per call with CUDA
events and GB/s against the algorithmic bytes (high, low, close, volume read once + 21 columns written, 4 B each).
    python tools/analyzer_bench.py [S ...]"""
import json, os, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.indicators import TechnicalAnalyzer
from ai_crypto_trader_b200.sweep import MarketData
peak = json.load(open(ROOT / "MEASURED_PEAKS.json"))["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0     # H100 SXM data sheet
for S in [int(x) for x in sys.argv[1:]] or [10, 50]:
    m = MarketData(synth.synth_ohlcv(S, 1_000_000)).materialise()
    torch.cuda.synchronize()
    for _ in range(3): ta = TechnicalAnalyzer(m)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): ta = TechnicalAnalyzer(m)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    gb = (4 + 21) * 4 * S * 1e6 / 1e9
    print(json.dumps({"symbols": S, "bars": 1000000, "ms": ms, "algorithmic_GB": gb, "GBps": gb / (ms * 1e-3), "frac_of_hbm_peak": gb / (ms * 1e-3) / peak,
                      "note": "TechnicalAnalyzer(market): 3 fused launches + batched NaN policy + last-bar readback"}))
    del m, ta
    torch.cuda.empty_cache()
