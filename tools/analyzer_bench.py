#!/usr/bin/env python
"""TechnicalAnalyzer (all 21 indicator columns + NaN policy: b200bt_analyzer) on S symbols x 1M bars: time per call with CUDA
events and GB/s against the algorithmic bytes (high, low, close, volume read once + 21 columns written, 4 B each).
    python tools/analyzer_bench.py [S ...]"""
import json, sys
import numpy as np
import torch
import harness
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.indicators import TechnicalAnalyzer
from ai_crypto_trader_b200.sweep import MarketData
peak = json.load(open(harness.ROOT / "MEASURED_PEAKS.json"))["hbm_gbs"] if (harness.ROOT / "MEASURED_PEAKS.json").exists() else 3350.0     # H100 SXM data sheet
for S in [int(x) for x in sys.argv[1:]] or [10, 50]:
    m = MarketData(synth.synth_ohlcv(S, 1_000_000)).materialise()
    ms = float(np.mean(harness.event_ms(lambda: TechnicalAnalyzer(m), 10, warmup=3)))
    gb = (4 + 21) * 4 * S * 1e6 / 1e9
    print(json.dumps({"symbols": S, "bars": 1000000, "ms": ms, "algorithmic_GB": gb, "GBps": gb / (ms * 1e-3), "frac_of_hbm_peak": gb / (ms * 1e-3) / peak,
                      **harness.card(), "note": "TechnicalAnalyzer(market): 3 fused launches + batched NaN policy + last-bar readback"}))
    del m
    torch.cuda.empty_cache()
