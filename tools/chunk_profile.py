#!/usr/bin/env python
"""One chunked evaluation of the bench workload (for `ncu --metrics gpu__time_duration.sum`)."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np, torch
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep, decode_population
S, N, POP = 10, 1_000_000, 1024
target = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
warm = int(sys.argv[2]) if len(sys.argv) > 2 else 8192
m = MarketData(synth.synth_ohlcv(S, N)); sw = PopulationSweep(m, mode="fused")
pop = synth.random_population(POP, seed=42)
indiv = torch.from_numpy(decode_population(pop, sw.period_row).view(np.uint8)).cuda()
fit = torch.empty(POP, dtype=torch.float64, device="cuda")
plan = sw.plan_chunks(pop, target_events=target, warm=warm)
for _ in range(2):
    sw.evaluate_device(indiv, None, POP, fit, plan=plan)
torch.cuda.synchronize()
print("done", sw.last_invalid_lanes)
