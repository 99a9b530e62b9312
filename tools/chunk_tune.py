#!/usr/bin/env python
"""Sweep of the time-chunking knobs on the bench workload (pop 1024 x 10 symbols x 1M bars)."""
import sys, itertools
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np, torch
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep, decode_population

S, N, POP = 10, 1_000_000, 1024
m = MarketData(synth.synth_ohlcv(S, N)); sw = PopulationSweep(m, mode="fused")
pop = synth.random_population(POP, seed=42)
packed = decode_population(pop, sw.period_row)
indiv = torch.from_numpy(packed.view(np.uint8)).cuda()
fit = torch.empty(POP, dtype=torch.float64, device="cuda")

def timed(plan, reps=3):
    for _ in range(2): sw.evaluate_device(indiv, None, POP, fit, plan=plan)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): sw.evaluate_device(indiv, None, POP, fit, plan=plan)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

from ai_crypto_trader_b200.sweep import evaluation_order
order = torch.from_numpy(evaluation_order(pop)).cuda()
for _ in range(2): sw.evaluate_device(indiv, order, POP, fit)
torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); [sw.evaluate_device(indiv, order, POP, fit) for _ in range(3)]; e1.record(); torch.cuda.synchronize()
ref = fit.clone(); print("fused %.2f ms" % (e0.elapsed_time(e1) / 3))
targets = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else (2048, 4096, 8192, 16384)
warms = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else (2048, 4096, 8192)
for target, warm in itertools.product(targets, warms):
    plan = sw.plan_chunks(pop, target_events=target, warm=warm)
    ms = timed(plan)
    print(f"target_events {target:6d} warm {warm:5d}: {ms:6.2f} ms  items {plan.n_seg:5d}  max K {int(plan.n_chunks.max()):3d}  invalid lanes {sw.last_invalid_lanes:4d}  close {bool(torch.allclose(ref, fit, rtol=1e-9, atol=1e-12, equal_nan=True))}")
