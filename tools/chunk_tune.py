#!/usr/bin/env python
"""Sweep of the time-chunking knobs on the bench workload (pop 1024 x 10 symbols x 1M bars)."""
import sys, itertools
import numpy as np, torch
import harness
from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population

S, N, POP = 10, 1_000_000, 1024
m, pop = harness.configs1(S, N, POP); sw = PopulationSweep(m, mode="fused")
print(", ".join(harness.card().values()))
packed = decode_population(pop, sw.period_row)
indiv = torch.from_numpy(packed.view(np.uint8)).cuda()
fit = torch.empty(POP, dtype=torch.float64, device="cuda")

def timed(plan, order=None, reps=3):
    return float(np.mean(harness.event_ms(lambda: sw.evaluate_device(indiv, order, POP, fit, plan=plan), reps, warmup=2)))

from ai_crypto_trader_b200.sweep import evaluation_order
order = torch.from_numpy(evaluation_order(pop)).cuda()
print("fused %.2f ms" % timed(None, order)); ref = fit.clone()
targets = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else (2048, 4096, 8192, 16384)
warms = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else (2048, 4096, 8192)
for target, warm in itertools.product(targets, warms):
    plan = sw.plan_chunks(pop, target_events=target, warm=warm)
    ms = timed(plan)
    print(f"target_events {target:6d} warm {warm:5d}: {ms:6.2f} ms  items {plan.n_seg:5d}  max K {int(plan.n_chunks.max()):3d}  invalid lanes {sw.last_invalid_lanes:4d}  close {bool(torch.allclose(ref, fit, rtol=1e-9, atol=1e-12, equal_nan=True))}")
