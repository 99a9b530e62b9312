#!/usr/bin/env python
"""Sweep of the thread-per-lane knobs on the bench workload (pop 1024 x 10 symbols x 1M bars).
    python tools/tile_tune.py [K list] [warm list]"""
import sys, itertools
import numpy as np, torch
import harness
from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population, evaluation_order

S, N, POP = 10, 1_000_000, 1024
m, pop = harness.configs1(S, N, POP); sw = PopulationSweep(m, mode="fused")
print(", ".join(harness.card().values()))
indiv = torch.from_numpy(decode_population(pop, sw.period_row).view(np.uint8)).cuda()
fit = torch.empty(POP, dtype=torch.float64, device="cuda")

def timed(plan, order=None, reps=3):
    return float(np.mean(harness.event_ms(lambda: sw.evaluate_device(indiv, order, POP, fit, plan=plan), reps, warmup=2)))

order = torch.from_numpy(evaluation_order(pop)).cuda()
print("fused %.2f ms" % timed(None, order)); ref = fit.clone()
ks = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else (0, 7, 11, 15)
warms = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else (4096, 8192)
orders = sys.argv[3].split(",") if len(sys.argv) > 3 else ("row_cost",)
for k, warm, ob in itertools.product(ks, warms, orders):
    plan = sw.plan_tiles(pop, warm=warm, order_by=ob, **({"chunks": k} if k else {}))
    ms = timed(plan)
    print(f"K {plan.K:3d} warm {warm:5d} order {ob:6s}: {ms:6.2f} ms  invalid lanes {sw.last_invalid_lanes:4d}  "
          f"close {bool(torch.allclose(ref, fit, rtol=1e-9, atol=1e-12, equal_nan=True))}")
