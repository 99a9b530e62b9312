#!/usr/bin/env python
"""Fused vs warp-per-chunk vs thread-per-lane sweep across population sizes (10 symbols x N bars).
    python tools/mode_crossover.py [N bars]"""
import sys
import numpy as np, torch
import harness
from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population, evaluation_order
S, N = 10, (int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000)
m, allpop = harness.configs1(S, N, 8192); sw = PopulationSweep(m, mode="fused")
print(", ".join(harness.card().values()))
def run(pop, plan):
    indiv = torch.from_numpy(decode_population(pop, sw.period_row).view(np.uint8)).cuda()
    order = torch.from_numpy(evaluation_order(pop)).cuda()
    fit = torch.empty(len(pop), dtype=torch.float64, device="cuda")
    f = lambda: sw.evaluate_device(indiv, order, len(pop), fit, plan=plan)
    return float(np.mean(harness.event_ms(f, 3, warmup=2)))
for P in (8, 32, 128, 512, 1024, 2048, 8192):
    pop = allpop[:P]
    tf = run(pop, None)
    res = []
    for target, warm in ((8192, 8192), (16384, 8192)):
        res.append("%6.2f" % run(pop, sw.plan_chunks(pop, target_events=target, warm=warm)))
    tp = sw.plan_tiles(pop)
    tt = run(pop, tp)
    print(f"pop {P:5d}: fused {tf:7.2f} ms | chunked(8k/8k, 16k/8k) {' '.join(res)} ms | tiled (K={tp.K}) {tt:6.2f} ms  "
          f"=> {P * S * N / tt / 1e6:8.1f} G evals/s")
