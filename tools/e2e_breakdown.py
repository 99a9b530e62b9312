#!/usr/bin/env python
"""Where the end-to-end generation time goes (bench.py's e2e leg, phase by phase; wall clock with syncs)."""
import numpy as np, torch
import harness
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep, decode_population, evaluation_order, predicted_events
S, N, POP = 10, 1_000_000, 1024
ohlcv_host = torch.from_numpy(synth.synth_ohlcv(S, N)).pin_memory()
pop = synth.random_population(POP, seed=42)
print(", ".join(harness.card().values()))
def T(f, n=5):
    ms, r = harness.wall_ms(f, n, warmup=1)
    return float(np.mean(ms)), r
ms, mk = T(lambda: MarketData(ohlcv_host)); print(f"MarketData (H2D 200 MB)      {ms:7.2f} ms")
ms, sw = T(lambda: PopulationSweep(mk)); print(f"PopulationSweep (RSI bank)   {ms:7.2f} ms")
ms, _ = T(lambda: sw.evaluate(pop)); print(f"evaluate (total)             {ms:7.2f} ms")
ms, packed = T(lambda: decode_population(pop, sw.period_row)); print(f"  decode_population          {ms:7.2f} ms")
ms, _ = T(lambda: np.unique(packed, return_index=True, return_inverse=True)); print(f"  np.unique                  {ms:7.2f} ms")
ms, _ = T(lambda: predicted_events(pop, N)); print(f"  predicted_events           {ms:7.2f} ms")
ms, _ = T(lambda: evaluation_order(pop)); print(f"  evaluation_order           {ms:7.2f} ms")
ms, plan = T(lambda: sw.plan(pop)); print(f"  plan (incl. the above)     {ms:7.2f} ms")
indiv = torch.from_numpy(packed.view(np.uint8)).cuda(); fit = torch.empty(POP, dtype=torch.float64, device="cuda")
ms, _ = T(lambda: sw.evaluate_device(indiv, None, POP, fit, plan=plan)); print(f"  evaluate_device            {ms:7.2f} ms")
