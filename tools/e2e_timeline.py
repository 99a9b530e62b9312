#!/usr/bin/env python
"""Host timeline of one end-to-end generation (bench.py's e2e leg) without intermediate synchronisation:
when does the host reach each point, and when is the device done."""
import time
import numpy as np, torch
import harness
from ai_crypto_trader_b200 import synth, sweep as sw_mod
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
S, N, POP = 10, 1_000_000, 1024
ohlcv_host = torch.from_numpy(synth.synth_ohlcv(S, N)).pin_memory()
pop = synth.random_population(POP, seed=42)
print(", ".join(harness.card().values()))
marks = []
def mark(name): marks.append((name, time.perf_counter()))
orig_plan, orig_dev, orig_decode = PopulationSweep.plan, PopulationSweep.evaluate_device, sw_mod.decode_population
def plan(self, p, **kw):
    mark("plan begin"); r = orig_plan(self, p, **kw); mark("plan end"); return r
def evd(self, *a, **k):
    mark("launch begin"); r = orig_dev(self, *a, **k); mark("launch end"); return r
def dec(*a, **k):
    mark("decode begin"); r = orig_decode(*a, **k); mark("decode end"); return r
PopulationSweep.plan, PopulationSweep.evaluate_device, sw_mod.decode_population = plan, evd, dec
def step():
    marks.clear(); mark("start")
    mk = MarketData(ohlcv_host); mark("MarketData returned")
    sw = PopulationSweep(mk); mark("PopulationSweep returned")
    f = sw.evaluate(pop); mark("evaluate returned")
    torch.cuda.synchronize(); mark("device idle")
for _ in range(3): step()
t0 = marks[0][1]
for name, t in marks: print(f"{(t - t0) * 1e3:8.2f} ms  {name}")

# where do the extra ~2 ms of the sweep inside the e2e step come from?
def timed(fn, n=5):
    return float(np.mean(harness.wall_ms(fn, n, warmup=1)[0]))
PopulationSweep.plan, PopulationSweep.evaluate_device, sw_mod.decode_population = orig_plan, orig_dev, orig_decode
mk = MarketData(ohlcv_host); sw = PopulationSweep(mk); sw.use_zones = False
print(f"evaluate() on a resident market / bank, no zone map : {timed(lambda: sw.evaluate(pop)):6.2f} ms")
dev_ohlcv = mk.ohlcv.clone()
print(f"MarketData(device tensor) + bank + evaluate          : {timed(lambda: PopulationSweep(MarketData(dev_ohlcv)).evaluate(pop)):6.2f} ms")
print(f"MarketData(pinned host) + bank + evaluate            : {timed(lambda: PopulationSweep(MarketData(ohlcv_host)).evaluate(pop)):6.2f} ms")
pinned_close = ohlcv_host[3]
def close_copy():
    c = torch.empty((S, N), dtype=torch.float32, device="cuda")
    c.copy_(pinned_close, non_blocking=True)
    return c
def close_and_bank(): return PopulationSweep(MarketData.from_close(close_copy()))
def close_only_step(): return close_and_bank().evaluate(pop)
print(f"pinned close only (40 MB) + bank + evaluate          : {timed(close_only_step):6.2f} ms")

# device time from the start of the step to the end of each of its prefixes, no synchronisation inside a prefix
r = [harness.event_ms(f, 1, warmup=2)[0] for f in (close_copy, close_and_bank, close_only_step)]
r.append(harness.wall_ms(close_only_step, 1, warmup=2)[0][0])
print("device timeline (ms since start): close copied %.2f, bank built %.2f, sweep done %.2f; wall %.2f" % tuple(r))
