#!/usr/bin/env python
"""Critical-path probe for the sweep kernel: time a single heavy / mid / light lane alone,
then one CTA and a full grid of heavy lanes (1M bars).  The heaviest lane's serial event chain is
the floor of the kernel time at small populations."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep

m = MarketData(synth.synth_ohlcv(1, 1_000_000))
sw = PopulationSweep(m)


def t(pop):
    sw.evaluate(pop); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); sw.evaluate(pop); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)


heavy = dict(synth.random_population(1, seed=1)[0], rsi_period=5, rsi_oversold=35, rsi_overbought=65, take_profit=1, stop_loss=1)
light = dict(heavy, rsi_period=30, rsi_oversold=15, rsi_overbought=85)
mid = dict(heavy, rsi_period=14, rsi_oversold=30, rsi_overbought=70)
for name, p in (("heavy", heavy), ("mid", mid), ("light", light)):
    ms = t([p]); n = sw.lane_stats()["n_records"][0, 0]
    print(f"{name:6s} single lane {ms:7.2f} ms  records {int(n):7d}  {ms * 1e6 / max(n, 1):7.1f} ns/event")
print("8 heavy lanes (1 CTA)      %.2f ms" % t([heavy] * 8))
sms = torch.cuda.get_device_properties(0).multi_processor_count
print("%d*16 heavy lanes (1 wave) %.2f ms" % (sms, t([heavy] * (sms * 16))))
print("%d*16 light lanes (1 wave) %.2f ms" % (sms, t([light] * (sms * 16))))
