#!/usr/bin/env python
"""One device-resident sweep of the configs[1] workload on the generation-3 population of a GA run (the population
bench.py's `evolved_population_value` times), for a launch list:
    ncu --metrics gpu__time_duration.sum --clock-control none -k regex:'lane_scan|chunk_|lane_combine|sweep_kernel' python tools/evolved_profile.py"""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np, torch
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep, decode_population
S, N, POP = 10, 1_000_000, 1024
m = MarketData(synth.synth_ohlcv(S, N)); sw = PopulationSweep(m)
pop = synth.random_population(POP, seed=42)
ga = GeneticAlgorithm(synth.param_ranges(), sw.fitness_function, population_size=POP, generations=3, random_seed=42)
ga.run(seeded_individuals=pop)
ev = ga.population
indiv = torch.from_numpy(decode_population(ev, sw.period_row).view(np.uint8)).cuda()
fit = torch.empty(POP, dtype=torch.float64, device="cuda")
plan = sw.plan(ev)
torch.cuda.synchronize()
print("PROFILE_START", flush=True)
for _ in range(2):
    sw.evaluate_device(indiv, None, POP, fit, plan=plan)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    sw.evaluate_device(indiv, None, POP, fit, plan=plan)
e1.record(); torch.cuda.synchronize()
print("ms per sweep (CUDA events, 5 sweeps)", e0.elapsed_time(e1) / 5, "invalid lanes", sw.last_invalid_lanes, "overflow", sw.last_pool_overflow,
      "pool blocks", [p.pool_blocks for p in plan], "used", [int(p.overflow[2]) for p in plan], "pool factor", sw._pool_factor)
import time
t0 = time.perf_counter()
for _ in range(5):
    sw.evaluate_device(indiv, None, POP, fit, plan=plan)
t1 = time.perf_counter(); torch.cuda.synchronize(); t2 = time.perf_counter()
print("host enqueue ms per sweep", (t1 - t0) / 5 * 1e3, "until done", (t2 - t0) / 5 * 1e3)
st = sw.lane_stats()
print("records", float(st["n_records"].sum()), "K", plan[0].K, "unique rows", len({p['rsi_period'] for p in ev}))
