#!/usr/bin/env python
"""Wall time of GA generations at a BASELINE config (default C5 shrunk to one GPU: pop 10000 x 50 symbols x 1M bars).

    python tools/ga_generation.py [--pop 10000] [--symbols 50] [--bars 1000000] [--generations 3] [--mode auto]

Prints one JSON line: per-generation wall time split into the device fitness sweep (CUDA events), host decode /
planning, and the reference-compatible host GA operators (selection, crossover, mutation).  Under torchrun the
population is sharded over ranks (ShardedFitness, one all-gather per generation).
"""
import argparse, json, os, time
import numpy as np, torch
import harness
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.dist import ShardedFitness
from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, GeneticAlgorithm
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep

ap = argparse.ArgumentParser()
ap.add_argument("--pop", type=int, default=10000)
ap.add_argument("--symbols", type=int, default=50)
ap.add_argument("--bars", type=int, default=1_000_000)
ap.add_argument("--generations", type=int, default=3)
ap.add_argument("--mode", default="auto")
ap.add_argument("--device-ga", action="store_true", help="GA operators on the GPU (DeviceGeneticAlgorithm)")
a = ap.parse_args()

world = int(os.environ.get("WORLD_SIZE", 1)); rank = int(os.environ.get("RANK", 0))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
if world > 1:
    torch.distributed.init_process_group("nccl")
t0 = time.perf_counter()
market = MarketData(synth.synth_ohlcv(a.symbols, a.bars))
t1 = time.perf_counter()
sweep = PopulationSweep(market, mode=a.mode)
torch.cuda.synchronize(); t2 = time.perf_counter()
fit = ShardedFitness(sweep.evaluate, device=market.device)
sweep_ms = []; diag = []
def batch(population):
    out = []
    w0 = time.perf_counter()
    [ms] = harness.event_ms(lambda: out.append(fit.batch(population)), 1, warmup=0)
    sweep_ms.append((ms, (time.perf_counter() - w0) * 1e3))
    diag.append({"unique": sweep.last_unique, "invalid_lanes": getattr(sweep, "last_invalid_lanes", 0),
                 "pool_overflow": getattr(sweep, "last_pool_overflow", False),
                 "records": float(sweep._stats[:, :, 0].sum().item())})
    return out[0]
def one(ind): return batch([ind])[0]
one.batch = batch
if a.device_ga:
    ga = DeviceGeneticAlgorithm(synth.param_ranges(False), batch, population_size=a.pop, generations=a.generations, random_seed=42)
else:
    ga = GeneticAlgorithm(synth.param_ranges(False), one, population_size=a.pop, generations=a.generations, random_seed=42)
w = time.perf_counter()
best = ga.run()
total = time.perf_counter() - w
if rank == 0:
    evals = (a.generations + 1)
    dev = [m[0] for m in sweep_ms]; wall = [m[1] for m in sweep_ms]
    per_gen = total / evals
    print(json.dumps({"workload": f"GA: pop {a.pop} x {a.symbols} symbols x {a.bars} bars, {a.generations} generations (+1 initial evaluation)",
                      **harness.card(), "n_gpus": world, "generation_wall_s": per_gen, "fitness_device_ms": dev, "fitness_wall_ms": wall,
                      "host_operator_s_per_generation": (total - sum(wall) / 1e3) / max(1, a.generations),
                      "bar_strategy_evals_per_generation": a.pop * a.symbols * a.bars,
                      "evals_per_s_in_sweep": a.pop * a.symbols * a.bars / (np.median(dev) * 1e-3),
                      "setup_s": {"synthetic_data": t1 - t0, "upload_and_rsi_bank": t2 - t1},
                      "per_evaluation": diag, "best_fitness": ga.best_fitness, "mode": a.mode,
                      "ga_operators": "device (csrc/ga_ops.cu)" if a.device_ga else "host (reference random stream)"}))
if world > 1:
    torch.distributed.destroy_process_group()
