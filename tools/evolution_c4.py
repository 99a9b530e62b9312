#!/usr/bin/env python
"""BASELINE configs[3]: the strategy-evolution loop -- 100 generations, population 4096, 20 symbols x 1M 1-minute bars,
RSI indicators on the 1m / 5m / 15m timeframes, on 1..8 H100 (torchrun: individuals sharded by rank, one all-gather per
generation, GA operators on the device).

    python tools/evolution_c4.py [--generations 100] [--population 4096] [--symbols 20] [--bars 1000000]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/evolution_c4.py

The loop is the reference's (services/strategy_evolution_service.py:644-655: GeneticAlgorithm(...).run(seeded=[current]))
with the fitness the reference composes in cross_validate_strategy (simulate -> metrics -> score, mean over symbols) and
the multi-timeframe indicator recipe of services/market_monitor_service.py:219-301: the gene `rsi_timeframe` selects which
clock's RSI row the entry / exit rule reads.  Prints one JSON object (rank 0): wall seconds of the whole loop and per
generation, the best fitness trajectory, and the record count of the last population.
"""
import argparse
import json
import os
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import numpy as np
import torch
import torch.distributed as dist


def run(generations=100, population=4096, symbols=20, bars=1_000_000, timeframes=(1, 5, 15), seed=42, device=None,
        operators="device"):
    """-> dict (identical on every rank).  Callable from bench.py with the process group already initialised."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.dist import ShardedFitness
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, GeneticAlgorithm
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    world = dist.get_world_size() if dist.is_initialized() else 1
    dev = device or torch.device("cuda", torch.cuda.current_device())

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    t_setup = time.perf_counter()
    market = MarketData(synth.synth_ohlcv(symbols, bars))
    sweep = PopulationSweep(market, timeframes=timeframes)             # RSI banks on every timeframe, aligned to the base clock
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t_setup
    ranges = dict(synth.param_ranges(), rsi_timeframe=(0, len(timeframes) - 1))
    fit = ShardedFitness(sweep.evaluate, device=dev)
    cls = DeviceGeneticAlgorithm if operators == "device" else GeneticAlgorithm
    ga = cls(ranges, fit, population_size=population, generations=generations, random_seed=seed)
    gen_s, unique = [], []
    barrier()
    t0 = time.perf_counter()
    ga.initialize_population()
    ga.evaluate_population()
    ga.record_generation(0)
    torch.cuda.synchronize()
    gen_s.append(time.perf_counter() - t0)
    unique.append(int(sweep.last_unique))
    for g in range(1, generations + 1):
        t1 = time.perf_counter()
        ga.evolve_generation(g) if operators == "device" else ga.evolve_generation()
        ga.evaluate_population()
        ga.record_generation(g)
        torch.cuda.synchronize()
        gen_s.append(time.perf_counter() - t1)
        unique.append(int(sweep.last_unique))
    barrier()
    total = time.perf_counter() - t0
    t = torch.tensor([total], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    hist = ga.get_generation_history()
    return {
        "workload": f"evolution loop: {generations} generations, population {population}, {symbols} symbols x {bars} 1-min bars, RSI on {'/'.join(str(k) + 'm' for k in timeframes)}",
        "n_gpus": world, "loop_s": float(t.item()), "per_generation_s": {"first": gen_s[0], "median": float(np.median(gen_s)), "last": gen_s[-1], "max": float(max(gen_s))},
        "setup_s": setup_s, "bank_rows": int(sweep.bank.shape[1]), "operators": operators,
        "best_fitness": [hist[0]["best_fitness"], hist[len(hist) // 2]["best_fitness"], hist[-1]["best_fitness"]],
        # the rule reads 7 of the 19 genes and the GA converges: individuals that decode to the same kernel parameters are
        # evaluated once (PopulationSweep.evaluate), so the bar-strategy evaluations actually computed are those of the
        # DISTINCT individuals of this rank's shard, summed over the generations
        "distinct_individuals_rank0": {"first": unique[0], "median": int(np.median(unique)), "last": unique[-1]},
        "evaluations_computed_rank0": int(sum(unique)) * symbols * bars,
        "evaluations_nominal": (generations + 1) * population * symbols * bars,
        "best_individual": ga.get_best_individual(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--generations", type=int, default=100)
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--symbols", type=int, default=20)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--operators", default="device", choices=["device", "host"])
    a = ap.parse_args()
    world, rank = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    out = run(a.generations, a.population, a.symbols, a.bars, operators=a.operators)
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
