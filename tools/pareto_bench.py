#!/usr/bin/env python
"""Cost of the multi-objective ranking (csrc/pareto.cu) and of one NSGA-II generation.

    python tools/pareto_bench.py [--reps 5] [--skip-generation] [--c4]

* b200bt_pareto_rank alone at n in {2047, 19999, 65536} x M in {2, 4} on uniform, anti-correlated (one large front) and
  chain (perfectly correlated: n fronts, the worst case of the peel) inputs, and at M = 8 on all-equal rows (one front of
  n points, the worst case of the crowding and order scans): CUDA events, median after a warm-up call, and the split into
  its kernels (dominance, peel, crowding, order, ...) from one torch.profiler run per case;
* the vectorised NumPy form of the same contract (tests/pareto_ref.pareto_numpy) at n = 2047 and 19999: host time, what
  the kernels replace;
* one NSGA-II generation (ParetoGeneticAlgorithm) at configs[1] size (1024 individuals x 10 symbols x 1M 1-minute bars,
  R = 2047 rows) split into operators, sweep + objective matrix, rank and survivor gather, alternated with one
  DeviceGeneticAlgorithm generation on the same market; with --c4 the same at configs[4] size (10 000 x 50 x 1M).
Prints one JSON line with the card's name and power limit.  Needs an H100; no fallback.
"""
import argparse
import json
import sys
import time

import numpy as np
import torch

import harness

sys.path.insert(0, str(harness.ROOT / "tests"))        # pareto_ref: the NumPy form of the ranking contract


def _time(fn, reps):
    ms = harness.event_ms(fn, reps)
    return {"ms_median": float(np.median(ms)), "ms_min": float(min(ms)), "ms_max": float(max(ms))}


def _kernel_split(fn):
    """Device time per kernel name (ms) of one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "pareto" in ev.name:
            name = ev.name.split("(")[0].replace("void ", "").replace("b200bt::", "").split("<")[0]
            split[name] = split.get(name, 0.0) + ev.device_time_total / 1e3
    return {k: round(v, 4) for k, v in split.items()}


def rank_leg(reps):
    import pareto_ref as pr
    from ai_crypto_trader_b200.pareto import ParetoRanker
    out = {}
    ranker = ParetoRanker()
    cases = [(n, M, kind) for n in (2047, 19999, 65536) for M in (2, 4) for kind in ("uniform", "anti", "chain")]
    cases += [(n, 8, "equal") for n in (2047, 19999, 65536)]        # one front of n points: the crowding scan's worst case
    for n, M, kind in cases:
        obj, mx = pr.make_input(kind, n, M)
        x = torch.from_numpy(obj).cuda()
        fn = lambda: ranker.rank(x, mx, with_key=True)
        t = _time(fn, reps)
        front = fn()[0]
        t["fronts"] = int(front.max().item()) + 1
        t["kernels_ms"] = _kernel_split(fn)
        out[f"n={n},M={M},{kind}"] = t
    return out


def host_leg():
    import pareto_ref as pr
    out = {}
    for n, M in ((2047, 2), (2047, 4), (19999, 4)):
        obj, mx = pr.make_input("uniform", n, M)
        t = time.perf_counter()
        pr.pareto_numpy(obj, mx)
        out[f"n={n},M={M},uniform"] = {"host_ms": (time.perf_counter() - t) * 1e3}
    return out


def generation_leg(pop, symbols, bars, rounds):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, ParetoGeneticAlgorithm
    from ai_crypto_trader_b200.pareto import objectives_from_goals
    from ai_crypto_trader_b200.sweep import DEFAULT_GOALS, MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(symbols, bars))
    ranges = synth.param_ranges()
    sweep = PopulationSweep(market)
    objectives = objectives_from_goals(DEFAULT_GOALS)
    nsga = ParetoGeneticAlgorithm(ranges, lambda p: sweep.evaluate_objectives_device(p, objectives), objectives,
                                  population_size=pop, generations=0, random_seed=42)
    nsga.initialize_population()
    nsga.evaluate_population()
    scalar = DeviceGeneticAlgorithm(ranges, sweep.evaluate, population_size=pop, generations=0, random_seed=42)
    scalar.initialize_population()
    scalar.evaluate_population()
    lib = nsga._lib
    rows = {"nsga2": [], "device_ga": []}
    gen = 1
    for _ in range(rounds):
        # NSGA-II, the steps of ParetoGeneticAlgorithm.evolve_generation timed one by one
        def operators():
            lib.call("b200bt_ga_next_generation", nsga.params.data_ptr(), nsga._key.data_ptr(), nsga._ranked.data_ptr(),
                     pop, len(nsga.names), nsga._lo, nsga._hi, nsga._is_int, 0.0, nsga.tournament_size,
                     nsga.crossover_rate, nsga.mutation_rate, nsga.seed, gen, nsga._sel.data_ptr(), nsga._next.data_ptr(),
                     lib.current_stream())
        [t_ops], _ = harness.wall_ms(operators)
        q = nsga._next[1:]
        [t_sweep], fq = harness.wall_ms(lambda: nsga._evaluate_rows(q))
        R = torch.cat([nsga.params, q])
        FR = torch.cat([nsga._obj, fq])
        [t_rank], (front, crowd, order, _) = harness.wall_ms(lambda: nsga._ranker.rank(FR, nsga.maximize))

        def gather():
            keep = order[:pop].long()
            nsga.params = R.index_select(0, keep)
            nsga._obj = FR.index_select(0, keep)
            nsga._front, nsga._crowding = front.index_select(0, keep), crowd.index_select(0, keep)
        [t_gather], _ = harness.wall_ms(gather)
        rows["nsga2"].append({"operators_ms": t_ops, "sweep_and_objectives_ms": t_sweep, "rank_ms": t_rank,
                              "survivor_gather_ms": t_gather, "total_ms": t_ops + t_sweep + t_rank + t_gather})
        # the scalar device GA, one generation: operators + sweep of the whole population
        [t_scalar], _ = harness.wall_ms(lambda: (scalar.evolve_generation(gen), scalar.evaluate_population()))
        rows["device_ga"].append({"total_ms": t_scalar})
        gen += 1
    med = lambda key, part: float(np.median([r[part] for r in rows[key]]))
    summary = {"nsga2_median_ms": {p: med("nsga2", p) for p in rows["nsga2"][0]},
               "device_ga_median_ms": med("device_ga", "total_ms")}
    summary["ranking_share_of_nsga2_generation"] = (summary["nsga2_median_ms"]["rank_ms"]
                                                    + summary["nsga2_median_ms"]["survivor_gather_ms"]) / \
        summary["nsga2_median_ms"]["total_ms"]
    return {"workload": f"population {pop} x {symbols} symbols x {bars} 1-minute bars, R = {2 * pop - 1} rows",
            "rounds": rows, **summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-generation", action="store_true")
    ap.add_argument("--c4", action="store_true", help="also the configs[4] generation (10 000 x 50 x 1M)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pareto_bench needs a CUDA device (H100); there is no CPU path")
    torch.cuda.set_device(0)
    out = {**harness.card(), "rank": rank_leg(a.reps), "host_numpy": host_leg()}
    if not a.skip_generation:
        out["generation_configs1"] = generation_leg(1024, 10, 1_000_000, a.rounds)
        if a.c4:
            out["generation_configs4"] = generation_leg(10_000, 50, 1_000_000, a.rounds)
        else:
            out["generation_configs4"] = "not measured"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
