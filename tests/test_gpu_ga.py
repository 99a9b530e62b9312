"""GA operators on the device (SURVEY 8-f2): distribution-level parity with the reference-compatible host operators,
determinism, elitism, range / integrality invariants, and a real optimisation run on the sweep."""
import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu


def _toy_fitness(population):
    # smooth, deterministic, all genes matter a little
    return [float(-(p["rsi_period"] - 17) ** 2 - 3.0 * (p["bollinger_std"] - 2.2) ** 2 + 0.01 * p["ema_long"]) for p in population]


def test_device_ga_invariants_and_determinism(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, _is_int_range
    ranges = synth.param_ranges()
    runs = []
    for _ in range(2):
        ga = DeviceGeneticAlgorithm(ranges, _toy_fitness, population_size=257, generations=6, random_seed=99)
        best = ga.run(seeded_individuals=[{"rsi_period": 400, "bollinger_std": -5.0}])      # clamped (:96-103)
        runs.append((best, [h["best_fitness"] for h in ga.get_generation_history()], ga.params.cpu().numpy().copy()))
        assert ga.population[0]["rsi_period"] >= 5
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1] and np.array_equal(runs[0][2], runs[1][2])
    hist = runs[0][1]
    assert all(b >= a for a, b in zip(hist, hist[1:])), "elitism keeps the best individual"
    assert hist[-1] > hist[0]
    final = runs[0][2]
    for g, name in enumerate(ranges):
        lo, hi = ranges[name]
        assert final[:, g].min() >= lo and final[:, g].max() <= hi, name
        if _is_int_range(lo, hi):
            assert np.array_equal(final[:, g], np.round(final[:, g])), name
    other = DeviceGeneticAlgorithm(ranges, _toy_fitness, population_size=257, generations=6, random_seed=100)
    other.run()
    assert not np.array_equal(other.params.cpu().numpy(), final)


def test_device_operators_match_host_operator_statistics(torch_cuda):
    """One generation from the same population and fitness: the device operators and the reference-compatible host
    operators (ai_crypto_trader_b200.genetic_algorithm.GeneticAlgorithm) agree on selection pressure, on how often a
    gene of an offspring differs from both candidate parents' values (mutation), and on mutation step sizes."""
    import random
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, GeneticAlgorithm
    ranges = synth.param_ranges()
    names = list(ranges)
    pop_n = 4000
    host = GeneticAlgorithm(ranges, lambda ind: 0.0, population_size=pop_n, generations=1, random_seed=5)
    host.initialize_population()
    base = [dict(p) for p in host.population]
    rng = np.random.default_rng(1)
    fitness = rng.standard_normal(pop_n).tolist()
    host.fitness_scores = list(fitness)
    random.seed(11)
    host.evolve_generation()
    host_next = np.array([[float(p[n]) for n in names] for p in host.population])

    dev = DeviceGeneticAlgorithm(ranges, lambda population: fitness, population_size=pop_n, generations=1, random_seed=7)
    dev.params.copy_(torch.from_numpy(np.array([[float(p[n]) for n in names] for p in base])).to(dev.device))
    dev.population, dev.fitness_scores = base, list(fitness)
    dev.evolve_generation(1)
    dev_next = dev.params.cpu().numpy()
    sel = dev._sel.cpu().numpy()

    base_m = np.array([[float(p[n]) for n in names] for p in base])
    n_elite = max(1, int(0.1 * pop_n))
    ranked = np.argsort(-np.array(fitness), kind="stable")
    # elites: identical rows, in rank order, on both sides
    assert np.array_equal(dev_next[:n_elite], base_m[ranked[:n_elite]])
    assert np.array_equal(host_next[:n_elite], base_m[ranked[:n_elite]])
    assert np.array_equal(sel[:n_elite], ranked[:n_elite])
    # tournament of 3 distinct: P(winner has rank r) = C(n-1-r, 2) / C(n, 3); compare the mean winner rank
    rank_of = np.empty(pop_n, dtype=np.int64)
    rank_of[ranked] = np.arange(pop_n)
    mean_rank = rank_of[sel[n_elite:]].mean()
    assert mean_rank == pytest.approx((pop_n - 3) / 4, rel=0.05)
    # mutation: a gene value found in no individual of the previous generation at that gene must come from mutation.
    # float genes almost surely change when mutated -> rate ~ 0.2; compare device and host on the same statistic.
    for g, name in enumerate(names):
        col_prev = set(base_m[:, g].tolist())
        novel_dev = np.mean([v not in col_prev for v in dev_next[n_elite:, g]])
        novel_host = np.mean([v not in col_prev for v in host_next[n_elite:, g]])
        assert novel_dev == pytest.approx(novel_host, abs=0.03), (name, novel_dev, novel_host)
    for g, name in enumerate(names):            # integer genes move by exactly +-max(1, int(0.1 range)) when they move
        lo, hi = ranges[name]
        if isinstance(lo, int) and isinstance(hi, int):
            step = max(1, int((hi - lo) * 0.1))
            vals = set(base_m[:, g].tolist())
            moved = [v for v in dev_next[n_elite:, g] if v not in vals]
            assert all(lo <= v <= hi for v in moved)
            assert all(((v - step) in vals) or ((v + step) in vals) or v in (lo, hi) for v in moved), name


def test_device_ga_on_the_sweep(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(2, 30_000))
    sweep = PopulationSweep(market)
    ga = DeviceGeneticAlgorithm(synth.param_ranges(), sweep.evaluate, population_size=96, generations=4, random_seed=3)
    best = ga.run()
    hist = [h["best_fitness"] for h in ga.get_generation_history()]
    assert len(hist) == 5 and all(b >= a for a, b in zip(hist, hist[1:]))
    assert ga.best_fitness == max(hist) and set(best) == set(synth.param_ranges())
    assert float(sweep.evaluate([best])[0]) == pytest.approx(ga.best_fitness, rel=1e-9)
