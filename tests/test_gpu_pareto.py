"""Multi-objective ranking on the GPU (csrc/pareto.cu) against its host restatement (tests/pareto_ref.py), bit for bit:
fronts, crowding (+inf included), crowded order and tournament key; the objective matrix against the lane and book stats;
NSGA-II generations of ParetoGeneticAlgorithm against tests/ga_ref.py and the oracle; StrategyEvolutionService.optimize_pareto."""
import asyncio

import numpy as np
import pytest
import torch

import ga_ref
import pareto_ref as pr

pytestmark = pytest.mark.gpu

REFERENCE_GOALS = {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]}
EXACT_MAX = 2047


def _rank_on_device(obj, maximize):
    from ai_crypto_trader_b200.pareto import pareto_rank
    dev = torch.from_numpy(np.ascontiguousarray(obj)).cuda()
    front, crowd, order, key = pareto_rank(dev, maximize, with_key=True)
    return tuple(t.cpu().numpy() for t in (front, crowd, order, key))


def _check(obj, maximize, label):
    want = (pr.pareto_exact if obj.shape[0] <= EXACT_MAX else pr.pareto_numpy)(obj, maximize)
    got = _rank_on_device(obj, maximize)
    for name, a, b in zip(("front", "crowding", "order", "key"), got, want):
        assert a.dtype == b.dtype and a.shape == b.shape, (name, label)
        if a.tobytes() != b.tobytes():
            ai, bi = (a.view(np.int64), b.view(np.int64)) if a.dtype == np.float64 else (a, b)
            diff = np.flatnonzero(ai != bi)
            pytest.fail(f"{label}: {name} differs at {len(diff)} places, first {diff[:4].tolist()}: "
                        f"{a[diff[:4]].tolist()} vs {b[diff[:4]].tolist()}")


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33])
def test_rank_small(kind, M, n):
    obj, mx = pr.make_input(kind, n, M)
    _check(obj, mx, (kind, n, M))


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [1000, 2047])
def test_rank_medium(kind, n, M):
    obj, mx = pr.make_input(kind, n, M)
    _check(obj, mx, (kind, n, M))


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 4, 8])
def test_rank_4101(kind, M):
    obj, mx = pr.make_input(kind, 4101, M)
    _check(obj, mx, (kind, 4101, M))


@pytest.mark.parametrize("kind,n,M", [("uniform", 19999, 4), ("anti", 19999, 2), ("chain", 19999, 1),
                                      ("chain", 19999, 3), ("ties", 19999, 3), ("nonfinite", 19999, 2),
                                      ("mixed", 19999, 8), ("equal", 19999, 4),
                                      ("uniform", 65536, 2), ("anti", 65536, 2), ("ties", 65536, 3),
                                      ("nonfinite", 65536, 4), ("mixed", 65536, 4)])
def test_rank_large(kind, n, M):
    obj, mx = pr.make_input(kind, n, M)
    _check(obj, mx, (kind, n, M))


def test_rank_is_deterministic_and_reuses_its_workspace():
    from ai_crypto_trader_b200.pareto import ParetoRanker
    obj, mx = pr.make_input("ties", 4101, 3)
    dev = torch.from_numpy(obj).cuda()
    r = ParetoRanker()
    first = [t.cpu().numpy() for t in r.rank(dev, mx, with_key=True)]
    for _ in range(3):
        again = [t.cpu().numpy() for t in r.rank(dev, mx, with_key=True)]
        assert all(a.tobytes() == b.tobytes() for a, b in zip(first, again))


def test_rank_reads_a_strided_matrix():
    obj, mx = pr.make_input("uniform", 500, 3)
    wide = torch.zeros((500, 7), dtype=torch.float64, device="cuda")
    wide[:, 2:5] = torch.from_numpy(obj).cuda()
    from ai_crypto_trader_b200.pareto import pareto_rank
    got = [t.cpu().numpy() for t in pareto_rank(wide[:, 2:5], mx, with_key=True)]
    for a, b in zip(got, pr.pareto_exact(obj, mx)):
        assert a.tobytes() == b.tobytes()


# -- objective matrix ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def market():
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    torch.cuda.set_device(0)
    return MarketData(synth.synth_ohlcv(3, 20000, seed_base=77))


def _population(n, seed):
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(n, seed=seed)
    return pop + [dict(pop[1]), dict(pop[5])]           # two duplicates: the deduplicated path


def test_objective_matrix_equals_fitness_and_lane_means(market):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import PopulationSweep
    sweep = PopulationSweep(market)
    pop = _population(96, 11)
    fitness = sweep.evaluate(pop)
    score = sweep.evaluate_objectives(pop, [("score", True)])
    assert score.shape == (len(pop), 1) and score[:, 0].tobytes() == fitness.tobytes()
    fields = list(_lib.LANE_STATS_FIELDS[:-1])
    for lo in range(0, len(fields), 8):
        names = fields[lo:lo + 8]
        got = sweep.evaluate_objectives(pop, [(n, True) for n in names])
        st = sweep.lane_stats()
        for j, name in enumerate(names):
            acc = np.zeros(len(pop))
            for s in range(market.S):
                acc = acc + st[name][:, s]
            want = acc / market.S
            assert got[:, j].tobytes() == want.tobytes(), name


def test_objective_matrix_of_the_book(market):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    sweep = PopulationSweep(market, aggregation="book")
    pop = _population(64, 12)
    names = ["sharpe_ratio", "max_drawdown", "win_rate", "profit_factor", "net_profit", "n_records"]
    got = sweep.evaluate_objectives(pop, [(n, n != "max_drawdown") for n in names])
    book = sweep.book_stats()
    for j, name in enumerate(names):
        assert got[:, j].tobytes() == np.ascontiguousarray(book[name]).tobytes(), name


# -- NSGA-II -------------------------------------------------------------------------------------------------------------
def _ga(market, seed=9, N=64, generations=5):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import ParetoGeneticAlgorithm
    from ai_crypto_trader_b200.pareto import objectives_from_goals
    from ai_crypto_trader_b200.sweep import PopulationSweep
    ranges = synth.param_ranges()
    sweep = PopulationSweep(market, rsi_periods=range(int(ranges["rsi_period"][0]), int(ranges["rsi_period"][1]) + 1))
    objectives = objectives_from_goals(REFERENCE_GOALS)
    ga = ParetoGeneticAlgorithm(ranges, lambda p: sweep.evaluate_objectives_device(p, objectives), objectives,
                                population_size=N, generations=generations, random_seed=seed)
    return ga, sweep, objectives


def _dominates(a, b):
    return bool(np.all(a >= b) and np.any(a > b))


def test_generations_against_the_oracle(market):
    ga, sweep, objectives = _ga(market)
    N, mx = ga.population_size, ga.maximize
    lo, hi, is_int = list(ga._lo), list(ga._hi), list(ga._is_int)
    ga.initialize_population()
    p0 = ga.params.cpu().numpy()
    f0 = sweep.evaluate_objectives(ga._to_dicts(p0), objectives)
    ga.evaluate_population()
    _, _, order, _ = pr.pareto_exact(f0, mx)
    assert ga.params.cpu().numpy().tobytes() == p0[order].tobytes()
    assert ga._obj.cpu().numpy().tobytes() == f0[order].tobytes()
    for t in range(1, 6):
        P, FP = ga.params.cpu().numpy(), ga._obj.cpu().numpy()
        ga.evolve_generation(t)
        Q = ga.last_offspring.cpu().numpy()
        _, want_q = ga_ref.next_generation(P, -np.arange(N, dtype=np.float64), np.arange(N, dtype=np.int32), lo, hi,
                                           is_int, 0.0, ga.tournament_size, ga.crossover_rate, ga.mutation_rate, ga.seed, t)
        assert Q.tobytes() == want_q.tobytes(), t
        FR = ga.last_objectives_R.cpu().numpy()
        assert FR.shape == (2 * N - 1, len(objectives))
        assert FR[:N].tobytes() == FP.tobytes()                       # the parents are not re-evaluated
        R = np.concatenate([P, Q[1:]])
        _, _, order, _ = pr.pareto_exact(FR, mx)
        assert ga.params.cpu().numpy().tobytes() == R[order[:N]].tobytes(), t
        assert ga._obj.cpu().numpy().tobytes() == FR[order[:N]].tobytes(), t


def test_run_is_reproducible_and_its_front_is_non_dominated(market):
    ga, sweep, objectives = _ga(market, seed=21)
    front = ga.run()
    again, _, _ = _ga(market, seed=21)
    again.run()
    assert again.population == ga.population
    assert again.objective_values.tobytes() == ga.objective_values.tobytes()
    assert again.front.tobytes() == ga.front.tobytes() and again.crowding.tobytes() == ga.crowding.tobytes()
    assert len(front) >= 1 and len(ga.generation_history) == 6
    assert all(h["front0_size"] >= 1 and h["n_fronts"] >= 1 for h in ga.generation_history)
    v = pr.values(np.array([[m["objectives"][n] for n, _ in objectives] for m in front]), ga.maximize)
    for a in range(len(v)):
        for b in range(len(v)):
            assert not _dominates(v[a], v[b])
    rows = sweep.evaluate_objectives([m["parameters"] for m in front], objectives)
    want = np.array([[m["objectives"][n] for n, _ in objectives] for m in front])
    assert rows.tobytes() == want.tobytes()
    assert ga.best_individual in [m["parameters"] for m in front]
    best0 = max(pr.values(want, ga.maximize)[:, 0])
    first = next(m for m in front if pr.values(np.array([[m["objectives"][n] for n, _ in objectives]]), ga.maximize)[0, 0]
                 == best0)
    assert ga.best_individual == first["parameters"]


def test_optimize_pareto_with_the_reference_goals(market):
    from ai_crypto_trader_b200.evolution import StrategyEvolutionService
    svc = StrategyEvolutionService(market, config={"evolution": {"optimization_goals": REFERENCE_GOALS}}, random_seed=4)
    front = asyncio.run(svc.optimize_pareto({"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30}))
    assert front
    for m in front:
        assert set(m["objectives"]) == {"sharpe_ratio", "max_drawdown", "win_rate", "profit_factor"}
        for name, (lo, hi) in svc.param_ranges.items():
            assert lo <= m["parameters"][name] <= hi, name
    rec = svc.evolution_records[-1]
    assert rec["algorithm"] == "nsga2" and rec["front_size"] == len(front)
