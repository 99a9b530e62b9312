"""The device GA operators (csrc/ga_ops.cu) draw for draw against their NumPy restatement (tests/ga_ref.py): `sel` equal
and every float64 of params_out / the initial population bit-equal, over population shapes, elite counts, tournament
sizes, rates, gene sets, fitness ties and infinities, seeds and generations; then DeviceGeneticAlgorithm.run against
ga_ref.run generation by generation.  The C entry points are called directly, so ranked and fitness are the test's."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

import ga_ref
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

SEED = 0x9E3779B97F4A7C15                  # both key words non-zero


# -- gene sets ---------------------------------------------------------------------------------------------------------

def _from_ranges(ranges):
    lo = np.array([float(v[0]) for v in ranges.values()])
    hi = np.array([float(v[1]) for v in ranges.values()])
    is_int = np.array([isinstance(v[0], int) and isinstance(v[1], int) for v in ranges.values()])
    return lo, hi, is_int


def _wide64():
    """64 genes: integer spans 0, 1..9 (step 1), 10, 37 and 3 999 999 999 (just under the 4e9 limit); float genes with
    lo = hi, a negative range, ranges crossing 0, tiny and huge spans."""
    genes = [(5, 5, True), (-3, -3, True)] + [(k, k + k, True) for k in range(1, 10)] + \
            [(0, 10, True), (-20, 17, True), (-2_000_000_000, 1_999_999_999, True), (0, 3_999_999_999, True)] + \
            [(2.5, 2.5, False), (0.0, 0.0, False), (-7.5, -0.5, False), (-1.0, 2.0, False), (-1e-3, 1e6, False),
             (1e-9, 3e-9, False), (-1e12, 1e12, False), (0.1, 0.7, False), (-123.456, -0.001, False)]
    while len(genes) < 64:
        genes.append(genes[len(genes) % 24])
    lo, hi, is_int = zip(*genes)
    return np.array(lo, np.float64), np.array(hi, np.float64), np.array(is_int)


def _genes(name):
    from ai_crypto_trader_b200 import synth
    if name == "synth":
        return _from_ranges(synth.param_ranges(False))
    if name == "synth_leverage":
        return _from_ranges(synth.param_ranges(True))
    if name == "one_float":
        return np.array([-0.75]), np.array([3.25]), np.array([False])
    if name == "one_int":
        return np.array([2.0]), np.array([7.0]), np.array([True])
    if name == "wide64":
        return _wide64()
    raise ValueError(name)


def _fitness(kind, pop, seed):
    rng = np.random.default_rng(seed)
    f = rng.standard_normal(pop)
    if kind == "ties":                       # a handful of values shared by many individuals
        f = np.round(f * 2.0) / 2.0
    elif kind == "neginf":
        f[rng.random(pop) < 0.3] = -np.inf
        f[:: max(1, pop // 7)] = -np.inf
    elif kind == "equal":
        f = np.full(pop, 1.25)
    elif kind == "nan":                      # straight to the kernel: a NaN contender never beats the current best
        f[rng.random(pop) < 0.2] = np.nan
    return f


# -- cases -------------------------------------------------------------------------------------------------------------

def _case(name, pop=257, genes="synth", elitism=0.1, tournament=3, cx=0.8, mr=0.2, fitness="normal", seed=SEED,
          generation=1):
    return dict(name=name, pop=pop, genes=genes, elitism=elitism, tournament=tournament, cx=cx, mr=mr, fitness=fitness,
                seed=seed, generation=generation)


CASES = [
    *[_case(f"pop{p}", pop=p, tournament=min(3, p)) for p in (1, 2, 3, 127, 128, 129, 257)],
    _case("pop4096 (configs[3])", pop=4096),
    _case("pop10000 (configs[4])", pop=10_000),
    _case("one elite, elitism 0", pop=3, elitism=0.0, tournament=2),
    _case("one elite, elitism 0.05", pop=3, elitism=0.05, tournament=2),
    _case("all elites, elitism 1", pop=129, elitism=1.0),
    _case("all elites, elitism 1e300", pop=129, elitism=1e300),
    _case("pop-1 elites, second child dropped", pop=129, elitism=128.5 / 129),
    _case("pop-1 elites at 128", pop=128, elitism=127.5 / 128),
    _case("elitism 0.29 x 100 = 28.999...", pop=100, elitism=0.29),
    _case("tournament 1", tournament=1),
    _case("tournament 8", tournament=8),
    _case("tournament = pop = 2", pop=2, tournament=2, elitism=0.0),
    _case("tournament = pop = 3", pop=3, tournament=3, elitism=0.0),
    _case("tournament = pop = 8", pop=8, tournament=8, elitism=0.0),
    *[_case(f"crossover {cx}, mutation {mr}", cx=cx, mr=mr) for cx in (0.0, 0.8, 1.0) for mr in (0.0, 0.2, 1.0)],
    _case("one float gene", genes="one_float", mr=0.5),
    _case("one integer gene", genes="one_int", mr=0.5),
    _case("synth, leverage ranges", genes="synth_leverage", mr=0.5),
    _case("64 genes", pop=1000, genes="wide64", mr=0.5),
    _case("64 genes, all mutate", pop=300, genes="wide64", mr=1.0, cx=1.0, tournament=8),
    _case("fitness ties", fitness="ties", tournament=8),
    _case("fitness -inf", fitness="neginf"),
    _case("fitness all equal", fitness="equal", tournament=5),
    _case("fitness NaN", fitness="nan"),
    _case("seed 0, generation 0", seed=0, generation=0),
    _case("seed 2^64-1, generation 2^32-1", seed=(1 << 64) - 1, generation=(1 << 32) - 1),
    _case("high seed word only, generation 2", seed=7 << 32, generation=2),
    _case("rates equal a drawn uniform", cx="drawn", mr="drawn", genes="wide64"),
]


def _drawn_rates(case, n_elite):
    """crossover_rate = pair 0's crossover uniform, mutation_rate = the first mutation uniform of slot n_elite: at these
    rates pair 0 crosses only if the test is !(u > rate) and gene 0 of slot n_elite mutates only if it is u < rate."""
    s, g = case["seed"], case["generation"]
    parents = ga_ref.Words(s, g, [0], ga_ref.PARENTS)
    parents.next(), parents.next()
    cx = float(parents.uniform()[0])
    mr = float(ga_ref.Words(s, g, [n_elite], ga_ref.MUTATION).uniform()[0])
    return cx, mr


@functools.lru_cache(maxsize=None)
def _inputs(i):
    case = CASES[i]
    lo, hi, is_int = _genes(case["genes"])
    pop = case["pop"]
    params = ga_ref.init(np.zeros((pop, len(lo))), 0, lo, hi, is_int, 1000 + i)
    key, ranked = ga_ref.rank(_fitness(case["fitness"], pop, i))
    if case["fitness"] == "nan":
        key = _fitness("nan", pop, i)                   # NaN straight to the kernel; ranked as DeviceGeneticAlgorithm would
    cx, mr = case["cx"], case["mr"]
    if cx == "drawn":
        cx, mr = _drawn_rates(case, ga_ref.elite_count(case["elitism"], pop))
    return params, key, ranked, lo, hi, is_int, cx, mr


@functools.lru_cache(maxsize=None)
def _reference(i):
    case = CASES[i]
    params, key, ranked, lo, hi, is_int, cx, mr = _inputs(i)
    st = ga_ref.Stats()
    sel, out = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, case["elitism"], case["tournament"], cx, mr,
                                      case["seed"], case["generation"], st)
    return sel, out, st


def _c_ranges(lo, hi, is_int):
    G = len(lo)
    return (C.c_double * G)(*lo.tolist()), (C.c_double * G)(*hi.tolist()), (C.c_int * G)(*[int(b) for b in is_int])


def _device_next(torch, params, key, ranked, lo, hi, is_int, elitism, tournament, cx, mr, seed, generation):
    from ai_crypto_trader_b200 import _lib
    dev = torch.device("cuda", 0)
    P = torch.from_numpy(np.ascontiguousarray(params, np.float64)).to(dev)
    F = torch.from_numpy(np.ascontiguousarray(key, np.float64)).to(dev)
    R = torch.from_numpy(np.ascontiguousarray(ranked, np.int32)).to(dev)
    sel = torch.full((P.shape[0],), -7, dtype=torch.int32, device=dev)       # sentinels: every entry must be written
    out = torch.full_like(P, float("nan"))
    _lib.call("b200bt_ga_next_generation", P.data_ptr(), F.data_ptr(), R.data_ptr(), P.shape[0], P.shape[1],
              *_c_ranges(lo, hi, is_int), float(elitism), int(tournament), float(cx), float(mr), int(seed),
              int(generation), sel.data_ptr(), out.data_ptr(), _lib.current_stream())
    torch.cuda.synchronize()
    return sel.cpu().numpy(), out.cpu().numpy()


def _device_init(torch, params, n_seeded, lo, hi, is_int, seed):
    from ai_crypto_trader_b200 import _lib
    P = torch.from_numpy(np.ascontiguousarray(params, np.float64)).to(torch.device("cuda", 0))
    _lib.call("b200bt_ga_init", P.data_ptr(), P.shape[0], P.shape[1], int(n_seeded), *_c_ranges(lo, hi, is_int),
              int(seed), _lib.current_stream())
    torch.cuda.synchronize()
    return P.cpu().numpy()


def _assert_bits_equal(got, want, what):
    g, w = np.ascontiguousarray(got, np.float64).view(np.uint64), np.ascontiguousarray(want, np.float64).view(np.uint64)
    assert g.shape == w.shape, what
    bad = np.argwhere(g != w)
    assert len(bad) == 0, f"{what}: {len(bad)} of {g.size} values differ, first at {bad[0].tolist()}: " \
                          f"device {got[tuple(bad[0])]!r}, restatement {want[tuple(bad[0])]!r}"


# -- next generation ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("i", range(len(CASES)), ids=[c["name"] for c in CASES])
def test_next_generation_matches_restatement(torch_cuda, i):
    case = CASES[i]
    params, key, ranked, lo, hi, is_int, cx, mr = _inputs(i)
    want_sel, want_out, _ = _reference(i)
    sel, out = _device_next(torch_cuda, params, key, ranked, lo, hi, is_int, case["elitism"], case["tournament"], cx, mr,
                            case["seed"], case["generation"])
    assert np.array_equal(sel, want_sel), f"sel differs at {np.nonzero(sel != want_sel)[0][:8].tolist()}"
    _assert_bits_equal(out, want_out, "params_out")


def test_cases_exercise_the_stream_and_the_fused_arithmetic():
    """Against vacuous passes: without these events the word order, the rejection loop and the fma modelling would go
    untested by the comparisons above."""
    total = ga_ref.Stats()
    for i in range(len(CASES)):
        total.add(_reference(i)[2])
    for i, _ in _INIT_CASES:
        total.add(_init_reference(i)[1])
    assert total.straddles > 0, "no uniform() straddled two Philox blocks"
    assert total.rejections > 0, "no tournament rejected a repeated contender"
    assert total.fma_mutation > 0, "no mutated gene where fma differs from two roundings"
    assert total.fma_init > 0, "no initial float gene where fma differs from two roundings"
    for name in ("all elites, elitism 1", "all elites, elitism 1e300"):
        i = next(k for k, c in enumerate(CASES) if c["name"] == name)
        params, _, ranked = _inputs(i)[:3]
        assert np.array_equal(_reference(i)[1], params[ranked])           # nothing bred: the ranked rows, copied


def test_drawn_rates_sit_on_the_comparison_boundary():
    i = next(k for k, c in enumerate(CASES) if c["cx"] == "drawn")
    case = CASES[i]
    cx, mr = _inputs(i)[6:]
    n_elite = ga_ref.elite_count(case["elitism"], case["pop"])
    assert (cx, mr) == _drawn_rates(case, n_elite) and 0.0 < cx < 1.0 and 0.0 < mr < 1.0
    params, key, ranked, lo, hi, is_int = _inputs(i)[:6]
    for rate_cx, rate_mr in ((np.nextafter(cx, 0.0), mr), (cx, np.nextafter(mr, 1.0))):   # one ulp moves each outcome
        _, out = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, case["elitism"], case["tournament"],
                                        rate_cx, rate_mr, case["seed"], case["generation"])
        assert not np.array_equal(out[n_elite:n_elite + 2], _reference(i)[1][n_elite:n_elite + 2])


# -- init --------------------------------------------------------------------------------------------------------------

_INIT_CASES = list(enumerate([
    (1, 0, "synth"), (1, 1, "synth"), (129, 0, "synth"), (129, 1, "wide64"), (129, 129, "wide64"), (257, 40, "one_float"),
    (4096, 0, "synth"), (4096, 1, "synth_leverage"), (10_000, 0, "synth"), (3000, 3000, "synth"), (2000, 0, "wide64"),
]))


@functools.lru_cache(maxsize=None)
def _init_inputs(i):
    pop, n_seeded, genes = _INIT_CASES[i][1]
    lo, hi, is_int = _genes(genes)
    rng = np.random.default_rng(50 + i)
    span = np.maximum(hi - lo, 1.0)
    params = np.full((pop, len(lo)), np.nan)
    # seeded rows: outside the ranges on both sides (clamped), non-integral on integer genes (kept as given)
    params[:n_seeded] = lo + rng.uniform(-0.5, 1.5, (n_seeded, len(lo))) * span + 0.37
    seed = SEED + i
    return params, n_seeded, lo, hi, is_int, seed


@functools.lru_cache(maxsize=None)
def _init_reference(i):
    st = ga_ref.Stats()
    return ga_ref.init(*_init_inputs(i), st), st


@pytest.mark.parametrize("i", [i for i, _ in _INIT_CASES], ids=[f"pop{p}-seeded{s}-{g}" for _, (p, s, g) in _INIT_CASES])
def test_init_matches_restatement(torch_cuda, i):
    params, n_seeded, lo, hi, is_int, seed = _init_inputs(i)
    got = _device_init(torch_cuda, params, n_seeded, lo, hi, is_int, seed)
    want = _init_reference(i)[0]
    _assert_bits_equal(got, want, "initial population")
    if n_seeded:
        assert (want[:n_seeded] == lo).any() and (want[:n_seeded] == hi).any(), "no seeded value was clamped"
        inside = (params[:n_seeded] > lo) & (params[:n_seeded] < hi)
        assert np.array_equal(want[:n_seeded][inside], params[:n_seeded][inside])
        if is_int.any():
            assert (want[:n_seeded][:, is_int] != np.round(want[:n_seeded][:, is_int])).any()


# -- whole run ---------------------------------------------------------------------------------------------------------

def _run_fitness(population):
    """Deterministic, with ties (rounded), NaN and -inf for some individuals."""
    out = []
    for p in population:
        if p["macd_fast"] == 13:
            out.append(float("nan"))
        elif p["ema_short"] in (7, 8):
            out.append(float("-inf"))
        else:
            out.append(float(round(-(p["rsi_period"] - 17) ** 2 - 3.0 * (p["bollinger_std"] - 2.2) ** 2
                                   + 0.01 * p["ema_long"] + 0.5 * p["stop_loss"])))
    return out


def _same(a, b):
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, float) and isinstance(b, float):
        return np.float64(a).view(np.uint64) == np.float64(b).view(np.uint64) or (math.isnan(a) and math.isnan(b))
    return type(a) is type(b) and a == b


def test_device_run_matches_restatement(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm
    ranges = synth.param_ranges()
    seeded = [{"rsi_period": 400, "bollinger_std": -5.0},                        # clamped; every other key missing
              {"rsi_period": 12.7, "stop_loss": 3.5, "unknown": 1.0},           # non-integral on integer genes
              {}]
    kw = dict(population_size=301, generations=5, mutation_rate=0.3, crossover_rate=0.7, elitism_pct=0.07,
              tournament_size=4, random_seed=(3 << 32) | 17)
    snaps = []
    holder = []

    def fitness(population):
        ga = holder[0]
        snaps.append((ga.params.cpu().numpy().copy(), ga._sel.cpu().numpy().copy()))
        return _run_fitness(population)

    ga = DeviceGeneticAlgorithm(ranges, fitness, **kw)
    holder.append(ga)
    best = ga.run(seeded_individuals=seeded)
    st = ga_ref.Stats()
    want = ga_ref.run(ranges, _run_fitness, seeded_individuals=seeded, stats=st, **kw)

    assert len(snaps) == len(want.params) == 6
    for g, (params, sel) in enumerate(snaps):
        _assert_bits_equal(params, want.params[g], f"generation {g} params")
        if g:
            assert np.array_equal(sel, want.sel[g - 1]), f"generation {g} sel"
    history = [{k: v for k, v in h.items() if k != "timestamp"} for h in ga.get_generation_history()]
    assert _same(history, want.history)
    assert _same(best, want.best_individual) and _same(ga.best_fitness, want.best_fitness)
    # the run saw what it is meant to: NaN, -inf and tied scores, clamped and non-integral seeded genes
    flat = [f for gen in want.fitness for f in gen]
    assert any(math.isnan(f) for f in flat) and any(f == -math.inf for f in flat)
    finite = [f for f in want.fitness[-1] if math.isfinite(f)]
    assert len(set(finite)) < len(finite)
    assert want.params[0][0, 0] == 30.0 and want.params[0][1, 0] == 12.7
