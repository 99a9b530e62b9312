"""Walk-forward evaluation on the GPU (csrc/walk_forward.cu, ai_crypto_trader_b200/walk_forward.py): segment lanes against
the C oracle run once per segment, a one-segment schedule against b200bt_sweep on the slice, invalid schedules, the device
decode against decode_population, the lockstep GA against DeviceGeneticAlgorithm alone, and the driver end to end."""
import ctypes as C
import math

import numpy as np
import pytest

import book_ref
from gpu_fixtures import torch_cuda  # noqa: F401
from oracle import sim_oracle

pytestmark = pytest.mark.gpu

GOALS = {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]}
BUSY = {"rsi_period": 5, "rsi_oversold": 35, "rsi_overbought": 65, "take_profit": 1, "stop_loss": 1}


@pytest.fixture(scope="module", params=[6001, 6000], ids=["ld-ragged", "ld-x4"])
def market(torch_cuda, request):
    """(sweep, host close [S][N], host bank [S][P][N]) of a 2-symbol 1-minute market starting at 07:13."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    N = request.param
    ohlcv = synth.synth_ohlcv(2, N, seed_base=77)
    m = MarketData(ohlcv, minute0=synth.EPOCH_2024_MINUTES + 7 * 60 + 13)
    sweep = PopulationSweep(m, optimization_goals=GOALS)
    return sweep, ohlcv[3].astype(np.float32), sweep.bank.cpu().numpy()


def _wf(sweep, **kw):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.walk_forward import WalkForward
    return WalkForward(sweep, synth.param_ranges(), **kw)


def _run(sweep, params, schedules, event_cap=0, packed=None, tables=None):
    """Lane stats {field: [J][S]} and events [J][S][cap] (or None) of schedules [[(start, end, index into params)]]
    (`tables`: segment_tables' output to use instead, e.g. with a record altered)."""
    import torch
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import _stats_fields, decode_population
    from ai_crypto_trader_b200.walk_forward import segment_tables
    packed = decode_population(params, sweep.period_row) if packed is None else packed
    indiv = torch.from_numpy(packed.view(np.uint8).copy()).cuda()
    seg, begin = segment_tables(schedules) if tables is None else tables
    S = sweep.market.S
    stats = torch.empty((len(schedules), S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device="cuda")
    events = torch.zeros((len(schedules), S, event_cap), dtype=torch.int32, device="cuda") if event_cap else None
    _wf(sweep).sweep_segments(indiv, len(packed), torch.from_numpy(seg.view(np.int64)).cuda(), torch.from_numpy(begin).cuda(), stats,
                              events, event_cap)
    return _stats_fields(stats.cpu().numpy()), None if events is None else events.cpu().numpy().view(np.uint32)


def _oracle(sweep, close, bank, params, sched, s):
    """(book stats dict, global event words) of schedule `sched` on symbol s: the oracle lane on each segment's slice,
    words shifted to global bars, records concatenated and scored as one list."""
    m = sweep.market
    words, pnls = [], []
    for a, b, k in sched:
        p = params[k]
        cfg = sim_oracle.config_of(m.minute0 + a * m.bar_minutes, m.bar_minutes, GOALS)
        row = sweep.period_row[int(p.get("rsi_period", 14))]
        _, ev, pn = sim_oracle.lane(close[s, a:b], bank[s, row, a:b], p, cfg, event_cap=b - a + 1)
        words.append(ev.astype(np.uint32) + np.uint32(a))
        pnls.append(pn)
    w = np.concatenate(words) if words else np.zeros(0, np.uint32)
    pn = np.concatenate(pnls) if pnls else np.zeros(0)
    return book_ref.book([w], [pn], sim_oracle.config_of(m.minute0, m.bar_minutes, GOALS)), w


def _check(sweep, close, bank, params, schedules, event_cap=0):
    got, ev = _run(sweep, params, schedules, event_cap)
    S = sweep.market.S
    want, want_ev = [], []
    for sched in schedules:
        lanes = [_oracle(sweep, close, bank, params, sched, s) for s in range(S)]
        want.append([o for o, _ in lanes])
        want_ev.append([w for _, w in lanes])
    flat_got = [{f: got[f][j, s] for f in got} for j in range(len(schedules)) for s in range(S)]
    sim_oracle.assert_lanes(flat_got, [w for row in want for w in row], "segments")
    if event_cap:
        sim_oracle.assert_events(ev, [[w[:event_cap] for w in row] for row in want_ev], "segments")
    return got, want_ev


def _random_schedules(rng, N, J, n_params):
    out = []
    for _ in range(J):
        k = int(rng.integers(1, 7))
        cuts = np.sort(rng.choice(np.arange(1, N), size=2 * k, replace=False))
        sched = []
        for i in range(k):
            a, b = int(cuts[2 * i]), int(cuts[2 * i + 1])
            if i and rng.random() < 0.4:
                a = sched[-1][1]                      # adjacent to the previous segment
            if b > a:
                sched.append((a, b, int(rng.integers(n_params))))
        out.append(sched)
    return out


def test_random_schedules_match_the_oracle(market):
    from ai_crypto_trader_b200 import synth
    sweep, close, bank = market
    rng = np.random.default_rng(11)
    params = synth.random_population(6, seed=4) + [dict(BUSY)]
    schedules = _random_schedules(rng, sweep.market.N, 10, len(params))
    schedules += [[(0, sweep.market.N, 6)], [(1, 2, 6)], [(4, 4004, 6)]]      # whole series, one bar, aligned start
    assert len(schedules) == 13                                                # not a multiple of 8 warps per CTA
    _check(sweep, close, bank, params, schedules, event_cap=sweep.market.N + 1)


def test_event_cap_below_the_record_count(market):
    sweep, close, bank = market
    params = [dict(BUSY)]
    schedules = [[(3, 1500, 0), (1500, 3001, 0), (3100, 5007, 0)]]
    got, want_ev = _check(sweep, close, bank, params, schedules, event_cap=7)
    assert got["n_records"][0, 0] > 7


def test_boundary_cases(market):
    """An entry on a segment's last bar, and a position force-closed at a boundary and re-entered on the next bar."""
    sweep, close, bank = market
    params = [dict(BUSY)]
    row = sweep.period_row[5]
    r = bank[0, row]
    sig = np.nonzero((r < 35) | (r > 65))[0]
    quiet = np.nonzero(~((r < 35) | (r > 65)))[0]
    quiet_set = set(quiet.tolist())
    t = int(next(x for x in sig if x - 1 in quiet_set and x > 10))
    # segment [t - 1, t + 1): bar t - 1 quiet, bar t enters and is force-closed on the same bar
    schedules = [[(t - 1, t + 1, 0)], [(t, t + 1, 0)]]
    # adjacent segments cut where the whole-series run holds a position and the next bar signals again
    # (a segment that starts on an entry of the whole-series run follows that run until it ends)
    _, words = _oracle(sweep, close, bank, params, [(0, sweep.market.N, 0)], 0)
    bars = (words & 0x3FFFFFFF).astype(np.int64)
    sig_set = set(sig.tolist())
    e = next(int(bars[i]) for i in range(0, len(bars) - 1, 2) if bars[i + 1] - bars[i] > 3 and bars[i] + 2 in sig_set)
    cut = e + 2
    schedules.append([(e, cut, 0), (cut, cut + 700, 0)])
    _, want_ev = _check(sweep, close, bank, params, schedules, event_cap=sweep.market.N)
    ev = want_ev[0][0]
    assert len(ev) == 2 and (ev[0] & 0x3FFFFFFF) == t and (ev[1] & 0x3FFFFFFF) == t and ev[1] & 0x40000000
    ev = want_ev[2][0]
    b = (ev & 0x3FFFFFFF).astype(np.int64)
    k = int(np.nonzero(b >= cut)[0][0])
    assert b[k - 1] == cut - 1 and ev[k - 1] & 0x40000000 and b[k] == cut and not ev[k] & 0x40000000


def test_one_segment_equals_the_sweep_on_the_slice(market):
    import torch
    from ai_crypto_trader_b200 import _lib, synth
    from ai_crypto_trader_b200.sweep import _stats_fields, decode_population
    sweep, _, _ = market
    m = sweep.market
    params = synth.random_population(16, seed=9) + [dict(BUSY)]
    packed = decode_population(params, sweep.period_row)
    for a, b in ((0, m.N), (1, 2), (13, 4010), (2000, m.N), (4, 4004)):
        got, _ = _run(sweep, params, [[(a, b, i)] for i in range(len(params))], packed=packed)
        indiv = torch.from_numpy(packed.view(np.uint8).copy()).cuda()
        stats = torch.empty((len(params), m.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device="cuda")
        cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=m.minute0 + a * m.bar_minutes, bar_minutes=m.bar_minutes,
                               primary=sweep.cfg.primary, secondary_mask=sweep.cfg.secondary_mask, variant=0)
        _lib.call("b200bt_sweep", m.close.data_ptr() + 4 * a, _lib.ld(m.close), sweep.bank.data_ptr() + 4 * a,
                  _lib.ld(sweep.bank), sweep.bank.shape[1], m.S, b - a, indiv.data_ptr(), None, len(params), C.byref(cfg),
                  stats.data_ptr(), None, 0, _lib.current_stream())
        want = _stats_fields(stats.cpu().numpy())
        for f in want:
            if f != "trade_hash":
                np.testing.assert_array_equal(got[f].view(np.uint64), want[f].view(np.uint64), err_msg=f"{f} on [{a}, {b})")


def test_invalid_schedules_are_lost_lanes_alone(market):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import decode_population
    from ai_crypto_trader_b200.walk_forward import segment_tables
    sweep, _, _ = market
    N, P = sweep.market.N, sweep.bank.shape[1]
    params = synth.random_population(3, seed=2)
    packed = decode_population(params, sweep.period_row)
    bad_row = packed.copy()
    bad_row["rsi_row"][1], bad_row["rsi_row"][2] = P, -1
    good = [[(10, 2000, 0), (2000, 3000, 0)], [(5, N, 0)]]
    invalid = [[], [(-1, 100, 0)], [(100, 100, 0)], [(200, 100, 0)], [(0, N + 1, 0)],
               [(0, 1000, 0), (999, 2000, 0)], [(0, 100, 3)], [(0, 100, -1)], [(0, 50, 0), (50, 100, 1)],
               [(0, 50, 0), (60, 100, 2)], [(0, 50, 0), (50, 100, 0)]]
    ref, _ = _run(sweep, params, good, packed=bad_row)
    mixed = [good[0]] + invalid + [good[1]]
    seg, begin = segment_tables(mixed)
    seg["reserved"][begin[len(mixed) - 2] + 1] = 1          # the last invalid schedule: a valid table but for reserved
    got, ev = _run(sweep, params, mixed, event_cap=8, packed=bad_row, tables=(seg, begin))
    for f in ref:
        np.testing.assert_array_equal(got[f][[0, -1]].view(np.uint64), ref[f].view(np.uint64), err_msg=f)
    lost = got["n_records"][1:-1]
    assert np.all(lost == -1) and np.all(np.isnan(got["score"][1:-1]))
    assert np.all(got["net_profit"][1:-1] == 0) and np.all(ev[1:-1] == 0)


def _decode_both(sweep, matrix, names, cols=None):
    import torch
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import decode_population
    from ai_crypto_trader_b200.walk_forward import DECODE_GENES
    cols = [names.index(g) if g in names else -1 for g in DECODE_GENES] if cols is None else cols
    table = np.full(max(sweep.period_row) + 1, -1, dtype=np.int32)
    for p, r in sweep.period_row.items():
        table[p] = r
    dev = torch.from_numpy(np.ascontiguousarray(matrix, dtype=np.float64)).cuda()
    out = torch.zeros(len(matrix) * C.sizeof(_lib.Individual), dtype=torch.uint8, device="cuda")
    _lib.call("b200bt_decode_individuals", dev.data_ptr(), matrix.shape[1], len(matrix), (C.c_int * 6)(*cols),
              (C.c_int32 * len(table))(*table.tolist()), len(table), out.data_ptr(), _lib.current_stream())
    want = decode_population([dict(zip(names, map(float, row))) for row in matrix], sweep.period_row)
    return out.cpu().numpy(), want.view(np.uint8)


def test_decode_matches_decode_population(market):
    from ai_crypto_trader_b200 import synth
    sweep, _, _ = market
    ranges = synth.param_ranges()
    names = list(ranges)
    rng = np.random.default_rng(5)
    M = np.stack([rng.integers(lo, hi + 1, 300).astype(np.float64) if isinstance(lo, int) and isinstance(hi, int)
                  else rng.uniform(lo, hi, 300) for lo, hi in ranges.values()], axis=1)
    got, want = _decode_both(sweep, M, names)
    np.testing.assert_array_equal(got, want)
    # edge values: fp32-exact thresholds, one ulp off either way, unrepresentable ones, sizes above 20
    cols = ["rsi_period", "rsi_oversold", "rsi_overbought", "take_profit", "stop_loss", "max_position_size"]
    f32 = lambda x, d: float(np.nextafter(np.float32(x), np.float32(d)))
    edge = [[14, 30.0, 70.0, 3, 2, 5], [5, 30.5, 69.5, 1, 1, 20], [30, f32(30, 99), f32(70, 0), 10, 5, 25],
            [7, f32(30, 0), f32(70, 99), 0.3, 0.7, 100], [9, 0.1, 70.1, 2.5, 1.25, 19.999999], [12, 33.3, 66.6, 1e-3, 4.9, 21]]
    edge += [[p, np.nextafter(30.0, 99), np.nextafter(70.0, 0), 3, 2, 5] for p in (5, 30)]
    got, want = _decode_both(sweep, np.array(edge, dtype=np.float64), cols)
    np.testing.assert_array_equal(got, want)
    # absent columns take decode_population's defaults
    got, want = _decode_both(sweep, np.array([[21.0, 25.0]], dtype=np.float64), ["rsi_period", "rsi_oversold"])
    np.testing.assert_array_equal(got, want)
    got, _ = _decode_both(sweep, np.array([[21.0]], dtype=np.float64), ["rsi_period"], cols=[-1] * 6)
    np.testing.assert_array_equal(got, _decode_both(sweep, np.array([[14.0]], dtype=np.float64), ["rsi_period"])[1])
    # a period outside the table decodes to row -1
    got, _ = _decode_both(sweep, np.array([[31.0], [40.0]], dtype=np.float64), ["x"], cols=[0, -1, -1, -1, -1, -1])
    assert np.all(got.view(np.int32).reshape(2, 10)[:, 0] == -1)


@pytest.fixture(scope="module")
def days_market(torch_cuda):
    """A 2-symbol 1-minute market of six days from 05:00: windows of 2 in-sample days and 1 out-of-sample day."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    N = 6 * 1440 - 300
    ohlcv = synth.synth_ohlcv(2, N, seed_base=91)
    m = MarketData(ohlcv, minute0=synth.EPOCH_2024_MINUTES + 300)
    return PopulationSweep(m, optimization_goals=GOALS, mode="fused"), ohlcv[3].astype(np.float32)


def _alone(sweep, a, b, seed, seeded, pop, generations):
    """DeviceGeneticAlgorithm on window [a, b) alone, its batch fitness b200bt_sweep on the slice: (fitness per generation,
    final matrix, best individual)."""
    import torch
    from ai_crypto_trader_b200 import _lib, synth
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm
    from ai_crypto_trader_b200.sweep import decode_population
    m = sweep.market
    cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=m.minute0 + a * m.bar_minutes, bar_minutes=m.bar_minutes,
                           primary=sweep.cfg.primary, secondary_mask=sweep.cfg.secondary_mask, variant=0)
    seen = []

    def batch(population):
        packed = decode_population(population, sweep.period_row)
        indiv = torch.from_numpy(packed.view(np.uint8).copy()).cuda()
        stats = torch.empty((len(population), m.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device="cuda")
        fit = torch.empty(len(population), dtype=torch.float64, device="cuda")
        _lib.call("b200bt_sweep", m.close.data_ptr() + 4 * a, _lib.ld(m.close), sweep.bank.data_ptr() + 4 * a,
                  _lib.ld(sweep.bank), sweep.bank.shape[1], m.S, b - a, indiv.data_ptr(), None, len(population),
                  C.byref(cfg), stats.data_ptr(), None, 0, _lib.current_stream())
        _lib.call("b200bt_fitness_reduce", stats.data_ptr(), len(population), m.S, fit.data_ptr(), _lib.current_stream())
        out = fit.cpu().numpy()
        seen.append(out)
        return out.tolist()

    ga = DeviceGeneticAlgorithm(synth.param_ranges(), batch, population_size=pop, generations=generations,
                                random_seed=seed)
    best = ga.run(seeded_individuals=[dict(seeded)] if seeded else None)
    return seen, ga.params.cpu().numpy(), best


def test_lockstep_equals_each_window_alone(days_market):
    from ai_crypto_trader_b200.walk_forward import plan_windows, window_seed
    sweep, _ = days_market
    m = sweep.market
    windows = plan_windows(m.minute0, m.bar_minutes, m.N, 2, 1)
    assert len(windows) == 4
    seeded = dict(BUSY, rsi_period=14)
    wf = _wf(sweep, population_size=32, generations=5, random_seed=2 ** 64 - 2)
    seeds = [window_seed(wf.random_seed, w) for w in range(4)]
    winners, best, _, params = wf.evolve([(a, b) for a, b, _, _ in windows], seeds, seeded)
    for w, (a, b, _, _) in enumerate(windows):
        seen, final, best_alone = _alone(sweep, a, b, seeds[w], seeded, 32, 5)
        assert len(seen) == len(wf.last_fitness) == 6
        for g in range(6):
            np.testing.assert_array_equal(wf.last_fitness[g][w].view(np.uint64), seen[g].view(np.uint64),
                                          err_msg=f"window {w} generation {g}")
        np.testing.assert_array_equal(params[w].cpu().numpy().view(np.uint64), final.view(np.uint64))
        assert winners[w] == best_alone


def test_end_to_end(days_market, monkeypatch):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.evolution import StrategyEvolutionService
    from ai_crypto_trader_b200.walk_forward import plan_windows, window_seed
    sweep, close = days_market
    m = sweep.market
    bank = sweep.bank.cpu().numpy()
    current = dict(BUSY, rsi_period=14, max_position_size=8)
    monkeypatch.setenv("GA_POPULATION_SIZE", "24")
    monkeypatch.setenv("GA_GENERATIONS", "3")
    svc = StrategyEvolutionService(m, config={"evolution": {"optimization_goals": GOALS}}, random_seed=17)
    rep = svc.walk_forward(current, in_sample_days=2, out_of_sample_days=1)
    assert rep is not None and rep["n_reoptimizations"] == 4 and len(svc.evolution_records) == 4
    windows = plan_windows(m.minute0, m.bar_minutes, m.N, 2, 1)
    deployed = [r["parameters"] for r in rep["windows"]]
    stitched = [(c, d, k) for k, (_, _, c, d) in enumerate(windows)]
    for s in range(m.S):
        want, _ = _oracle(sweep, close, bank, deployed, stitched, s)
        sim_oracle.assert_lanes([{f: rep["stitched_stats"][f][s] for f in rep["stitched_stats"]}], [want], f"stitched {s}")
    for k, r in enumerate(rep["windows"]):
        assert r["in_sample"] == windows[k][:2] and r["out_of_sample"] == windows[k][2:]
        assert r["in_sample_fitness"] == max(h["best_fitness"] for h in r["history"])   # the best so far
        ins, oos = r["in_sample_stats"], r["out_of_sample_stats"]
        days_is, days_oos = (windows[k][1] - windows[k][0]) / 1440, (windows[k][3] - windows[k][2]) / 1440
        e = r["efficiency"]
        if ins["net_profit"] > 0:
            assert e == pytest.approx((oos["net_profit"] / days_oos) / (ins["net_profit"] / days_is))
        else:
            assert math.isnan(e)

    wf = _wf(sweep, population_size=16, generations=2, random_seed=3)
    never = {"min_sharpe_ratio": -1e300, "max_drawdown": 1e300, "min_win_rate": -1.0}
    rep = wf.run(current, 2, 1, reoptimize="when_needed", evolution_config=never)
    assert rep["n_reoptimizations"] == 0 and all(r["parameters"] == current for r in rep["windows"])
    always = {"min_sharpe_ratio": 1e300}
    rep = wf.run(current, 2, 1, reoptimize="when_needed", evolution_config=always)
    assert rep["n_reoptimizations"] == 4
    prev = current
    for k, (a, b, _, _) in enumerate(windows):
        winners, _, _, _ = wf.evolve([(a, b)], [window_seed(3, k)], prev)
        assert rep["windows"][k]["parameters"] == winners[0]
        prev = winners[0]

    book = StrategyEvolutionService(m, config={"evolution": {"optimization_goals": GOALS}}, aggregation="book")
    assert book.walk_forward(current, 2, 1) is None
