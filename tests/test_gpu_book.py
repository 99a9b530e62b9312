"""Book-level metrics on the GPU (b200bt_book_metrics, PopulationSweep(aggregation="book")) against a record-by-record
oracle: the C oracle's lanes (oracle/sim_oracle.c, event words and record pnl) merged and walked by tests/book_ref.py.

Markets are planted so that the merged order is exercised: several symbols are copies of one series (their records fall
on the same bars, so ties across symbols are ordered by symbol index), a lane that is in the market on almost every bar
puts an entry and its force-close on the last bar of several symbols, and one symbol's RSI rows are NaN (it never
trades).  Counts, trade hash, days and merged-pair durations must match exactly; float statistics, score and fitness to
rel 1e-9 (NaN and inf included)."""
import ctypes

import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

PERIODS = (5, 9, 14, 21)
SOURCE = [0, 1, 0, 2, 0]          # symbol s is a copy of synthetic series SOURCE[s]
QUIET = 4                         # this symbol's RSI rows are NaN: no threshold compare is true, it never trades
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)
NEVER = dict(rsi_period=14, rsi_oversold=0, rsi_overbought=100)


def _population(n=22, seed=11):
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(n, seed=seed)
    for p in pop:
        p["rsi_period"] = PERIODS[int(p["rsi_period"]) % len(PERIODS)]
    return pop + [dict(DENSE), dict(NEVER), dict(DENSE, max_position_size=12, rsi_overbought=60)]


def _market(torch, n_bars, bar_minutes=1, minute0=None, source=SOURCE, quiet=QUIET):
    """(MarketData, RSI bank [S][P][N] on the device, host close [S][N], host bank)."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    close = np.ascontiguousarray(synth.synth_ohlcv(max(source) + 1, n_bars)[3][source])
    kw = dict(bar_minutes=bar_minutes) if minute0 is None else dict(bar_minutes=bar_minutes, minute0=minute0)
    market = MarketData.from_close(torch.from_numpy(close).cuda(), **kw)
    bank = PopulationSweep(market, rsi_periods=PERIODS, mode="fused").bank.clone()
    if quiet is not None:
        bank[quiet] = float("nan")
    return market, bank, close, bank.cpu().numpy()


def _books(close, bank, population, cfg):
    """Oracle books [pop] (dicts) and lanes [pop][S] of `population`."""
    import book_ref
    from oracle import sim_oracle
    lanes, evs, pns = sim_oracle.population(close, bank, {p: i for i, p in enumerate(PERIODS)}, population, cfg,
                                            event_cap=close.shape[1] + 2)
    return [book_ref.book(e, p, cfg) for e, p in zip(evs, pns)], lanes


def _book_sweep(market, bank, **kw):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    return PopulationSweep.from_bank(market, bank, PERIODS, aggregation="book", **kw)


@pytest.mark.parametrize("case, bar_minutes, gap", [
    ("1-minute bars", 1, None),
    ("7-minute bars", 7, None),
    ("1440-minute bars", 1440, None),
    ("glued series", 1, (7001, 2 * 1440 + 17)),
])
def test_book_matches_the_oracle(torch_cuda, case, bar_minutes, gap):
    from oracle import sim_oracle
    N = 20_000
    market, bank, close, bank_h = _market(torch_cuda, N, bar_minutes)
    pop = _population()
    sweep = _book_sweep(market, bank)
    cfg = sim_oracle.config_of(market.minute0, bar_minutes)
    if gap is not None:
        sweep.set_gap(*gap)
        cfg.gap_bar, cfg.gap_minutes = gap
    fit = sweep.evaluate(pop)
    want, lanes = _books(close, bank_h, pop, cfg)
    got = sweep.book_stats()
    sim_oracle.assert_lanes(got, want, case)
    np.testing.assert_allclose(fit, [w["score"] for w in want], rtol=1e-9, atol=1e-11, equal_nan=True)
    # the planted shapes are there: ties across symbols, the last bar's entry + force-close, a quiet symbol, an empty book
    i_dense = len(pop) - 3
    assert lanes["n_records"][:, QUIET].max() == 0 and want[len(pop) - 2]["n_records"] == 0
    assert int(lanes["n_records"][i_dense, 0]) > N // 4
    assert np.array_equal(got["profitable_symbols"][:, 0], got["profitable_symbols"][:, 2])
    assert not got["profitable_symbols"][:, QUIET].any()
    # lane_stats() keeps describing the per-symbol lanes of the same sweep
    sim_oracle.assert_lanes(sweep.lane_stats(), lanes, f"{case}: lanes")


def test_last_bar_entry_and_force_close_across_symbols(torch_cuda):
    """Ends the series where the dense lane is flat on the second-to-last bar: it enters on the last bar of every copy of
    series 0 and is force-closed there, so bar N - 1 holds two records of each of those symbols."""
    from oracle import sim_oracle
    from ai_crypto_trader_b200 import synth
    cfg = sim_oracle.config_of(synth.EPOCH_2024_MINUTES, 1)
    for N in range(3000, 3040):
        market, bank, close, bank_h = _market(torch_cuda, N)
        _, ev, _ = sim_oracle.lane(close[0], bank_h[0, 0], DENSE, cfg, event_cap=N + 2)
        if len(ev) >= 2 and (int(ev[-2]) & 0x3FFFFFFF) == N - 1 and (int(ev[-1]) & 0x3FFFFFFF) == N - 1:
            break
    else:
        pytest.fail("no length in 3000..3039 puts an entry on the last bar")
    pop = _population()
    sweep = _book_sweep(market, bank)
    sweep.evaluate(pop)
    want, _ = _books(close, bank_h, pop, cfg)
    sim_oracle.assert_lanes(sweep.book_stats(), want, f"N = {N}")


def test_single_symbol_book_is_its_lane(torch_cuda):
    from oracle import sim_oracle
    N = 30_000
    market, bank, _, _ = _market(torch_cuda, N, source=[1], quiet=None)
    sweep = _book_sweep(market, bank)
    sweep.evaluate(_population())
    got, lane = sweep.book_stats(), sweep.lane_stats()
    sim_oracle.assert_lanes(got, {f: lane[f][:, 0] for f in lane}, "one symbol")


@pytest.mark.parametrize("schedule", ["fused", "chunked", "tiled"])
def test_every_schedule_gives_the_oracle_books(torch_cuda, schedule):
    from oracle import sim_oracle
    N = 150_000
    market, bank, close, bank_h = _market(torch_cuda, N)
    pop = _population(14, seed=5)
    opts = {"fused": dict(mode="fused"),
            "chunked": dict(mode="chunked"),
            "tiled": dict(mode="tiled")}[schedule]
    from ai_crypto_trader_b200.sweep import PopulationSweep
    sweep = PopulationSweep.from_bank(market, bank, PERIODS, aggregation="book", **opts)
    if schedule != "fused":
        sweep.chunk_options = dict(pool_scale=4.0, **({"chunks": 16} if schedule == "tiled" else {"target_events": 2000}))
    fit = sweep.evaluate(pop)
    want, _ = _books(close, bank_h, pop, sim_oracle.config_of(market.minute0, 1))
    sim_oracle.assert_lanes(sweep.book_stats(), want, schedule)
    np.testing.assert_allclose(fit, [w["score"] for w in want], rtol=1e-9, atol=1e-11, equal_nan=True)


GOALS = [
    {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]},
    {"primary": "sortino_ratio", "secondary": ["expectancy"]},
    {"primary": "calmar_ratio", "secondary": []},
    {"primary": "profit_per_day", "secondary": ["max_drawdown"]},
    {"primary": "recovery_factor", "secondary": ["win_rate"]},
    {"primary": "expectancy", "secondary": ["profit_factor", "expectancy"]},
    {"primary": "return_pct", "secondary": ["max_drawdown", "win_rate", "profit_factor"]},
    {"primary": "no_such_key", "secondary": ["win_rate"]},
] + [{"primary": k, "secondary": []} for k in ("profit_factor", "win_rate", "net_profit", "total_trades", "max_drawdown",
                                               "total_profit", "total_loss", "largest_profit", "largest_loss",
                                               "average_profit", "average_loss")]


@pytest.mark.parametrize("advanced", [False, True])
def test_every_score_rule(torch_cuda, advanced):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    N = 20_000
    market, bank, close, bank_h = _market(torch_cuda, N, bar_minutes=7)
    pop = _population(10, seed=3)
    for goals in GOALS:
        sweep = PopulationSweep.from_bank(market, bank, PERIODS, optimization_goals=goals, aggregation="book",
                                          score_on_advanced=advanced)
        fit = sweep.evaluate(pop)
        cfg = sim_oracle.config_of(market.minute0, 7, goals=goals, advanced=advanced)
        want, _ = _books(close, bank_h, pop, cfg)
        np.testing.assert_allclose(fit, [w["score"] for w in want], rtol=1e-9, atol=1e-11, equal_nan=True,
                                   err_msg=str(goals))


def _same(a, b):
    for f in a:
        np.testing.assert_array_equal(a[f], b[f], err_msg=f)


def test_results_do_not_depend_on_the_event_cap_guess_slicing_or_duplicates(torch_cuda):
    N = 40_000
    market, bank, _, _ = _market(torch_cuda, N)
    pop = _population()
    exact = _book_sweep(market, bank)
    fit = exact.evaluate(pop)
    ref = exact.book_stats()
    assert exact.book_resweeps == 0
    # a learnt cap far below the busiest lane: the books that lost records are swept again with the exact cap
    guess = _book_sweep(market, bank)
    guess._book_cap = 8
    np.testing.assert_array_equal(guess.evaluate(pop), fit)
    assert guess.book_resweeps > 0
    _same(guess.book_stats(), ref)
    # the learnt cap of a second evaluation
    np.testing.assert_array_equal(exact.evaluate(pop), fit)
    _same(exact.book_stats(), ref)
    # a budget of a few individuals per slice
    sliced = _book_sweep(market, bank, max_event_bytes=3 * market.S * 4 * int(ref["n_records"].max()))
    np.testing.assert_array_equal(sliced.evaluate(pop), fit)
    _same(sliced.book_stats(), ref)
    # duplicates are booked once and expanded
    idx = [3, 0, 3, len(pop) - 3, 5, 0, len(pop) - 3]
    dup = _book_sweep(market, bank)
    np.testing.assert_array_equal(dup.evaluate([dict(pop[i]) for i in idx]), fit[idx])
    got = dup.book_stats()
    for f in ref:
        np.testing.assert_array_equal(got[f], ref[f][idx], err_msg=f)


def test_lost_records_mark_the_book(torch_cuda):
    """An event buffer smaller than a lane's records: that individual's book is n_records = -1, score NaN."""
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population
    N = 10_000
    market, bank, _, _ = _market(torch_cuda, N)
    pop = [DENSE, NEVER]
    sweep = PopulationSweep.from_bank(market, bank, PERIODS, event_cap=64)
    sweep.evaluate(pop)
    packed = decode_population(pop, sweep.period_row)
    indiv = torch_cuda.from_numpy(packed.view(np.uint8)).cuda()
    book = torch_cuda.zeros((2, _lib.LANE_STATS_WORDS), dtype=torch_cuda.float64, device="cuda")
    fit = torch_cuda.zeros(2, dtype=torch_cuda.float64, device="cuda")
    _lib.call("b200bt_book_metrics", market.close.data_ptr(), _lib.ld(market.close), market.S, N, indiv.data_ptr(), 2,
              ctypes.byref(sweep.cfg),
              sweep._stats.data_ptr(), sweep._events.data_ptr(), 64, book.data_ptr(), fit.data_ptr(),
              _lib.current_stream())
    b, f = book.cpu().numpy(), fit.cpu().numpy()
    assert b[0, 0] == -1 and np.isnan(f[0])
    assert b[1, 0] == 0 and f[1] == 0.0


def test_default_aggregation_is_the_mean(torch_cuda):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    market, bank, _, _ = _market(torch_cuda, 10_000)
    pop = _population()
    mean = PopulationSweep.from_bank(market, bank, PERIODS)
    fit = mean.evaluate(pop)
    np.testing.assert_allclose(fit, mean.lane_stats()["score"].mean(axis=1), rtol=1e-12, equal_nan=True)
    with pytest.raises(RuntimeError):
        mean.book_stats()
