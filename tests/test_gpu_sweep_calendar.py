"""The calendar of the sweep's daily buckets and its score rules, through every schedule, against the C oracle.

Cross-validation trains on two pieces of a series glued together (PopulationSweep.set_gap): records from `gap_bar` on lie
`gap_minutes` later on the calendar.  From 131 072 bars up such folds go through the time-chunked kernels, where the
calendar day of a record is formed in chunk_partial_kernel (the fused kernel and the exact fallback: batch_core) and the
days that cross chunk and 128-record step boundaries are merged in lane_combine_kernel.  Every lane here is compared with
oracle/sim_oracle.c (int64 calendar, record-by-record two-pass statistics) on

  fused           one warp per lane, serial in time
  chunked         warp per chunk, forced into many chunks (a few hundred predicted events per chunk, up to 64 chunks)
  tiled           thread per chunk, K = 16 explicit chunks (chunk c starts at floor(N c / K) & ~511)
  tiled_fallback  tiled without warm-up or repair: lanes in a position at a chunk start take the exact fallback, which
                  reads the gap from the host config

1. A seam with a dense lane (an event on every bar) across it, against chunk, step and day boundaries.
2. The largest calendar the 32-bit minutes accept (every day number above 2^31 / 1440).
3. Every score rule (sim_cases.json alt_goals, every primary key with no and with all secondaries) on 150 000 bars,
   with lanes that never trade, trade once, trade with a zero position size and only win.
4. cross_validate_population at a length whose training folds take the time-chunked path.

The RSI rows the oracle is fed are the sweep's own bank (its correctness is tests/test_gpu_indicators.py's business)."""
import json
from pathlib import Path

import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
SCHEDULES = {
    "fused": dict(mode="fused"),
    "chunked": dict(mode="chunked", chunk_options=dict(target_events=300, max_chunks=64, warm=256, pool_scale=4.0)),
    "tiled": dict(mode="tiled", chunk_options=dict(chunks=16, pool_scale=4.0)),
    "tiled_fallback": dict(mode="tiled", chunk_options=dict(chunks=16, warm=0, max_repair_rounds=0, pool_scale=4.0)),
}
# (pool_scale: lanes that trade on every bar of a random walk record ~4x the events the cost model predicts; a pool
# overflow would send them to the exact fallback instead of the chunk kernels under test)
N1 = 1 << 16                      # section 1: tiled chunk c starts at 4096 c
CHUNK = N1 // 16
CAP = 2048                        # event words kept per lane
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)


# -- shared helpers ------------------------------------------------------------------------------------------------------
def _sweeps(market, bank, periods, goals=None, advanced=False, event_cap=0, gap=(0, 0)):
    """One PopulationSweep per schedule over the same bank."""
    from ai_crypto_trader_b200.sweep import PopulationSweep
    out = {}
    for name, opt in SCHEDULES.items():
        sw = PopulationSweep.from_bank(market, bank, periods, optimization_goals=goals, event_cap=event_cap,
                                       mode=opt["mode"], score_on_advanced=advanced)
        sw.chunk_options = dict(opt.get("chunk_options", {}))
        sw.set_gap(*gap)
        out[name] = sw
    return out


def _check_path(name, sw, population, S):
    """The schedule really ran its kernels: several chunks, and the fallback variant took the fallback."""
    plans = sw._last_plans
    if name == "fused":
        assert not plans
        return
    assert len(plans) == 1
    if name == "chunked":
        assert int(plans[0].n_chunks.max()) >= 16, plans[0].n_chunks
    else:
        assert plans[0].K == 16
    invalid = plans[0].invalid.cpu().numpy()
    if name == "tiled_fallback":
        assert sw.last_invalid_lanes > 0
    else:
        assert sw.last_invalid_lanes < len(population) * S
    return invalid


# -- 1. glued series -----------------------------------------------------------------------------------------------------
def _seam_close(gap_bar, half=320, seed=3):
    """Symbol 0: constant 100 except an alternating window of 2 * half bars around the seam, on which the DENSE lane
    records an event on every bar (>128 records on each side, so its day spans 128-record steps and the seam); outside the
    window it holds its position.  Symbol 1: an ordinary random walk."""
    from ai_crypto_trader_b200 import synth
    rng = np.random.default_rng(seed + gap_bar)
    c = np.full(N1, 100.0)
    a, b = max(1, gap_bar - half), min(N1 - 1, gap_bar + half)
    t = np.arange(a, b)
    c[t] = 100.0 + np.where(t % 2 == 0, 0.5, -0.5) + rng.uniform(-0.2, 0.2, len(t))
    return np.stack([c, synth.synth_symbol(7, N1)["close"]]).astype(np.float32)


def _seam_population():
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(29, seed=17)
    pop[0].update(DENSE)
    pop[1].update(DENSE, rsi_oversold=-1, rsi_overbought=1)          # the short mirror
    pop[2].update(rsi_oversold=-1, rsi_overbought=101)                # never trades
    pop[3].update(DENSE, take_profit=0.3, stop_loss=0.3)              # fewer, larger trades
    return pop


DAY = 1440
# (gap_bar, gap_minutes, minute0 % 1440, bar_minutes, the dense lane's records on both sides of the seam share a day)
SEAM_CASES = [
    (2 * CHUNK, 1, 0, 1, True),                     # on a tiled chunk start, the open day continues
    (2 * CHUNK - 1, 1439, 0, 1, False),             # one bar before a chunk start
    (5 * CHUNK + 1, 1440, 1439, 1, False),          # one bar after it; first bar one minute before midnight
    (7 * CHUNK + 1234, 1441, 0, 1, False),          # strictly inside a chunk
    (9 * CHUNK + 700, 1, 1439, 1, True),
    (1, 1, 0, 1, False),                            # the seam after the first bar (no dense record before it)
    (1, 3 * DAY + 17, 1439, 1, False),
    (N1 - 1, DAY, 0, 1, False),                     # only the last bar (the dense lane's close) after the seam
    (N1 - 1, 5 * DAY + 777, 1439, 1, False),
    (3 * CHUNK, 1, 0, 7, True),                     # 7-minute bars
    (11 * CHUNK + 5, 1441, 1439, 7, False),
    (6 * CHUNK, 2 * DAY + 1, 1439, 1440, False),    # one bar per day: no gap can merge or split a day (see below)
]


def _seam_case(torch, gap_bar, gap_minutes, m0_mod, bar_minutes, minute0=None):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    if minute0 is None:
        minute0 = synth.EPOCH_2024_MINUTES // DAY * DAY + 30 * DAY + m0_mod
    close = _seam_close(gap_bar)
    market = MarketData.from_close(torch.from_numpy(close).cuda(), minute0=minute0, bar_minutes=bar_minutes)
    population = _seam_population()
    base = PopulationSweep(market, mode="fused")
    bank = base.bank.cpu().numpy()
    cfg = sim_oracle.config_of(minute0, bar_minutes, gap_bar=gap_bar, gap_minutes=gap_minutes)
    want, want_ev, _ = sim_oracle.population(close, bank, base.period_row, population, cfg, CAP)
    plain, _, _ = sim_oracle.population(close, bank, base.period_row, population, sim_oracle.config_of(minute0, bar_minutes))
    sweeps = _sweeps(market, base.bank, base.periods, event_cap=CAP, gap=(gap_bar, gap_minutes))
    where = f"gap_bar {gap_bar}, gap_minutes {gap_minutes}, minute0 {minute0}, bar_minutes {bar_minutes}"
    failed = []                       # every schedule is checked, so that a failure names all the schedules it shows on
    for name, sw in sweeps.items():
        fit = sw.evaluate(population)
        st = sw.lane_stats()
        try:
            sim_oracle.assert_lanes(st, want, f"{name}, {where}")
            sim_oracle.assert_events(sw.events(), want_ev, f"{name}, {where}")
            np.testing.assert_allclose(fit, (want["score"][:, 0] + want["score"][:, 1]) / 2, rtol=1e-9, atol=1e-11,
                                       equal_nan=True, err_msg=f"{name}: fitness")
        except AssertionError as e:
            failed.append(str(e))
        invalid = _check_path(name, sw, population, 2)
        if name in ("chunked", "tiled"):
            assert invalid[0, 0] == 0, f"{name}: the dense lane went through the exact fallback"
    assert not failed, "\n".join(failed)
    return close, population, want, want_ev, plain, minute0


@pytest.mark.parametrize("gap_bar, gap_minutes, m0_mod, bar_minutes, seam_in_day", SEAM_CASES)
def test_glued_series_match_oracle_on_every_schedule(torch_cuda, gap_bar, gap_minutes, m0_mod, bar_minutes, seam_in_day):
    close, population, want, want_ev, plain, minute0 = _seam_case(torch_cuda, gap_bar, gap_minutes, m0_mod, bar_minutes)
    # the dense lane really records on both sides of the seam, across 128-record steps
    bars = want_ev[0][0] & 0x3FFFFFFF
    n0 = int(want["n_records"][0, 0])
    assert n0 <= CAP and np.any(bars >= gap_bar)
    if gap_bar > 1:
        assert np.sum((bars < gap_bar) & (bars >= gap_bar - 320)) > 128
    if gap_bar < N1 - 1:
        assert np.sum(bars >= gap_bar) > 128
    # ... and its records next to the seam share a calendar day exactly in the cases that say so
    if gap_bar > 1:
        day = lambda b: (minute0 + int(b) * bar_minutes + (gap_minutes if b >= gap_bar else 0)) // DAY
        assert (day(bars[bars < gap_bar][-1]) == day(bars[bars >= gap_bar][0])) == seam_in_day
    # the gap changes the statistics (one bar per day: a gap only renumbers days, never merges or splits them)
    changed = (want["n_days"] != plain["n_days"]) | (want["sharpe_ratio"] != plain["sharpe_ratio"])
    if bar_minutes == DAY:
        assert not changed.any()
    else:
        assert changed.any(), "the gap changes no lane's days: the case does not test the calendar"
    assert np.any(want["n_days"] > 1) and np.any(want["n_negative_days"] > 0)


def test_case_list_has_seams_inside_a_day():
    assert sum(c[-1] for c in SEAM_CASES) >= 3


def test_zero_gap_minutes_is_bit_identical_to_no_gap(torch_cuda):
    """gap_bar > 0 with gap_minutes = 0 is the plain calendar, on every schedule."""
    torch = torch_cuda
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    gap_bar = 4 * CHUNK + 3
    close = _seam_close(gap_bar)
    market = MarketData.from_close(torch.from_numpy(close).cuda(), minute0=28_000_000 + 1439, bar_minutes=1)
    population = _seam_population()
    base = PopulationSweep(market, mode="fused")
    with_gap = _sweeps(market, base.bank, base.periods, gap=(gap_bar, 0))
    without = _sweeps(market, base.bank, base.periods)
    for name in SCHEDULES:
        f1 = with_gap[name].evaluate(population)
        r1 = with_gap[name]._stats.cpu().numpy()
        f0 = without[name].evaluate(population)
        r0 = without[name]._stats.cpu().numpy()
        np.testing.assert_array_equal(r1.view(np.uint64), r0.view(np.uint64), err_msg=name)
        np.testing.assert_array_equal(f1.view(np.uint64), f0.view(np.uint64), err_msg=name)


# -- 2. the limit of the 32-bit calendar ---------------------------------------------------------------------------------
def test_largest_accepted_calendar_matches_oracle(torch_cuda):
    """minute0 + N * bar_minutes + gap_minutes = 2^32 - 1441, the largest value the entry points accept: every record's
    minute needs the 32nd bit, every day number is above 2^31 / 1440 (tests/test_abi.py: one minute more is refused)."""
    gap_bar, gap_minutes, bar_minutes = 3 * CHUNK + 17, 1441, 1
    minute0 = (1 << 32) - 1441 - N1 * bar_minutes - gap_minutes
    assert minute0 // DAY > (1 << 31) // DAY
    _, _, want, _, plain, _ = _seam_case(torch_cuda, gap_bar, gap_minutes, None, bar_minutes, minute0=minute0)
    assert np.any((want["n_days"] != plain["n_days"]) | (want["sharpe_ratio"] != plain["sharpe_ratio"]))


# -- 3. score rules through the time-chunked schedules -------------------------------------------------------------------
N3 = 150_000
ONE_TRIP_ROW, WINNER_ROW = 97, 98       # crafted RSI rows, addressed as these rsi_period values


def _goal_sets():
    from oracle import sim_oracle
    meta = json.loads((GOLD / "sim_cases.json").read_text())
    sets = [(alt["goals"], alt["advanced"]) for alt in meta["alt_goals"]]
    sets.append((None, False))                                            # the default goals
    every = ["max_drawdown", "win_rate", "profit_factor", "expectancy"]
    for table, advanced in ((sim_oracle._PRIMARY, False), (sim_oracle._PRIMARY_ADV, True)):
        for primary in table:
            for secondary in ([], every):
                sets.append(({"primary": primary, "secondary": secondary}, advanced))
    return sets


def _winner_row(close, tp):
    """RSI row 50 everywhere except 10 on entry bars chosen so that every long trade reaches its take-profit `tp`
    (the only exit: RSI 50 never crosses 70 and the stop-loss is out of reach) before the last bar."""
    px = close.astype(np.float64)
    row = np.full(len(px), 50.0, dtype=np.float32)
    t = 200
    while t < len(px) - 1:
        hit = np.nonzero((px[t + 1:t + 20_001] - px[t]) / px[t] >= tp)[0]
        if not len(hit):
            hit = np.nonzero((px[t + 1:] - px[t]) / px[t] >= tp)[0]
        if not len(hit) or t + 1 + hit[0] >= len(px) - 1:
            break
        row[t] = 10.0
        t = t + 2 + int(hit[0])
    return row


@pytest.fixture(scope="module")
def score_market(torch_cuda):
    torch = torch_cuda
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    close = np.stack([synth.synth_symbol(s, N3)["close"] for s in (5, 6)]).astype(np.float32)
    market = MarketData.from_close(torch.from_numpy(close).cuda(), minute0=synth.EPOCH_2024_MINUTES + 1439, bar_minutes=1)
    base = PopulationSweep(market, mode="fused")
    one_trip = np.full(N3, 50.0, dtype=np.float32)
    one_trip[100] = 10.0                                   # a single entry; its forced close at N - 1
    extra = np.stack([np.stack([one_trip, _winner_row(close[s], 0.003)]) for s in range(2)])
    bank = np.concatenate([base.bank.cpu().numpy(), extra], axis=1)
    periods = list(base.periods) + [ONE_TRIP_ROW, WINNER_ROW]
    pop = synth.random_population(16, seed=23)
    pop += [dict(rsi_period=14, rsi_oversold=-1, rsi_overbought=101),                        # no records
            dict(rsi_period=ONE_TRIP_ROW, take_profit=1e4, stop_loss=1e4),                    # one round trip
            dict(rsi_period=9, rsi_oversold=35, rsi_overbought=65, max_position_size=0),     # zero PnL
            dict(rsi_period=WINNER_ROW, take_profit=0.3, stop_loss=1e4)]                       # every trade a winner
    return market, close, bank, periods, pop


def test_score_rules_match_oracle_on_time_chunked_schedules(torch_cuda, score_market):
    torch = torch_cuda
    from oracle import sim_oracle
    market, close, bank, periods, population = score_market
    bank_dev = torch.from_numpy(bank).cuda()
    period_row = {p: i for i, p in enumerate(periods)}
    n_edge = 4
    sets = _goal_sets()
    assert len(sets) >= 12 + 1 + 2 * 18
    saw_nan = saw_inf = False
    for goals, advanced in sets:
        cfg = sim_oracle.config_of(market.minute0, 1, goals, advanced=advanced)
        want, _, _ = sim_oracle.population(close, bank, period_row, population, cfg)
        if goals is None:
            # the edge lanes are what they claim to be
            st = want[-n_edge:]
            assert (st["n_records"][0] == 0).all() and (st["n_records"][1] == 2).all()
            assert (st["net_profit"][2] == 0).all() and (st["n_records"][2] > 10).all()
            assert np.isinf(st["profit_factor"][2]).all()
            assert (st["n_losses"][3] * 2 == st["n_records"][3]).all() and (st["n_wins"][3] * 2 == st["n_records"][3]).all()
            assert (st["n_records"][3] > 20).all()
        want_fit = (want["score"][:, 0] + want["score"][:, 1]) / 2
        saw_nan |= bool(np.isnan(want["score"]).any())
        saw_inf |= bool(np.isinf(want["score"]).any())
        for name, sw in _sweeps(market, bank_dev, periods, goals=goals, advanced=advanced).items():
            fit = sw.evaluate(population)
            where = f"{name}, goals {goals}, advanced {advanced}"
            sim_oracle.assert_lanes(sw.lane_stats(), want, where)
            np.testing.assert_allclose(fit, want_fit, rtol=1e-9, atol=1e-11, equal_nan=True, err_msg=f"{where}: fitness")
            _check_path(name, sw, population, 2)
    assert saw_nan and saw_inf


# -- 4. cross-validation on the time-chunked path ------------------------------------------------------------------------
def test_cross_validation_on_chunked_training_folds_matches_oracle(torch_cuda):
    """cross_validate_population at 200 000 bars, k = 4: every training fold (150 000 bars, glued with a gap for the
    inner folds) takes the time-chunked path, every test fold (50 000 bars) the fused one."""
    torch = torch_cuda
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    S, N, K = 2, 200_000, 4
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=8)
    market = MarketData(ohlcv, minute0=synth.EPOCH_2024_MINUTES + 1439)
    sweep = PopulationSweep(market, mode="fused")
    population = synth.random_population(12, seed=31)
    population[0].update(rsi_oversold=35, rsi_overbought=65, rsi_period=5, take_profit=1, stop_loss=1)
    bank = sweep.bank.cpu().numpy()
    close = ohlcv[3]
    ses = StrategyEvaluationSystem(config={})
    cv = ses.cross_validate_population(population, market.close, sweep.bank, sweep.periods, market.minute0, 1, K)
    fold = N // K
    for f in range(K):
        a, b = f * fold, (f + 1) * fold if f < K - 1 else N
        tr_close = np.concatenate([close[:, :a], close[:, b:]], axis=1)
        tr_bank = np.concatenate([bank[:, :, :a], bank[:, :, b:]], axis=2)
        # the training fold's shape takes the time-chunked path in cross_validate_population's mode="auto"
        tr_market = MarketData.from_close(torch.from_numpy(np.ascontiguousarray(tr_close)).cuda(), minute0=market.minute0)
        auto = PopulationSweep.from_bank(tr_market, torch.from_numpy(np.ascontiguousarray(tr_bank)).cuda(), sweep.periods,
                                         mode="auto")
        assert tr_market.N >= auto.chunk_min_bars and auto.plan(population) is not None
        te_market = MarketData.from_close(torch.from_numpy(np.ascontiguousarray(close[:, a:b])).cuda())
        assert PopulationSweep.from_bank(te_market, torch.from_numpy(np.ascontiguousarray(bank[:, :, a:b])).cuda(),
                                         sweep.periods, mode="auto").plan(population) is None
        gap = (a, b - a) if 0 < a and b < N else (0, 0)
        m0 = market.minute0 + (b if a == 0 else 0)
        want_tr, _, _ = sim_oracle.population(tr_close, tr_bank, sweep.period_row, population,
                                              sim_oracle.config_of(m0, 1, gap_bar=gap[0], gap_minutes=gap[1]))
        want_te, _, _ = sim_oracle.population(close[:, a:b], bank[:, :, a:b], sweep.period_row, population,
                                              sim_oracle.config_of(market.minute0 + a, 1))
        if gap[0]:
            plain, _, _ = sim_oracle.population(tr_close, tr_bank, sweep.period_row, population, sim_oracle.config_of(m0, 1))
            assert np.any(plain["sharpe_ratio"] != want_tr["sharpe_ratio"]), f"fold {f}: the gap changes nothing"
        for side, want in (("train", want_tr), ("test", want_te)):
            cv_close = ("sharpe_ratio", "max_drawdown", "win_rate", "profit_factor", "score")    # the fields a fold reports
            sim_oracle.assert_lanes({k: cv[f"{side}_{k}"][f] for k in ("n_records",) + cv_close}, want,
                                    f"fold {f} {side}", exact=("n_records",), close=cv_close)
            np.testing.assert_allclose(cv[f"{side}_return_pct"][f], want["net_profit"] / 10000.0 * 100, rtol=1e-9,
                                       atol=1e-11, err_msg=f"fold {f} {side} return_pct")
