"""Backtest overfitting on the GPU (csrc/overfitting.cu):

* per-day PnL rows (b200bt_daily_pnl, PopulationSweep.daily_pnl) against the reference's own daily buckets
  (tests/golden/book_reference.json), against oracle/sim_oracle.c lane records bucketed on the host (tests/cscv_ref.py)
  on several bar clocks and glued series, across the three sweep schedules, and against the book pass at full size;
* CSCV (b200bt_cscv) bit for bit against tests/cscv_ref.cscv_exact;
* StrategyEvaluationSystem.backtest_overfitting end to end against the oracle pipeline."""
import json
from pathlib import Path

import numpy as np
import pytest

import cscv_ref
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
PERIODS = (5, 9, 14, 21)
SOURCE = [0, 1, 0, 2, 0]
QUIET = 4
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)
NEVER = dict(rsi_period=14, rsi_oversold=0, rsi_overbought=100)


def _population(n=22, seed=11):
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(n, seed=seed)
    for p in pop:
        p["rsi_period"] = PERIODS[int(p["rsi_period"]) % len(PERIODS)]
    return pop + [dict(DENSE), dict(NEVER), dict(DENSE, max_position_size=12, rsi_overbought=60)]


def _market(torch, n_bars, bar_minutes=1):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    close = np.ascontiguousarray(synth.synth_ohlcv(max(SOURCE) + 1, n_bars)[3][SOURCE])
    market = MarketData.from_close(torch.from_numpy(close).cuda(), bar_minutes=bar_minutes)
    bank = PopulationSweep(market, rsi_periods=PERIODS, mode="fused").bank.clone()
    bank[QUIET] = float("nan")
    return market, bank, close, bank.cpu().numpy()


def _day_rows(close, bank, population, cfg, row_of):
    """Host lane rows [pop][S][D] of the C oracle's records."""
    from oracle import sim_oracle
    N = close.shape[1]
    _, evs, pns = sim_oracle.population(close, bank, row_of, population, cfg, event_cap=N + 2)
    return np.array([[cscv_ref.lane_rows(ev, pn, cfg, N) for ev, pn in zip(*lanes)] for lanes in zip(evs, pns)])


def _close_rows(got, want, where):
    """rel 1e-12 on every day with records (scaled by the day's magnitude), exact 0 elsewhere."""
    np.testing.assert_array_equal(got == 0, want == 0, err_msg=f"{where}: days without records")
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=where)


def test_book_rows_are_the_reference_daily_buckets(torch_cuda):
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    meta = json.loads((GOLD / "book_reference.json").read_text())
    arrays = np.load(GOLD / "book_reference.npz")
    for case in meta["cases"]:
        name, bm = case["name"], case["bar_minutes"]
        market = MarketData.from_close(torch_cuda.from_numpy(arrays[f"close_{name}"]).cuda(), minute0=meta["minute0"],
                                       bar_minutes=bm)
        bank = torch_cuda.from_numpy(np.ascontiguousarray(arrays[f"rsi_{name}"])).cuda()
        sweep = PopulationSweep.from_bank(market, bank, meta["periods"])
        book, _, first = sweep.daily_pnl([b["params"] for b in case["books"]])
        book = book.cpu().numpy()
        assert first == meta["minute0"] // 1440
        assert book.shape[1] == (meta["minute0"] + (case["n_bars"] - 1) * bm) // 1440 - first + 1
        for i, b in enumerate(case["books"]):
            days = np.unique((meta["minute0"] + arrays[f"bar_{name}_{i}"] * bm) // 1440) - first
            want = np.array([float(v) for v in b["daily_returns"]])
            assert len(want) == len(days) or b["n_records"] < 2
            np.testing.assert_allclose(book[i, days], want if len(want) else np.zeros(len(days)), rtol=1e-12, atol=0,
                                       err_msg=f"{name} book {i}")
            rest = np.ones(book.shape[1], dtype=bool)
            rest[days] = False
            assert np.all(book[i, rest] == 0.0), (name, i)
            assert b["n_records"] == 0 or np.all(book[i, days] != 0.0)


def _midnight_gap(minute0, gap_bar):
    """A gap that puts the first bar after the seam exactly on a midnight, 3 calendar days on."""
    return 3 * 1440 - (minute0 + gap_bar) % 1440


@pytest.mark.parametrize("case, bar_minutes, n_bars, gap", [
    ("1-minute bars", 1, 20_000, None),
    ("7-minute bars", 7, 20_000, None),
    ("1440-minute bars", 1440, 3_000, None),
    ("glued, seam inside a day", 1, 20_000, (7001, 2 * 1440 + 17)),
    ("glued, seam on a midnight", 1, 20_000, (9001, "midnight")),
])
def test_lane_rows_match_the_oracle(torch_cuda, case, bar_minutes, n_bars, gap):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    market, bank, close, bank_h = _market(torch_cuda, n_bars, bar_minutes)
    pop = _population()
    sweep = PopulationSweep.from_bank(market, bank, PERIODS)
    cfg = sim_oracle.config_of(market.minute0, bar_minutes)
    if gap is not None:
        gap_minutes = _midnight_gap(market.minute0, gap[0]) if gap[1] == "midnight" else gap[1]
        sweep.set_gap(gap[0], gap_minutes)
        cfg.gap_bar, cfg.gap_minutes = gap[0], gap_minutes
    book, lanes, first = sweep.daily_pnl(pop)
    want = _day_rows(close, bank_h, pop, cfg, sweep.period_row)
    first_w, D = cscv_ref.calendar(cfg, n_bars)
    assert first == first_w and lanes.shape == (len(pop), market.S, D)
    got = lanes.cpu().numpy()
    _close_rows(got, want, case)
    np.testing.assert_array_equal(book.cpu().numpy(), np.array([cscv_ref.book_row(list(g)) for g in got]))
    assert not got[:, QUIET].any() and not got[len(pop) - 2].any()         # a never-trading symbol and individual
    if gap is not None:
        prev, seam = (cscv_ref.day_of(np.array([gap[0] - 1, gap[0]]), cfg) - first).tolist()
        assert seam - prev >= 2 and not got[:, :, prev + 1:seam].any()     # the skipped days are zero columns
        assert got[:, :, prev].any() and got[:, :, seam].any()


def test_last_bar_entry_and_force_close(torch_cuda):
    from ai_crypto_trader_b200.sweep import PopulationSweep
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
    _, lanes, _ = PopulationSweep.from_bank(market, bank, PERIODS).daily_pnl(pop)
    _close_rows(lanes.cpu().numpy(), _day_rows(close, bank_h, pop, cfg, {p: i for i, p in enumerate(PERIODS)}),
                f"N = {N}")


def test_rows_do_not_depend_on_the_schedule(torch_cuda):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    market, bank, _, _ = _market(torch_cuda, 150_000)
    pop = _population(14, seed=5)
    rows = {}
    for mode in ("fused", "chunked", "tiled"):
        sweep = PopulationSweep.from_bank(market, bank, PERIODS, mode=mode)
        if mode != "fused":
            sweep.chunk_options = dict(pool_scale=4.0, **({"chunks": 16} if mode == "tiled" else {"target_events": 2000}))
        book, lanes, _ = sweep.daily_pnl(pop)
        rows[mode] = (book.cpu().numpy(), lanes.cpu().numpy())
    for mode in ("chunked", "tiled"):
        for a, b in zip(rows["fused"], rows[mode]):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), mode
    # duplicates are swept once and expanded; a tight budget slices the population; a too-small max_bytes is refused
    sweep = PopulationSweep.from_bank(market, bank, PERIODS, max_event_bytes=1 << 20)
    idx = [3, 0, 3, len(pop) - 3, 0]
    book, lanes, _ = sweep.daily_pnl([dict(pop[i]) for i in idx])
    assert np.array_equal(lanes.cpu().numpy(), rows["fused"][1][idx]) and np.array_equal(book.cpu().numpy(), rows["fused"][0][idx])
    with pytest.raises(ValueError, match="bytes"):
        sweep.daily_pnl(pop, max_bytes=1000)


def _bits_equal(a, b, what):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (what, np.max(np.abs(a - b)))


def _check_cscv(torch, x, B, where):
    from ai_crypto_trader_b200.overfitting import cscv
    got = cscv(torch.from_numpy(np.ascontiguousarray(x)).cuda(), B)
    want = cscv_ref.cscv_exact(x, B)
    for k in ("sel", "n_below", "n_tied"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=f"{where}: {k}")
    for k in ("is_sr", "oos_sr", "mu", "m2", "m3", "m4", "sharpe"):
        _bits_equal(got[k], want[k], f"{where}: {k}")
    assert got["block_days"] == want["block_days"] and got["dropped_days"] == want["dropped_days"]
    return got, want


@pytest.mark.parametrize("N, T, B", [(2, 11, 2), (33, 205, 20), (1000, 333, 16), (4097, 50, 4), (4097, 170, 16)])
def test_cscv_matches_the_exact_restatement(torch_cuda, N, T, B):
    rng = np.random.default_rng(N + T + B)
    x = rng.normal(0.001, 0.02, (N, T)) * rng.uniform(0.5, 2.0, (N, 1))
    if N > 2:
        x[N // 2] = 0.0                              # never trades
        x[N // 3] = 0.004                            # constant: zero variance
        x[1] += 0.05                                 # a dominant trial, duplicated further down: exact in-sample ties
        x[N - 1] = x[1]
    got, _ = _check_cscv(torch_cuda, x, B, f"N={N} T={T} B={B}")
    if N > 2:
        assert np.all(got["sel"] == 1) and np.all(got["n_tied"] >= 1)        # ties go to the lowest index


def test_cscv_full_size_books(torch_cuda):
    """configs[1] at full size (1024 individuals x 10 symbols x 1M bars): the book rows against the book pass, then CSCV
    of those rows at B = 16 bit for bit."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    S, N, POP = 10, 1_000_000, 1024
    market = MarketData(synth.synth_ohlcv(S, N))
    pop = synth.random_population(POP, seed=42)
    sweep = PopulationSweep(market, aggregation="book")
    sweep.evaluate(pop)
    st = sweep.book_stats()
    book, _, _ = sweep.daily_pnl(pop)
    rows = book.cpu().numpy()
    net, scale = st["net_profit"], np.abs(rows).sum(axis=1)
    assert np.all(np.abs(rows.sum(axis=1) - net) <= 1e-9 * np.maximum(np.abs(net), 1e-3 * scale))
    nz = rows != 0
    assert np.array_equal(nz.sum(axis=1), st["n_days"].astype(np.int64))     # no day with records sums to exactly 0
    sharpe = np.zeros(POP)
    for i in range(POP):
        d = rows[i, nz[i]]
        if st["n_records"][i] >= 2 and len(d) > 1 and np.std(d) > 0:
            sharpe[i] = np.mean(d) / np.std(d) * np.sqrt(252)
    np.testing.assert_allclose(sharpe, st["sharpe_ratio"], rtol=1e-9, atol=1e-12)
    _check_cscv(torch_cuda, rows, 16, "configs[1] books")


def test_backtest_overfitting_end_to_end(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.overfitting import deflated_sharpe, summarize
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    S, N = 3, 150_000
    ohlcv = synth.synth_ohlcv(S, N)
    market = MarketData(ohlcv)
    base = synth.random_population(200, seed=21)
    pop = base + [dict(base[i]) for i in range(0, 112, 2)]               # 256 with 56 duplicates
    ses = StrategyEvaluationSystem(config={})
    sweep = PopulationSweep(market)
    res = ses.backtest_overfitting(pop, market, n_blocks=16, sweep=sweep)
    # the oracle pipeline: C-oracle records -> host rows -> cscv_exact
    _, unique, expand = sweep._unique(pop)
    cfg = sim_oracle.config_of(market.minute0, 1)
    lanes = _day_rows(ohlcv[3], sweep.bank.cpu().numpy(), unique, cfg, sweep.period_row)
    want = cscv_ref.cscv_exact(np.array([cscv_ref.book_row(list(g)) for g in lanes]), 16)
    summ = summarize(want["is_sr"], want["oos_sr"], want["n_below"], want["n_tied"], len(unique))
    dsr = deflated_sharpe(want, len(unique))
    assert res["n_trials"] == len(unique) < len(pop) and res["n_combinations"] == 12870
    assert res["first_day"] == market.minute0 // 1440
    np.testing.assert_array_equal(res["sel"], want["sel"])
    assert res["pbo"] == summ["pbo"] and res["prob_oos_loss"] == summ["prob_oos_loss"]
    np.testing.assert_allclose(res["sharpe"], want["sharpe"][expand], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(res["deflated_sharpe"], dsr[expand], rtol=1e-9, atol=1e-12, equal_nan=True)
    best = int(np.argmax(res["sharpe"]))
    assert res["best"]["index"] == best and res["best"]["sharpe"] == res["sharpe"][best]
    assert set(res["degradation"]) == {"slope", "intercept", "r2"}
    assert ses.backtest_overfitting(pop, market, n_blocks=3, sweep=sweep) == {}
