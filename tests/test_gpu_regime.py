"""Market regimes on the GPU (csrc/regime.cu):

* b200bt_class_stats (PopulationSweep.class_stats) against tests/book_ref.book on the filtered records of
  oracle/sim_oracle.c lanes: random labellings with R = 1..8, labels >= R, alternating labels that split every pair, one
  class, empty classes, a shared label row; 1-, 7- and 1440-minute bars, a glued series, the last bar's entry and
  force-close, a never-trading and a dense lane; the fused, chunked and tiled schedules;
* the partition invariants, R = 1 against lane_stats() and the lost-records rows;
* b200bt_regime_labels against tests/regime_ref.py fed the device's own average rows, and points against
  indicators.multi_timeframe_indicators on the market cut at their bar;
* MarketRegimeService end to end against the oracle pipeline, and the configs[1] market at full size."""
import asyncio
import ctypes as C

import numpy as np
import pytest

import regime_ref
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

PERIODS = (5, 9, 14, 21)
SOURCE = [0, 1, 0, 2, 0]
QUIET = 4
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)
NEVER = dict(rsi_period=14, rsi_oversold=0, rsi_overbought=100)
ROW = {p: k for k, p in enumerate(PERIODS)}


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


def check_classes(views, evs, pns, labels, R, cfg, where):
    """Every class of every lane against regime_ref.class_stats of the oracle's records; float statistics to rel 1e-9 with
    no absolute floor.  A failure names lane (i, s) by its flat index i S + s."""
    from oracle import sim_oracle
    S = len(evs[0])
    want = [regime_ref.class_stats(evs[i][s], pns[i][s], labels[s if labels.shape[0] > 1 else 0], R, cfg)
            for i in range(len(evs)) for s in range(S)]
    for r in range(R):
        sim_oracle.assert_lanes({k: v.reshape(-1) for k, v in views[r].items()}, [w[r] for w in want],
                                f"{where} class {r}", atol=0)


def _labellings(S, N, rng):
    """(name, labels uint8 [S or 1][N], R)."""
    out = [(f"random R={R}", rng.integers(0, R, (S, N)).astype(np.uint8), R) for R in range(1, 9)]
    out += [("labels >= R", rng.integers(0, 7, (S, N)).astype(np.uint8), 4),
            ("alternating bars", np.broadcast_to((np.arange(N) % 2).astype(np.uint8), (S, N)).copy(), 2),
            ("one class, two empty", np.zeros((S, N), np.uint8), 3),
            ("shared row", rng.integers(0, 5, (1, N)).astype(np.uint8), 5)]
    return out


@pytest.mark.parametrize("case, bar_minutes, n_bars, gap, mode", [
    ("1-minute bars", 1, 20_000, None, "fused"),
    ("7-minute bars", 7, 20_000, None, "fused"),
    ("1440-minute bars", 1440, 3_000, None, "fused"),
    ("glued series", 1, 20_000, (7001, 2 * 1440 + 17), "fused"),
    ("chunked schedule", 1, 150_000, None, "chunked"),
    ("tiled schedule", 1, 150_000, None, "tiled"),
])
def test_class_stats_match_the_oracle(torch_cuda, case, bar_minutes, n_bars, gap, mode):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    market, bank, close, bank_h = _market(torch_cuda, n_bars, bar_minutes)
    pop = _population() if n_bars <= 20_000 else _population(8, seed=5)
    sweep = PopulationSweep.from_bank(market, bank, PERIODS, mode=mode)
    if mode != "fused":
        sweep.chunk_options = dict(pool_scale=4.0, **({"chunks": 16} if mode == "tiled" else {"target_events": 2000}))
    cfg = sim_oracle.config_of(market.minute0, bar_minutes)
    if gap is not None:
        sweep.set_gap(*gap)
        cfg.gap_bar, cfg.gap_minutes = gap
    _, evs, pns = sim_oracle.population(close, bank_h, ROW, pop, cfg, event_cap=market.N + 2)
    lengths = [len(ev) for lanes in evs for ev in lanes]
    assert min(lengths) == 0 and max(lengths) > 100
    rng = np.random.default_rng(bar_minutes + n_bars)
    for name, labels, R in _labellings(market.S, market.N, rng):
        out, views = sweep.class_stats(pop, torch_cuda.from_numpy(labels).cuda(), R)
        assert tuple(out.shape) == (R, len(pop), market.S, 20)
        check_classes(views, evs, pns, labels, R, cfg, f"{case} / {name}")


def test_last_bar_entry_and_force_close(torch_cuda):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    cfg = sim_oracle.config_of(28_401_120, 1)
    for N in range(3000, 3040):
        market, bank, close, bank_h = _market(torch_cuda, N)
        _, ev, _ = sim_oracle.lane(close[0], bank_h[0, 0], DENSE, cfg, event_cap=N + 2)
        if len(ev) >= 2 and (int(ev[-2]) & 0x3FFFFFFF) == N - 1 and (int(ev[-1]) & 0x3FFFFFFF) == N - 1:
            break
    else:
        pytest.fail("no length in 3000..3039 puts an entry on the last bar")
    cfg = sim_oracle.config_of(market.minute0, 1)
    pop = _population()
    _, evs, pns = sim_oracle.population(close, bank_h, ROW, pop, cfg, event_cap=N + 2)
    labels = np.zeros((market.S, N), np.uint8)
    labels[:, -1] = 1                                   # the last bar's entry and force-close form class 1
    labels[:, N // 2:N - 1] = 2
    _, views = PopulationSweep.from_bank(market, bank, PERIODS).class_stats(pop, torch_cuda.from_numpy(labels).cuda(), 3)
    check_classes(views, evs, pns, labels, 3, cfg, "last bar")
    assert views[1]["n_records"].max() == 2


def test_invariants_shared_rows_and_lost_records(torch_cuda):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    market, bank, close, _ = _market(torch_cuda, 30_000)
    pop = _population()
    sweep = PopulationSweep.from_bank(market, bank, PERIODS)
    S, N = market.S, market.N
    # R = 1, every label 0: the lane's own stats
    _, views = sweep.class_stats(pop, torch_cuda.zeros((S, N), dtype=torch_cuda.uint8, device="cuda"), 1)
    sim_oracle.assert_lanes(views[0], sweep.lane_stats(), "R=1", atol=0)
    # a partition (every label < R): class sums of the counts are the lane's, net profit within rounding
    rng = np.random.default_rng(3)
    labels = torch_cuda.from_numpy(rng.integers(0, 6, (S, N)).astype(np.uint8)).cuda()
    _, views = sweep.class_stats(pop, labels, 6)
    lanes = sweep.lane_stats()
    for k in ("n_records", "n_wins", "n_losses"):
        assert np.array_equal(sum(v[k] for v in views), lanes[k]), k
    scale = np.abs(lanes["total_profit"]) + np.abs(lanes["total_loss"])
    assert np.all(np.abs(sum(v["net_profit"] for v in views) - lanes["net_profit"]) <= 1e-9 * scale)
    # one shared row is bit-equal to the row repeated for every symbol, and to its expanded view
    row = labels[2:3]
    a, _ = sweep.class_stats(pop, row, 6)
    b, _ = sweep.class_stats(pop, row.expand(S, N).contiguous(), 6)
    c, _ = sweep.class_stats(pop, row.expand(S, N), 6)
    assert torch_cuda.equal(a.view(torch_cuda.int64), b.view(torch_cuda.int64))
    assert torch_cuda.equal(a.view(torch_cuda.int64), c.view(torch_cuda.int64))
    # an event buffer too small for a lane: n_records -1, score NaN, zeros, in every class
    small = PopulationSweep.from_bank(market, bank, PERIODS, event_cap=4)
    small.evaluate(pop)
    indiv = torch_cuda.from_numpy(small._unique(pop)[0].view(np.uint8)).cuda()
    R = 3
    out = torch_cuda.empty((R, len(pop), S, 20), dtype=torch_cuda.float64, device="cuda")
    _lib.call("b200bt_class_stats", market.close.data_ptr(), _lib.ld(market.close), S, N, indiv.data_ptr(), len(pop),
              C.byref(small.cfg), small._stats.data_ptr(), small._events.data_ptr(), 4, labels.data_ptr(), N, R,
              out.data_ptr(), _lib.current_stream())
    got = out.cpu().numpy()
    n_rec = small._stats[:, :, 0].cpu().numpy()
    lost = n_rec > 4
    assert lost.any() and (~lost).any()
    for r in range(R):
        assert np.all(got[r][lost][:, 0] == -1.0) and np.all(np.isnan(got[r][lost][:, 12]))
        assert np.all(got[r][lost][:, 1:12] == 0.0)
        assert np.all(got[r][~lost][:, 0] >= 0.0)


def _regime_close(rng, bar_minutes, days_per_segment=2):
    """Close prices with stretches that rise, fall, stay flat, swing wildly, drift gently up / down and chop."""
    per_day = 1440 // bar_minutes
    k = np.sqrt(bar_minutes)
    segments = [(1e-4 * bar_minutes, 2e-5 * k), (-1e-4 * bar_minutes, 2e-5 * k), (0.0, 1e-6 * k), (0.0, 0.1 * k),
                (2.5e-5 * bar_minutes, 2e-6 * k), (-2.5e-5 * bar_minutes, 2e-6 * k), (0.0, 5e-3 * k)]
    steps = []
    for drift, vol in segments:
        n = days_per_segment * per_day
        steps.append(drift + vol * rng.standard_normal(n))
    x = np.concatenate(steps)
    return (100.0 * np.exp(np.cumsum(x))).astype(np.float32)


def _threshold_close(row, thr):
    """The window's deciding statistics sit within 1e-12 relative of a threshold."""
    near = lambda v, t: np.isfinite(v) and abs(v - t) <= 1e-12 * max(abs(t), 1e-300)
    return (near(row["volatility"], thr["volatile"]["volatility"]) or near(row["change_pct"], thr["bull"]["price_change"])
            or near(row["change_pct"], thr["bear"]["price_change"]) or near(abs(row["change_pct"]), thr["ranging"]["price_range"])
            or near(row["up_frac"], thr["bull"]["trend_strength"]) or near(row["down_frac"], thr["bear"]["trend_strength"])
            or near(row["mean_strength"], thr["ranging"]["trend_strength"]))


@pytest.mark.parametrize("bar_minutes, sample_minutes", [(1, 60), (1, 15), (5, 60), (5, 15)])
def test_labels_match_the_restatement(torch_cuda, bar_minutes, sample_minutes):
    from ai_crypto_trader_b200 import regime
    from ai_crypto_trader_b200.sweep import MarketData
    rng = np.random.default_rng(bar_minutes * 100 + sample_minutes)
    close = np.stack([_regime_close(rng, bar_minutes), _regime_close(rng, bar_minutes)])
    market = MarketData.from_close(torch_cuda.from_numpy(close).cuda(), minute0=28_401_120 + 35, bar_minutes=bar_minutes)
    labels, windows = regime.regime_labels(market, sample_minutes)
    rows = regime.trend_rows(market).cpu().numpy()
    got_labels = labels.cpu().numpy()
    thr = regime.thresholds_from_env()
    branches, near = set(), 0
    for s in range(market.S):
        want_labels, want = regime_ref.symbol_labels(rows[0, s], rows[1, s], rows[2, s], rows[3, s], market.minute0,
                                                     bar_minutes, sample_minutes, thr)
        got = windows[s]
        assert len(got) == len(want) > 5
        for g, w in zip(got, want):
            assert g["start_minute"] == w["start_minute"] and g["n_points"] == w["n_points"]
            for k in ("change_pct", "mean_strength", "up_frac", "down_frac", "sideways_frac"):
                assert g[k] == pytest.approx(w[k], rel=1e-12, abs=1e-12, nan_ok=True), k
            assert g["volatility"] == pytest.approx(w["volatility"], rel=1e-9, nan_ok=True)
            if g["label"] != w["label"]:
                assert _threshold_close(w, thr), (s, w)
                near += 1
            branches.add(w["branch"])
        # bar labels follow the device's own windows exactly
        dev_rows = [dict(start_minute=int(g["start_minute"]), label=int(g["label"])) for g in got]
        assert np.array_equal(got_labels[s], regime_ref.bar_labels(market.N, market.minute0, bar_minutes, dev_rows))
        if near == 0:
            assert np.array_equal(got_labels[s], want_labels)
    print(f"bar {bar_minutes} / sample {sample_minutes}: {near} windows within 1e-12 of a threshold; branches {sorted(branches)}")
    assert {"volatile", "bull", "bear", "ranging", "default bull", "default bear"} <= branches, branches
    # primary: one symbol's labels for every symbol
    shared, _ = regime.regime_labels(market, sample_minutes, primary=1)
    assert shared.stride(0) == 0 and torch_cuda.equal(shared[0], labels[1])


def test_points_are_the_monitor_on_the_cut_market(torch_cuda):
    from ai_crypto_trader_b200 import indicators, regime
    from ai_crypto_trader_b200.sweep import MarketData
    rng = np.random.default_rng(5)
    close = _regime_close(rng, 1, 1)
    ohlcv = np.stack([close, close, close, close, np.ones_like(close)])[:, None, :]      # [5][1][N]
    market = MarketData(ohlcv, bar_minutes=1)
    rows = regime.trend_rows(market).cpu().numpy()
    idx, _, _, trend, strength = regime_ref.points(rows[0, 0], rows[1, 0], rows[2, 0], rows[3, 0], market.minute0, 1, 60)
    for j in (0, 7, len(idx) // 2, len(idx) - 1):
        t = int(idx[j])
        cut = MarketData(np.ascontiguousarray(ohlcv[:, :, :t + 1]), minute0=market.minute0, bar_minutes=1)
        mon = indicators.multi_timeframe_indicators(cut, 0)
        assert mon["trend"] == regime_ref.TREND_NAMES[trend[j]], t
        assert mon["trend_strength"] == pytest.approx(strength[j], rel=1e-6), t


def test_service_end_to_end(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.regime import SCORED_REGIMES, MarketRegimeService
    from ai_crypto_trader_b200.sweep import MarketData
    from oracle import sim_oracle
    rng = np.random.default_rng(9)
    close = np.stack([_regime_close(rng, 1), _regime_close(rng, 1)])
    market = MarketData.from_close(torch_cuda.from_numpy(close).cuda(), bar_minutes=1, symbols=["BTCUSDC", "ETHUSDC"])
    svc = MarketRegimeService(market)
    pop = synth.random_population(24, seed=4)
    perf = svc.regime_performance(pop)
    labels = svc.labels().cpu().numpy()
    assert np.array_equal(labels[0], labels[1])                      # PRIMARY_TRADING_SYMBOL's labels everywhere
    cfg = sim_oracle.config_of(market.minute0, 1)
    bank_h = svc.sweep.bank.cpu().numpy()
    lanes, evs, pns = sim_oracle.population(close, bank_h, svc.sweep.period_row, pop, cfg, event_cap=market.N + 2)
    seen = set()
    for i, p in enumerate(perf):
        for k in ("sharpe_ratio", "win_rate", "max_drawdown", "profit_factor"):
            assert p[k] == pytest.approx(np.mean(lanes[k][i]), rel=1e-9), (i, k)
        classes = [regime_ref.class_stats(evs[i][s], pns[i][s], labels[s], 4, cfg) for s in range(market.S)]
        want = {}
        for r, name in enumerate(SCORED_REGIMES):
            n = sum(c[r]["n_records"] for c in classes)
            if n == 0:
                continue
            loss = sum(c[r]["total_loss"] for c in classes)
            want[name] = {"trade_count": int(n), "win_rate": sum(c[r]["n_wins"] for c in classes) / n,
                          "profit_factor": sum(c[r]["net_profit"] for c in classes) / abs(loss) if loss != 0 else 1,
                          "sharpe_ratio": np.mean([c[r]["sharpe_ratio"] for c in classes]),
                          "max_drawdown": np.mean([c[r]["max_drawdown"] for c in classes])}
        assert set(p["regime_performance"]) == set(want), i
        for name, w in want.items():
            g = p["regime_performance"][name]
            assert g["trade_count"] == w["trade_count"]
            for k in ("win_rate", "profit_factor", "sharpe_ratio", "max_drawdown"):
                assert g[k] == pytest.approx(w[k], rel=1e-9, abs=1e-12), (i, name, k)
            seen.add(name)
    assert len(seen) >= 3, seen
    for regime in SCORED_REGIMES:
        scores = [svc._calculate_regime_score(p, regime) for p in perf]
        best = sorted(range(len(pop)), key=lambda j: scores[j], reverse=True)[0]
        chosen = asyncio.run(svc.select_strategy_for_regime(regime, pop))
        assert chosen is pop[best] and svc.regime_strategy_mapping[regime] == best
    assert svc.regime_scores(pop).shape == (len(pop), 4)
    assert asyncio.run(svc.select_strategy_for_regime("bull", [])) is None


def test_full_size_partition_and_oracle_slice(torch_cuda):
    """configs[1]: 1024 random individuals x 10 symbols x 1M 1-minute bars."""
    from ai_crypto_trader_b200 import regime, synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    S, N, POP = 10, 1_000_000, 1024
    ohlcv = synth.synth_ohlcv(S, N)
    market = MarketData(ohlcv)
    sweep = PopulationSweep(market)
    pop = synth.random_population(POP, seed=42)
    labels, _ = regime.regime_labels(market)
    out, views = sweep.class_stats(pop, labels, 5)
    lanes = sweep.lane_stats()
    for k in ("n_records", "n_wins", "n_losses"):
        assert np.array_equal(sum(v[k] for v in views), lanes[k]), k
    scale = np.abs(lanes["total_profit"]) + np.abs(lanes["total_loss"])
    assert np.all(np.abs(sum(v["net_profit"] for v in views) - lanes["net_profit"]) <= 1e-9 * scale)
    cfg = sim_oracle.config_of(market.minute0, 1)
    lab = labels.cpu().numpy()
    close = ohlcv[3]
    rng = np.random.default_rng(1)
    picks = [(int(i), int(s)) for i, s in zip(rng.integers(0, POP, 64), rng.integers(0, S, 64))]
    for i, s in picks:
        row = sweep.bank[s, sweep.period_row[pop[i]["rsi_period"]]].cpu().numpy()
        _, ev, pn = sim_oracle.lane(close[s], row, pop[i], cfg, event_cap=N + 2)
        want = regime_ref.class_stats(ev, pn, lab[s], 5, cfg)
        for r in range(5):
            sim_oracle.assert_lanes({k: v[i, s] for k, v in views[r].items()}, want[r],
                                    f"full size lane ({i}, {s}) class {r}", atol=0)
