"""GPU trade-sequence Monte-Carlo (csrc/trade_mc.cu) against the reference's records, the C oracle and the NumPy
restatement tests/trade_mc_ref.py: trip PnL bit for bit, every path's final equity and drawdown bit for bit."""
import numpy as np
import pytest

import trade_mc_ref as R
from conftest import unjson
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

SMEM_TRIPS = 6144          # csrc/trade_mc.cu TMC_SMEM_TRIPS: larger lanes take the L2 form


@pytest.fixture(scope="module")
def mc(torch_cuda):
    from ai_crypto_trader_b200.trade_monte_carlo import TradeMonteCarlo
    return TradeMonteCarlo()


def _golden_sweep(meta, arrays):
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    syms = sorted({c["symbol"] for c in meta["cases"]})
    ohlcv = np.zeros((5, len(syms), meta["n_bars"]), dtype=np.float32)
    for j, s in enumerate(syms):
        ohlcv[3, j] = arrays[f"close_{s}"]
    market = MarketData(ohlcv, minute0=meta["minute0"])
    names = list(dict.fromkeys(c["name"] for c in meta["cases"]))
    by_name = {c["name"]: c["params"] for c in meta["cases"]}
    sweep = PopulationSweep(market, rsi_periods=meta["periods"], optimization_goals=meta["goals"])
    return sweep, syms, names, [dict(by_name[n]) for n in names]


def test_trip_pnl_matches_reference_records_on_golden_cases(torch_cuda, sim_golden):
    meta, arrays = sim_golden
    sweep, syms, names, population = _golden_sweep(meta, arrays)
    population = population + [dict(population[0])]          # a duplicate: swept once, returned twice
    trip, n_trips, fee = sweep.trade_pnl(population)
    trip, n_trips, fee = trip.cpu().numpy(), n_trips.cpu().numpy(), fee.cpu().numpy()
    assert np.array_equal(trip[-1], trip[0]) and np.array_equal(n_trips[-1], n_trips[0])
    for c in meta["cases"]:
        i, j, key = names.index(c["name"]), syms.index(c["symbol"]), c["key"]
        pnl = arrays[f"pnl_{key}"]
        T = len(pnl) // 2
        assert n_trips[i, j] == T == c["n_records"] // 2, key
        assert np.array_equal(trip[i, j, :T], pnl[1::2]), key                  # bit-identical float64
        if T:
            assert np.array_equal(np.full(T, -fee[i, j]), pnl[0::2]), key


def test_trip_pnl_matches_c_oracle_on_tiled_sweep(torch_cuda):
    """262 144-bar lanes through the thread-per-lane schedule, with a lane that never trades, one whose only position is
    force-closed on the last bar, and long and short trips."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import indicators_ref, sim_oracle
    S, N = 2, 262_144
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=7)
    market = MarketData(ohlcv)
    sweep = PopulationSweep(market, mode="tiled")
    pop = synth.random_population(30, seed=17)
    pop[0].update(rsi_oversold=0, rsi_overbought=100)                                     # never enters
    pop[1].update(rsi_period=14, rsi_oversold=45, rsi_overbought=100, take_profit=1e4, stop_loss=1e4)  # one long, held
    pop[2].update(rsi_oversold=35, rsi_overbought=65, rsi_period=5, take_profit=1, stop_loss=1)       # always trading
    trip, n_trips, fee = (t.cpu().numpy() for t in sweep.trade_pnl(pop))
    assert sweep.plan(pop) is not None and type(sweep.plan(pop)[0]).__name__ == "TilePlan"
    bank = np.stack([indicators_ref.rsi_bank(ohlcv[3, s], sweep.periods) for s in range(S)])
    want, events, pnls = sim_oracle.population(ohlcv[3], bank, sweep.period_row, pop, sim_oracle.config_of(market.minute0, 1),
                                               event_cap=N + 1)
    sides = set()
    for s in range(S):
        for i, p in enumerate(pop):
            ev, pnl = events[i][s], pnls[i][s]
            T = int(want["n_records"][i, s]) // 2
            assert n_trips[i, s] == T, (i, s)
            assert np.array_equal(trip[i, s, :T], pnl[1::2]), (i, s)
            assert fee[i, s] == 10000 * (min(p.get("max_position_size", 5), 20) / 100) * 0.001
            sides |= set((ev[0::2] >> 31).tolist())
            if i == 1:
                assert T == 1 and (ev[-1] & 0x3FFFFFFF) == N - 1, "force-closed on the last bar"
    assert n_trips[0].tolist() == [0, 0]
    assert sides == {0, 1}, "long and short trips"


def _synthetic_lanes(Ts, seed=3):
    rng = np.random.default_rng(seed)
    ld = max(max(Ts), 1)
    trips = np.zeros((len(Ts), ld))
    fees = np.zeros(len(Ts))
    for r, T in enumerate(Ts):
        trips[r, :T] = rng.normal(0.3, 12.0, T) * rng.choice([1.0, 4.0], T)
        fees[r] = [0.5, 1.0, 0.25][r % 3]
    return trips, np.array(Ts, dtype=np.int32), fees


@pytest.mark.parametrize("method,block_len", [("bootstrap", 1), ("bootstrap", 7), ("shuffle", 1)])
def test_paths_bit_equal_oracle(torch_cuda, mc, method, block_len):
    """Lanes of T = 0, 1, 2, 33, 5000 and one above the shared-memory budget in one call, non-zero path offset."""
    torch = torch_cuda
    Ts = [0, 1, 2, 33, 5000, SMEM_TRIPS + 857]
    trips, nt, fees = _synthetic_lanes(Ts)
    ids = [40 + r for r in range(len(Ts))]
    n, off, seed = 192, 1000, 777
    finals, maxdd = mc.simulate(torch.from_numpy(trips).cuda(), nt, fees, n, method, block_len, 10000.0, seed,
                                path_offset=off, lane_ids=ids)
    finals, maxdd = finals.cpu().numpy(), maxdd.cpu().numpy()
    for r, T in enumerate(Ts):
        wf, wd = R.simulate(fees[r], trips[r, :T], n, seed, method, lane_id=ids[r], path_offset=off, block_len=block_len)
        assert np.array_equal(finals[r], wf), (method, T)
        assert np.array_equal(maxdd[r], wd), (method, T)
    assert (finals[0] == 10000.0).all() and (maxdd[0] == 0).all()


@pytest.mark.parametrize("method", ["bootstrap", "shuffle"])
def test_paths_do_not_depend_on_sharding_or_other_lanes(torch_cuda, mc, method):
    torch = torch_cuda
    Ts = [700, 33, 5000, SMEM_TRIPS + 100]
    trips, nt, fees = _synthetic_lanes(Ts, seed=9)
    dev = torch.from_numpy(trips).cuda()
    M = 2048
    whole = [t.cpu().numpy() for t in mc.simulate(dev, nt, fees, M, method, 3, 10000.0, 42, path_offset=5)]
    a = [t.cpu().numpy() for t in mc.simulate(dev, nt, fees, M // 2, method, 3, 10000.0, 42, path_offset=5)]
    b = [t.cpu().numpy() for t in mc.simulate(dev, nt, fees, M // 2, method, 3, 10000.0, 42, path_offset=5 + M // 2)]
    for k in range(2):
        assert np.array_equal(whole[k], np.concatenate([a[k], b[k]], axis=1))
    for r in range(len(Ts)):                                 # alone, with its lane id, it draws the same paths
        alone = mc.simulate(dev[r:r + 1], nt[r:r + 1], fees[r:r + 1], M, method, 3, 10000.0, 42, path_offset=5,
                            lane_ids=[r])
        assert np.array_equal(alone[0].cpu().numpy()[0], whole[0][r])
        assert np.array_equal(alone[1].cpu().numpy()[0], whole[1][r])


def test_shuffle_keeps_the_final_equity(torch_cuda, mc):
    """A permutation of the trips sums the same records in another order: every path's final equity equals the original
    order's to 1e-9 relative."""
    torch = torch_cuda
    Ts = [1, 57, 3000, SMEM_TRIPS + 1]
    trips, nt, fees = _synthetic_lanes(Ts, seed=4)
    finals, _ = mc.simulate(torch.from_numpy(trips).cuda(), nt, fees, 4096, "shuffle", 1, 10000.0, 8)
    finals = finals.cpu().numpy()
    for r, T in enumerate(Ts):
        E, _ = R.walk(fees[r], trips[r, :T], np.arange(T)[None, :])
        np.testing.assert_allclose(finals[r], np.float32(E[0]), rtol=1e-9, atol=0)


def _assert_blocks(got, want, key):
    for p, v in want["percentiles"].items():
        assert got["percentiles"][p]["equity"] == v["equity"], (key, p)                   # exact order statistics
        assert got["percentiles"][p]["pct_change"] == v["pct_change"], (key, p)
    gm, wm = got["risk_metrics"], want["risk_metrics"]
    assert gm["var"] == pytest.approx(wm["var"], rel=1e-12, abs=1e-12), key
    for k in ("median", "p95", "max"):
        assert gm["max_drawdown"][k] == wm["max_drawdown"][k], (key, k)
    assert gm["max_drawdown"]["mean"] == pytest.approx(wm["max_drawdown"]["mean"], rel=1e-10, abs=1e-15), key
    for k in ("cvar", "prob_profit", "prob_loss"):
        assert gm[k] == pytest.approx(wm[k], rel=1e-10, abs=1e-15), (key, k)
    for k in ("equity", "pct_change"):
        assert got["expected"][k] == pytest.approx(want["expected"][k], rel=1e-10, abs=1e-12), (key, k)


@pytest.mark.parametrize("method,block_len", [("bootstrap", 1), ("bootstrap", 4), ("shuffle", 1)])
def test_monte_carlo_trades_matches_oracle_dict(torch_cuda, sim_golden, method, block_len):
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from oracle import simulate_ref
    meta, arrays = sim_golden
    case = next(c for c in meta["cases"] if c["key"] == "fast_rsi_tight_0")
    period = case["params"].get("rsi_period", 14)
    pts = simulate_ref.market_points(arrays[f"close_{case['symbol']}"], arrays[f"rsi_{case['symbol']}_{period}"],
                                     "SYN000USDT", meta["minute0"])
    ses = StrategyEvaluationSystem(config={"evolution": {"optimization_goals": meta["goals"]}})
    got = ses.monte_carlo_trades("s1", dict(case["params"]), pts, num_simulations=3001, simulation_method=method,
                                 block_len=block_len, seed=99)
    fee, trips = R.trips_from_records(simulate_ref.simulate_trades(dict(case["params"]), pts))
    finals, maxdd = R.simulate(fee, trips, 3001, 99, method, lane_id=0, block_len=block_len)
    want = R.statistics(finals, maxdd, 10000.0, 0.95)
    assert got["num_trades"] == len(trips) and got["num_simulations"] == 3001 and got["symbol"] == "SYN000USDT"
    m = case["metrics"]
    assert got["original"]["max_drawdown"] == pytest.approx(unjson(m["max_drawdown"]), rel=1e-10)
    assert got["original"]["return_pct"] == pytest.approx(unjson(m["return_pct"]), rel=1e-10)
    _assert_blocks(got, want, method)
    assert ses.monte_carlo_trades("s1", dict(case["params"]), pts, simulation_method="no_such_method") == {}
    assert ses.monte_carlo_trades("s1", dict(case["params"]), []) == {}


def test_monte_carlo_population_matches_oracle_on_sampled_lanes(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import indicators_ref, sim_oracle
    S, N, P, M = 2, 262_144, 32, 600
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=11)
    market = MarketData(ohlcv)
    sweep = PopulationSweep(market)
    pop = synth.random_population(P, seed=21)
    ses = StrategyEvaluationSystem(config={})
    out = ses.monte_carlo_population(pop, market, sweep=sweep, num_simulations=M, seed=5)
    assert out["var"].shape == (P, S) and out["percentile_equity"].shape == (P, S, 9)
    bank = np.stack([indicators_ref.rsi_bank(ohlcv[3, s], sweep.periods) for s in range(S)])
    want, _, pnls = sim_oracle.population(ohlcv[3], bank, sweep.period_row, pop, sim_oracle.config_of(market.minute0, 1),
                                          event_cap=N + 1)
    for s in range(S):
        for i in range(s, P, 7):
            p = pop[i]
            trips = pnls[i][s][1::2]
            fee = 10000 * (min(p.get("max_position_size", 5), 20) / 100) * 0.001
            assert out["num_trades"][i, s] == len(trips)
            assert out["original_max_drawdown"][i, s] == pytest.approx(float(want["max_drawdown"][i, s]), rel=1e-9, abs=1e-12)
            finals, maxdd = R.simulate(fee, trips, M, 5, "bootstrap", lane_id=i * S + s)
            st = R.statistics(finals, maxdd, 10000.0, 0.95)
            np.testing.assert_array_equal(out["percentile_equity"][i, s],
                                          [st["percentiles"][k]["equity"] for k in st["percentiles"]])
            assert out["mdd_p95"][i, s] == st["risk_metrics"]["max_drawdown"]["p95"], (i, s)
            assert out["mdd_max"][i, s] == st["risk_metrics"]["max_drawdown"]["max"], (i, s)
            assert out["var"][i, s] == pytest.approx(st["risk_metrics"]["var"], rel=1e-12, abs=1e-12), (i, s)
            assert out["expected_equity"][i, s] == pytest.approx(st["expected"]["equity"], rel=1e-10), (i, s)


def test_trade_pnl_refuses_a_population_over_the_byte_budget(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(1, 20_000))
    sweep = PopulationSweep(market)
    pop = synth.random_population(8, seed=1)
    with pytest.raises(ValueError, match="bytes"):
        sweep.trade_pnl(pop, max_bytes=1000)
    fit = sweep.evaluate(pop)              # the sweep still evaluates afterwards
    assert np.all(np.isfinite(fit))
