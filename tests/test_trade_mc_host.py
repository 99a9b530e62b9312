"""The trade-sequence Monte-Carlo restatement (tests/trade_mc_ref.py) on the host: the original trade order through its trip
PnL and equity walk reproduces the reference's own metrics, the shuffle is a bijection with uniform position marginals,
and the bootstrap index stream is oracle/mc_ref's."""
import numpy as np
import pytest
from scipy import stats

import trade_mc_ref as R
from conftest import unjson
from oracle import mc_ref, simulate_ref


def _records(meta, arrays, case):
    sym = case["symbol"]
    period = case["params"].get("rsi_period", 14)
    pts = simulate_ref.market_points(arrays[f"close_{sym}"], arrays[f"rsi_{sym}_{period}"], f"SYN{sym:03d}USDT",
                                     meta["minute0"])
    return simulate_ref.simulate_trades(dict(case["params"]), pts)


def test_original_order_reproduces_reference_drawdown_and_net_profit(sim_golden):
    """All 20 golden cases: the trip PnL equals the reference's exit records, and walking the trips in their own order
    gives the reference's max_drawdown, net profit and final equity bit for bit."""
    meta, arrays = sim_golden
    assert len(meta["cases"]) == 20
    for case in meta["cases"]:
        key = case["key"]
        fee, trips = R.trips_from_records(_records(meta, arrays, case))
        pnl = arrays[f"pnl_{key}"]
        assert np.array_equal(trips, pnl[1::2]) and np.array_equal(np.full(len(trips), -fee), pnl[0::2]), key
        T = len(trips)
        E, dd = R.walk(fee, trips, np.arange(T, dtype=np.int64)[None, :])
        m = case["metrics"]
        assert float(dd[0]) == unjson(m["max_drawdown"]), key
        assert R.net_profit(fee, trips) == unjson(m["net_profit"]), key
        assert float(E[0]) == arrays[f"equity_{key}"][-1], key


def test_walk_follows_the_per_record_rule_on_ties_and_empty_lanes():
    # T = 0: initial capital, no drawdown
    E, dd = R.walk(1.0, np.zeros(0), np.zeros((3, 0), dtype=np.int64))
    assert (E == 10000.0).all() and (dd == 0).all()
    # a trip that exactly refunds the fee ties the peak: not a new peak, its drawdown is 0
    E, dd = R.walk(10.0, np.array([10.0, 25.0, -100.0]), np.array([[0, 1, 2]]))
    assert E[0] == 10000.0 - 30 + 35 - 100
    want = max((10000.0 - 9990.0) / 10000.0, (10015.0 - 10005.0) / 10015.0, (10015.0 - 9905.0) / 10015.0)
    assert dd[0] == want


def test_feistel_shuffle_is_a_permutation_exhaustive():
    for T in range(1, 4097):
        idx = R.shuffle_indices(T, 3, seed=1234 + T, lane_id=T % 7, path_offset=T)
        assert (np.sort(idx, axis=1) == np.arange(T)).all(), T


@pytest.mark.parametrize("T", [4097, 12_345, 65_536, 65_537, 333_333, 1 << 20])
def test_feistel_shuffle_is_a_permutation_sampled(T):
    idx = R.shuffle_indices(T, 1, seed=77, lane_id=3, path_offset=5)
    assert np.array_equal(np.sort(idx[0]), np.arange(T))


@pytest.mark.parametrize("T", [3, 4, 5, 8, 16, 33, 64, 100, 1000])
def test_feistel_shuffle_position_marginals_are_uniform(T):
    """Chi-square of the trip found at a few positions over 20 000 keyed paths (fixed seed: deterministic)."""
    n = 20_000
    idx = R.shuffle_indices(T, n, seed=11, lane_id=5)
    for pos in sorted({0, 1, T // 2, T - 1}):
        p = stats.chisquare(np.bincount(idx[:, pos], minlength=T)).pvalue
        assert p > 1e-3, (T, pos, p)


@pytest.mark.parametrize("T", [3, 8, 33, 100, 1000])
def test_feistel_shuffle_positions_0_and_1_are_uncorrelated(T):
    """A uniform permutation has corr(pi(0), pi(1)) = -1/(T-1); the keyed family stays within 5 standard errors."""
    n = 20_000
    idx = R.shuffle_indices(T, n, seed=23, lane_id=2)
    r = np.corrcoef(idx[:, 0], idx[:, 1])[0, 1]
    assert abs(r + 1 / (T - 1)) < 5 / np.sqrt(n), (T, r)


@pytest.mark.parametrize("T,block_len", [(1, 1), (2, 1), (45, 1), (45, 5), (1000, 16), (1000, 1000)])
def test_bootstrap_block_rule_is_mc_ref_s(T, block_len):
    """Lane id 1 puts mc_ref's bootstrap mode word in the same counter slot: the trip index stream of T trips is
    mc_ref._increments' day-index stream over a table of T returns for T steps, path offset and block length included."""
    table = np.arange(T, dtype=np.float32)                # value = index (exact in fp32)
    want = mc_ref._increments(1, 40, T, 2024, 3, table, block_len, True).T.astype(np.int64)
    assert np.array_equal(R.bootstrap_indices(T, 40, 2024, lane_id=1, path_offset=3, block_len=block_len), want)


def test_paths_do_not_depend_on_sharding_or_other_lanes():
    trips = np.linspace(-40, 55, 37)
    a = R.simulate(3.0, trips, 64, seed=5, method="shuffle", lane_id=9)
    b0 = R.simulate(3.0, trips, 32, seed=5, method="shuffle", lane_id=9)
    b1 = R.simulate(3.0, trips, 32, seed=5, method="shuffle", lane_id=9, path_offset=32)
    assert np.array_equal(a[0], np.concatenate([b0[0], b1[0]])) and np.array_equal(a[1], np.concatenate([b0[1], b1[1]]))


def test_statistics_blocks_have_the_result_schema():
    rng = np.random.default_rng(0)
    finals = (10000 + rng.normal(0, 50, 1001)).astype(np.float32)
    maxdd = rng.uniform(0, 0.1, 1001).astype(np.float32)
    st = R.statistics(finals, maxdd, 10000.0, 0.95)
    assert list(st["percentiles"]) == ["1", "5", "10", "25", "50", "75", "90", "95", "99"]
    assert set(st["percentiles"]["5"]) == {"equity", "pct_change"}
    assert set(st["risk_metrics"]["max_drawdown"]) == {"mean", "median", "p95", "max"}
    assert st["risk_metrics"]["max_drawdown"]["p95"] == np.percentile(maxdd.astype(np.float64), 95)
