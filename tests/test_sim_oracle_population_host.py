"""oracle/sim_oracle.py's population runner and lane check on the CPU: population() is a loop of lane() byte for byte,
and assert_lanes() holds the exact fields exact and the float fields to max(rtol |want|, atol), NaN and infinities
included."""
import numpy as np
import pytest

from oracle import indicators_ref, sim_oracle

PERIODS = (5, 14)
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)


@pytest.fixture(scope="module")
def market():
    from ai_crypto_trader_b200 import synth
    close = synth.synth_ohlcv(2, 3000)[3]
    bank = np.stack([indicators_ref.rsi_bank(close[s], PERIODS) for s in range(2)])
    pop = synth.random_population(10, seed=3)
    for p in pop:
        p["rsi_period"] = PERIODS[int(p["rsi_period"]) % 2]
    pop[1].pop("rsi_period")                                      # reads period 14
    return close, bank, pop + [dict(DENSE)], sim_oracle.config_of(synth.EPOCH_2024_MINUTES, 1)


@pytest.mark.parametrize("workers", [1, 4])
@pytest.mark.parametrize("by", ["dict", "callable"])
def test_population_is_a_loop_of_lanes(market, by, workers):
    close, bank, pop, cfg = market
    row_of = {5: 0, 14: 1} if by == "dict" else (lambda p: 0 if p.get("rsi_period", 14) == 5 else 1)
    cap = close.shape[1] + 2
    stats, events, pnl = sim_oracle.population(close, bank, row_of, pop, cfg, event_cap=cap, workers=workers)
    plain, none_ev, none_pn = sim_oracle.population(close, bank, row_of, pop, cfg, workers=workers)
    assert stats.dtype == sim_oracle.STATS_DTYPE and stats.shape == (len(pop), 2)
    assert none_ev is None and none_pn is None
    assert stats.tobytes() == plain.tobytes()
    for i, p in enumerate(pop):
        for s in range(2):
            st, ev, pn = sim_oracle.lane(close[s], bank[s, 0 if p.get("rsi_period", 14) == 5 else 1], p, cfg, cap)
            assert stats[i, s].tobytes() == st.tobytes(), (i, s)
            assert events[i][s].tobytes() == ev.tobytes() and pnl[i][s].tobytes() == pn.tobytes(), (i, s)
    assert int(stats["n_records"][-1].min()) > 500                # the dense lane fills its event lists


def _stats(market):
    close, bank, pop, cfg = market
    return sim_oracle.population(close, bank, {5: 0, 14: 1}, pop, cfg)[0]


def _changed(want, field, value, at=(3, 1)):
    got = want.copy()
    got[field][at] = value
    return got


def test_assert_lanes_refuses_each_kind_of_difference(market):
    want = _stats(market)
    sim_oracle.assert_lanes(want.copy(), want, "same")
    w = float(want["net_profit"][3, 1])
    assert w != 0.0
    cases = [("n_wins", want["n_wins"][3, 1] + 1),
             ("trade_hash", int(want["trade_hash"][3, 1]) ^ (1 << 63)),
             ("net_profit", w * (1 + 2e-9)),
             ("sharpe_ratio", np.nan),
             ("profit_factor", -np.inf)]
    ref = {"sharpe_ratio": 1.5, "profit_factor": np.inf}            # the want side of the NaN and infinity cases
    for field, value in cases:
        base = _changed(want, field, ref[field]) if field in ref else want
        with pytest.raises(AssertionError, match=f"lanes: {field} .* first at \\(3, 1\\)"):
            sim_oracle.assert_lanes(_changed(base, field, value), base, "lanes")


def test_assert_lanes_accepts_nan_and_differences_within_tolerance(market):
    want = _changed(_changed(_stats(market), "sharpe_ratio", np.nan), "profit_factor", np.inf)
    w = float(want["net_profit"][3, 1])
    sim_oracle.assert_lanes(want.copy(), want, "NaN against NaN, inf against inf")
    sim_oracle.assert_lanes(_changed(want, "net_profit", w * (1 + 0.5e-9)), want, "rtol")
    small = _changed(want, "total_loss", 3e-12, at=(0, 0))
    sim_oracle.assert_lanes(_changed(small, "total_loss", 3e-12 + 0.9e-11, at=(0, 0)), small, "atol")
    with pytest.raises(AssertionError):
        sim_oracle.assert_lanes(_changed(small, "total_loss", 3e-12 + 1.1e-11, at=(0, 0)), small, "beyond atol")


def test_assert_lanes_reads_mappings_and_dict_lists(market):
    want = _stats(market)
    as_map = {f: want[f] for f in sim_oracle.STATS_FIELDS}
    sim_oracle.assert_lanes(as_map, want, "mapping")
    rows = [{f: (int(r[f]) if f == "trade_hash" else float(r[f])) for f in sim_oracle.STATS_FIELDS} for r in want[:, 0]]
    sim_oracle.assert_lanes(rows, want[:, 0], "dicts")
    rows[2]["trade_hash"] ^= 1 << 63
    with pytest.raises(AssertionError, match="trade_hash"):
        sim_oracle.assert_lanes(rows, want[:, 0], "dicts")


def test_assert_events_compares_the_recorded_words(market):
    close, bank, pop, cfg = market
    _, events, _ = sim_oracle.population(close, bank, {5: 0, 14: 1}, pop, cfg, event_cap=64)
    buf = np.full((len(pop), 2, 80), 7, dtype=np.uint32)
    for i in range(len(pop)):
        for s in range(2):
            buf[i, s, :len(events[i][s])] = events[i][s]
    sim_oracle.assert_events(buf, events, "padded")
    i = next(i for i in range(len(pop)) if len(events[i][1]))
    buf[i, 1, 0] ^= 1
    with pytest.raises(AssertionError, match=f"lane \\({i}, 1\\)"):
        sim_oracle.assert_events(buf, events, "flipped")
