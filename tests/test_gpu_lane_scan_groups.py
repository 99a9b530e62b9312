"""Thread-per-lane scan: machines with several events inside one 4-bar group.

Inside a 4-bar group a machine's thresholds move with every event, so each bar after an event is screened against
different thresholds than the group started with.  The existing tiled tests rarely put several events of one lane into
one group; the population below puts machines with 1, 2, 3 and 4 events in the same group into one packed warp:
inverted thresholds that fire on every bar, a take-profit / stop-loss so small that a position closes on the bar after
it opened, ordinary lanes, and one lane whose price screen passes on a bar that the float64 exit test then rejects."""
import numpy as np
import pytest

from gpu_fixtures import torch_cuda

N_BARS = 40_001               # not a multiple of the 128-bar tile: a ragged last tile
PERIODS = (5, 7)              # at most two RSI rows per warp (the scan's packing rule)
NEAR_BAND = 3                 # the lane whose planted bar sits inside the fp32 screening band
SW_MARGIN = 1e-6              # relative width of that band (csrc/sweep_dev.cuh)


def _population():
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(64, seed=11)
    for i, p in enumerate(pop):
        p["rsi_period"] = PERIODS[(i // 8) % 2]
    for i in range(0, 3):       # long on every flat bar, out again on the next: four events per group
        pop[i].update(rsi_oversold=99, rsi_overbought=1, take_profit=1 + i, stop_loss=1)
    pop[NEAR_BAND].update(rsi_period=5, rsi_oversold=45, rsi_overbought=100, take_profit=1, stop_loss=1)   # price exits only
    for i in range(4, 12):      # exits on the bar after the entry (both triggers within one tick)
        pop[i].update(rsi_oversold=30 + i, rsi_overbought=70 - i, take_profit=0.0001 * i, stop_loss=0.0001 * i)
    for i in range(12, 20):     # inverted, but not on every bar
        pop[i].update(rsi_oversold=55 + i, rsi_overbought=45 - i)
    return pop


def _near_band_price(e: np.float32, tp: float) -> np.float32:
    """the largest fp32 price whose float64 return on entry price `e` stays below `tp` (no take-profit exit)"""
    p = np.float32(np.float64(e) * (1.0 + tp))
    while (np.float64(p) - np.float64(e)) / np.float64(e) >= tp:
        p = np.nextafter(p, np.float32(0))
    return p


def _market_data():
    """synthetic closes with one planted bar: after an entry of the NEAR_BAND lane, a price on its take-profit band"""
    from ai_crypto_trader_b200 import synth
    from oracle import indicators_ref, sim_oracle
    ohlcv = synth.synth_ohlcv(1, N_BARS, first_symbol=6)
    close = ohlcv[3, 0]
    p = _population()[NEAR_BAND]
    cfg = sim_oracle.config_of(0, 1)
    _, ev, _ = sim_oracle.lane(close, indicators_ref.rsi_bank(close, [5])[0], p, cfg, event_cap=N_BARS + 1)
    entries = [int(w) for w in ev if not (w & 0x40000000) and N_BARS // 2 < int(w & 0x3fffffff) < N_BARS - 2]
    t = entries[0] & 0x3fffffff
    e, tp = close[t], p["take_profit"] / 100
    close[t + 1] = _near_band_price(e, tp)
    # the screen passes (price at or above the fp32 threshold the kernel holds), the fp32 test cannot decide ...
    hi_c, hi_d = np.float32((1.0 + tp) * (1.0 - SW_MARGIN)), np.float32((1.0 + tp) * (1.0 + SW_MARGIN))
    assert e * hi_c <= close[t + 1] < e * hi_d
    # ... and the float64 test rejects: the position is still open after the planted bar
    _, ev2, _ = sim_oracle.lane(close, indicators_ref.rsi_bank(close, [5])[0], p, cfg, event_cap=N_BARS + 1)
    bars = ev2 & 0x3fffffff
    k = int(np.searchsorted(bars, t))
    assert bars[k] == t and bars[k + 1] > t + 1
    return ohlcv


def _group_counts(ohlcv, population, periods):
    """events per (lane, 4-bar group) by the C oracle, for the first warp"""
    from oracle import indicators_ref, sim_oracle
    close = ohlcv[3, 0]
    bank = indicators_ref.rsi_bank(close, list(periods))
    cfg = sim_oracle.config_of(0, 1)
    seen = set()
    for p in population[:32]:
        _, ev, _ = sim_oracle.lane(close, bank[list(periods).index(p["rsi_period"])], p, cfg, event_cap=N_BARS + 1)
        seen.update(np.unique(np.bincount((ev & 0x3fffffff) // 4)).tolist())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [
    dict(warm=64, chunks=8, order_by="identity"),      # warm-up shorter than a tile
    dict(warm=4096, chunks=5, order_by="identity"),
])
def test_tiled_groups_with_several_events_match_fused(torch_cuda, opts):
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    ohlcv = _market_data()
    population = _population()
    assert {1, 2, 3, 4} <= _group_counts(ohlcv, population, PERIODS)   # the first warp needs 1 to 4 passes in a group
    market = MarketData(ohlcv)
    cap = N_BARS + 1
    tiled = PopulationSweep(market, event_cap=cap, mode="tiled", chunk_options=opts)
    fused = PopulationSweep(market, event_cap=cap, mode="fused")
    f_f = fused.evaluate(population)
    st_f, ev_f = fused.lane_stats(), fused.events()
    live = np.arange(cap)[None, None, :] < st_f["n_records"][:, :, None]
    for _ in range(2):                          # the second sweep of the bank goes through the zone map
        f_t = tiled.evaluate(population)
        st_t = tiled.lane_stats()
        np.testing.assert_array_equal(st_t["n_records"], st_f["n_records"])
        np.testing.assert_array_equal(st_t["trade_hash"], st_f["trade_hash"])
        np.testing.assert_array_equal(tiled.events()[live], ev_f[live])
        np.testing.assert_allclose(f_t, f_f, rtol=1e-9, atol=1e-11)
    assert tiled._zones is not None
    assert st_f["n_records"][0, 0] > N_BARS // 2      # (the every-bar lanes really fire on every other bar at least)
