"""Host-side logic of the population sweep that needs no GPU: decoding GA dicts into kernel records, the scheduling
cost model, duplicate detection, shard arithmetic."""
import numpy as np
import pytest

from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.dist import shard_bounds
from ai_crypto_trader_b200.sweep import (_duplicate_classes, _f32_down, _f32_up, costs_from_packed, decode_population,
                                         evaluation_order, lane_cost, lane_costs, predicted_events)

ROWS = {p: i for i, p in enumerate(range(5, 31))}


def test_decode_population_matches_the_scalar_rules():
    pop = synth.random_population(300, seed=8)
    pop[0].update(rsi_oversold=30.1, rsi_overbought=69.9, take_profit=2.7312, stop_loss=0.5519)   # leverage floats
    pop[1].update(max_position_size=50)                                                             # capped at 20 % (:762)
    pop[2].pop("rsi_period")                                                                        # default 14
    rec = decode_population(pop, ROWS)
    for i, p in enumerate(pop):
        assert rec["rsi_row"][i] == ROWS[int(p.get("rsi_period", 14))]
        assert rec["rsi_lo"][i] == _f32_up(float(p["rsi_oversold"])) and rec["rsi_hi"][i] == _f32_down(float(p["rsi_overbought"]))
        # fp32 thresholds decide exactly like the float64 compares of the reference for every fp32 RSI value nearby
        for r in np.nextafter(np.float32(p["rsi_oversold"]), np.float32([-np.inf, np.inf])):
            assert (float(r) < float(p["rsi_oversold"])) == (r < rec["rsi_lo"][i])
        for r in np.nextafter(np.float32(p["rsi_overbought"]), np.float32([-np.inf, np.inf])):
            assert (float(r) > float(p["rsi_overbought"])) == (r > rec["rsi_hi"][i])
        assert rec["take_profit"][i] == p["take_profit"] / 100 and rec["stop_loss"][i] == p["stop_loss"] / 100
        assert rec["position_size"][i] == 10000 * (min(p.get("max_position_size", 5), 20) / 100)
    with pytest.raises(KeyError):
        decode_population([{"rsi_period": 99}], ROWS)
    assert decode_population([], ROWS).shape == (0,)


@pytest.mark.filterwarnings("ignore:invalid value encountered in cast")
def test_decode_population_refuses_any_period_outside_the_bank():
    """A period however large, or not a number, is a KeyError, found without a table as long as the period (1e9 would
    be an 8 GB one), next to valid individuals."""
    for period in (31, 1e9, 2.0 ** 62, 1e300, np.inf, -np.inf, np.nan, -1, 4):
        with pytest.raises(KeyError):
            decode_population([{"rsi_period": 14}, {"rsi_period": period}], ROWS)
    assert decode_population([{"rsi_period": 30.9}, {"rsi_period": 5}], ROWS)["rsi_row"].tolist() == [25, 0]


def test_cost_model_variants_agree():
    pop = synth.random_population(500, seed=3)
    scalar = np.array([lane_cost(p) for p in pop])
    assert np.allclose(lane_costs(pop), scalar, rtol=1e-12)
    rec = decode_population(pop, ROWS)
    assert np.allclose(costs_from_packed(rec, list(range(5, 31))), scalar, rtol=1e-6)     # thresholds are fp32 there
    assert np.allclose(predicted_events(pop, 1000), 0.27 * scalar * 1000)
    order = evaluation_order(pop)
    assert sorted(order.tolist()) == list(range(500))
    per = np.array([p["rsi_period"] for p in pop])[order]
    assert np.all(np.diff(per) >= 0)                      # same period adjacent
    assert 0 < scalar.min() and scalar.max() < 1


def test_duplicate_classes():
    pop = synth.random_population(64, seed=5)
    assert _duplicate_classes(decode_population(pop, ROWS)) is None
    twins = pop + [dict(pop[3]), dict(pop[7], macd_fast=9, ema_long=77), dict(pop[3], atr_period=9)]   # same 6 effective genes
    rec = decode_population(twins, ROWS)
    first, cls = _duplicate_classes(rec)
    assert len(first) == 64 and cls.shape == (67,)
    assert np.array_equal(rec[first][cls], rec)
    assert cls[64] == cls[3] and cls[66] == cls[3] and cls[65] == cls[7]


def test_shard_bounds_cover_the_range():
    for n in (0, 1, 7, 8, 1000):
        for world in (1, 2, 3, 8):
            spans = [shard_bounds(n, world, r) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            assert all(hi - lo <= per for lo, hi, per in spans)


@pytest.mark.parametrize("n,order_by", [(1024, "row_cost"), (333, "row_cost"), (31, "row_thresholds"), (1024, "row_thresholds"),
                                        (70, "identity")])
def test_pack_warps_seats_every_individual_once_and_keeps_two_rows_per_warp(n, order_by):
    """Thread slots of the thread-per-lane scan (sweep.pack_warps): whole warps, every individual seated exactly once, at
    most WARP_RSI_ROWS distinct bank rows per warp (the kernel flags a warp that breaks the rule; only the identity order
    may), the most expensive warps dispatched first."""
    from ai_crypto_trader_b200.sweep import WARP_RSI_ROWS, pack_warps
    pop = synth.random_population(n, seed=n)
    pred = predicted_events(pop, 1_000_000)
    slots = pack_warps(pop, pred, order_by)
    assert slots.dtype == np.int32 and slots.size % 32 == 0
    seated = slots[slots >= 0]
    assert sorted(seated.tolist()) == list(range(n))
    warps = slots.reshape(-1, 32)
    rows = np.array([int(p["rsi_period"]) for p in pop])
    if order_by != "identity":
        for w in warps:
            assert len(set(rows[w[w >= 0]].tolist())) <= WARP_RSI_ROWS
        cost = np.where(warps >= 0, pred[np.maximum(warps, 0)], 0.0).sum(axis=1)
        assert np.all(np.diff(cost) <= 1e-9)                  # dispatch order: most expensive first
        # packing is dense: empty seats only where a third row would have entered a warp
        assert warps.shape[0] <= -(-n // 32) + len(set(rows.tolist()))
    # an explicit row per individual (several timeframes) overrides the period
    rows2 = rows + 100 * (np.arange(n) % 3)
    s2 = pack_warps(pop, pred, "row_cost", rows=rows2).reshape(-1, 32)
    for w in s2:
        assert len(set(rows2[w[w >= 0]].tolist())) <= WARP_RSI_ROWS
    assert sorted(s2[s2 >= 0].tolist()) == list(range(n))
