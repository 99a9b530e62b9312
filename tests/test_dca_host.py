"""The DCA restatements (tests/dca_ref.py) against the reference's own run (tests/golden/dca_reference.json), and the host
decoding of ai_crypto_trader_b200/dca.py: precision, interval tables, order sizes, genes.  No GPU needed."""
import json
import math
import random
from datetime import timedelta
from pathlib import Path

import numpy as np
import pytest

import dca_ref

GOLDEN = Path(__file__).resolve().parent / "golden" / "dca_reference.json"
POSITION_FIELDS = ("total_invested", "total_quantity", "average_price", "last_purchase_price", "current_value",
                   "profit_loss", "profit_loss_pct", "last_purchase_tick")


def load_cases():
    fx = json.loads(GOLDEN.read_text())
    out = []
    for case in fx["cases"]:
        c = dict(case)
        ticks = [np.cumsum(fx["series"][n]["close"]) for n in case["bars"]]          # 1/16 price ticks
        c["closes"] = np.array([t / 16 for t in ticks], dtype=np.float32).astype(np.float64)
        c["highs"] = np.array([(t + fx["series"][n]["high"]) / 16 for t, n in zip(ticks, case["bars"])],
                              dtype=np.float32).astype(np.float64)
        if case["labels"]:
            runs = fx["label_runs"][case["labels"]]
            c["labels"] = np.array([[v for v, n in runs for _ in range(n)]], dtype=np.uint8)
        out.append(c)
    return out


CASES = load_cases()


def precision_of(case):
    from ai_crypto_trader_b200.dca import quantity_precision
    return [quantity_precision(st) for st in (case["steps"] or [None] * len(case["symbols"]))]


def run_both(case):
    from ai_crypto_trader_b200 import dca
    svc = dca.Service(case["config"], case["symbols"])
    dip = np.stack([dca_ref.dip_series(case["highs"][s], case["closes"][s], case["minute0"], case["bar_minutes"])
                    for s in range(len(case["symbols"]))])
    prec = precision_of(case)
    ticks = dca_ref.simulate_ticks(case["closes"], case["highs"], case["minute0"], case["bar_minutes"], case["start_bar"],
                                   svc, labels=case["labels"], precision=prec, usdc_balance=case["usdc"], dip=dip)
    dec = dca.decode_individual({}, case["config"], case["symbols"], case["bar_minutes"])
    events = dca_ref.simulate(case["closes"], dip, case["minute0"], case["bar_minutes"], case["start_bar"], dec,
                              labels=case["labels"], precision=prec, usdc_balance=case["usdc"])
    return ticks, events


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_restatements_equal_the_reference_run(case):
    ticks, events = run_both(case)
    for form in (ticks, events):
        for s, sym in enumerate(case["symbols"]):
            want = case["positions"][sym]
            got = form["stats"][s]
            assert [list(p) for p in form["purchases"][s]] == want["purchases"], (case["name"], sym)
            for f in POSITION_FIELDS:
                assert got[f] == want[f], (case["name"], sym, f, got[f], want[f])
            assert got["next_scheduled_us"] == case["next_scheduled_us"][sym]
            assert got["last_dip_tick"] == case["last_dip_tick"][sym]
        assert form["service"] == case["service"], case["name"]
    assert ticks["order_total"] == case["service_total_invested"]
    for s in range(len(case["symbols"])):
        for f, v in ticks["stats"][s].items():
            assert events["stats"][s][f] == v, (case["name"], s, f)
    assert ticks["day"] == events["day"]


def test_fixture_covers_the_cases():
    kinds = {}
    for case in CASES:
        for p in case["positions"].values():
            for q in p["purchases"]:
                kinds[q[1]] = kinds.get(q[1], 0) + 1
    assert set(kinds) == {"scheduled", "dip", "rebalance"}
    assert any(q[3] == 0.0 for c in CASES for p in c["positions"].values() for q in p["purchases"])   # precision 0
    assert {1, 5} <= {c["bar_minutes"] for c in CASES}
    # a drop landing exactly on the threshold: 1024 -> 960 is 6.25 %
    assert any(q[1] == "dip" and q[2] == 960.0 for c in CASES if c["name"].startswith("dips")
               for p in c["positions"].values() for q in p["purchases"])


def test_dip_series_against_the_literal_klines():
    rng = np.random.default_rng(3)
    for bm, m0 in ((1, 28_401_120), (5, 28_401_120 + 7), (1440, 28_401_120), (60, 28_401_120 + 1439)):
        N = max(40, 12 * 1440 // bm)
        close = np.round(1000 * np.exp(np.cumsum(0.01 * rng.standard_normal(N))) * 16) / 16
        high = close + np.round(rng.random(N) * 64) / 16
        high[::97] = 0.0
        close[::97] = 0.0
        got = dca_ref.dip_series(high, close, m0, bm)
        for b in list(range(min(N, 300))) + list(rng.integers(0, N, 300)):
            want = dca_ref.dip_of(dca_ref.klines_high(high, m0, bm, int(b)), float(close[b]))
            assert (math.isnan(want) and math.isnan(got[b])) or got[b] == want, (bm, b)


def test_quantity_precision():
    from ai_crypto_trader_b200.dca import quantity_precision
    assert quantity_precision(None) == 6
    assert quantity_precision("0.00001000") == 0            # str(1e-05) is scientific
    assert quantity_precision("0.00010000") == 4
    assert quantity_precision("0.00100000") == 3
    assert quantity_precision("1.00000000") == 0
    assert quantity_precision(0.1) == 1


def test_interval_tables_against_timedelta():
    from ai_crypto_trader_b200 import dca
    block = {"adaptive_scheduling": True, "interval_hours": 7.3,
             "scheduling_strategies": {"market_regime_based": {"bull_interval_hours": 48, "bear_interval_hours": 12.5,
                                                               "crab_interval_hours": 1, "volatile_interval_hours": 6},
                                       "weighted_scheduling": {"enabled": True, "weight_factors": {"day_of_week": 0.37}}},
             "symbol_settings": [{"symbol": "B", "interval_hours": 30, "allocation": 0.7, "base_order_size_usdc": 40}]}
    d = dca.decode_individual({}, block, ["A", "B"], 1)
    iv = d["individual"]
    for lab, h in enumerate((48, 12.5, 7.3, 6, 7.3)):
        for wk in (0, 1):
            f = 1.0 + 0.2 * 0.37 * wk
            want = timedelta(hours=max(h * 0.5, min(h * 1.5, h * f))) // timedelta(microseconds=1)
            assert iv.later_us[0][lab][wk] == want and d["first_us"][0, lab, wk] == want
    assert d["first_us"][1, 2, 0] == 30 * 3_600_000_000 and iv.later_us[1][2][0] == 30 * 3_600_000_000
    assert iv.later_us[0][2][1] % 60_000_000 != 0                               # a sub-minute remainder
    assert list(d["target"]) == [0.5, 0.7]
    assert iv.order[0][0][0] == 100 and iv.order[1][0][0] == 40 and iv.order[1][1][0] == 60.0
    off = dca.decode_individual({"adaptive_scheduling": 0}, block, ["A", "B"], 1)["individual"]
    assert all(off.later_us[0][lab][wk] == 7.3 * 3_600_000_000 for lab in range(5) for wk in range(2))


def test_gene_decoding():
    from ai_crypto_trader_b200 import dca, _lib
    ranges = dca.dca_param_ranges()
    assert set(ranges) == {"interval_hours", "base_order_size_usdc", "price_dip_detection", "dip_threshold_pct",
                           "additional_dip_allocation", "max_dip_frequency_days", "adaptive_scheduling",
                           "bull_interval_hours", "bear_interval_hours", "volatile_interval_hours", "day_of_week_weight",
                           "increase_in_bear_market", "bear_market_adjustment", "periodic_rebalancing",
                           "rebalance_interval_days", "max_deviation_pct"}
    assert ranges["max_dip_frequency_days"] == (1, 30) and isinstance(ranges["rebalance_interval_days"][0], int)
    rng = random.Random(4)
    for _ in range(20):
        g = {k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi)) for k, (lo, hi) in ranges.items()}
        d = dca.decode_individual(g, {}, ["A", "B", "C"], 5)
        iv = d["individual"]
        assert iv.dip_cooldown_minutes == g["max_dip_frequency_days"] * 1440
        assert iv.rebalance_period == -(-g["rebalance_interval_days"] * 1440 // 5)
        assert iv.flags == (g["price_dip_detection"] and _lib.DCA_DIP) | (g["periodic_rebalancing"] and _lib.DCA_REBALANCE)
        assert iv.dip_threshold_pct == g["dip_threshold_pct"] and iv.max_deviation_pct == g["max_deviation_pct"]
        bear = g["increase_in_bear_market"]
        base = g["base_order_size_usdc"]
        dipped = base * (1.0 + g["additional_dip_allocation"]) if g["price_dip_detection"] else base
        want = max(20, min(500, dipped * (g["bear_market_adjustment"] if bear else 1)))
        assert iv.order[0][1][1] == want
        assert iv.order[0][0][0] == max(20, min(500, base))
    # missing keys: the config block, then the __init__ defaults
    d = dca.decode_individual({}, {"dip_threshold_pct": 3.5}, ["A"], 1)["individual"]
    assert d.dip_threshold_pct == 3.5 and d.dip_cooldown_minutes == 7 * 1440 and d.rebalance_period == 30 * 1440
    assert dca.rebalance_period(0, 1) == 1 and dca.rebalance_period(-3, 5) == 1 and dca.rebalance_period(1, 7) == 206
    with pytest.raises(ValueError):
        dca.rebalance_period(1.5, 1)
    with pytest.raises(ValueError):
        dca.decode_individual({"interval_hours": -1.0}, {}, ["A"], 1)
