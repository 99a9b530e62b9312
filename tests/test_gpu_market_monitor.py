"""GPU checks of b200bt_market_monitor / b200bt_indicator_combinations (csrc/market_monitor.cu) and the market_monitor
module:
* rows bit-equal to tests/market_monitor_ref.py on sampled bars of small markets, for W in {1, 13, 14, 15, 26, 27, 50,
  100}, on and off the 15-minute grid, with partial last buckets (avg_volume to rel 1e-12);
* the combination halves bit-equal to the restatement applied to the kernel's own snapshot halves;
* b200bt_indicator_combinations and the drop-in against the reference's outputs (tests/golden), None entries and the
  error dict included;
* labels equal to the selected field of the rows, the label-only path giving the same labels;
* PopulationSweep.class_stats with trend labels against tests/regime_ref.py on the C oracle's records;
* the configs[1] market (10 symbols x 1M 1-minute bars, W = 100): a seeded sample of 2 000 rows bit-equal, and on every
  row codes in range and validity from the first full frames onwards."""
import math

import numpy as np
import pytest

import market_monitor_ref as ref
from gpu_fixtures import torch_cuda
from test_gpu_regime import check_classes
from test_market_monitor_host import DICTS, FIXTURE, _equal, _leaves

pytestmark = pytest.mark.gpu

MINUTE0 = 28_401_120


def _synth(S, N, minute0=MINUTE0, seed=1234):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    return MarketData(synth.synth_ohlcv(S, N, seed_base=seed), minute0=minute0, bar_minutes=1)


def _bits_equal(g, w):
    g, w = float(g), float(w)
    return (math.isnan(g) and math.isnan(w)) or np.float64(g).view(np.uint64) == np.float64(w).view(np.uint64)


def _as_dict(row):
    """A row's snapshot half as the market_update dict the combinations read."""
    from ai_crypto_trader_b200 import _lib
    d = {k: float(row[k]) for k in _lib.MM_SNAPSHOT_FIELDS}
    d["trend"] = _lib.MM_TRENDS[int(row["trend"])]
    for k, bit in _lib.MM_HAS.items():
        if not int(row["present"]) & bit:
            d.pop(k, None)
        elif k in _lib.MM_OPTIONAL_FIELDS:
            d[k] = float(row[k])
    return d


def check_combination_half(row, where):
    from ai_crypto_trader_b200 import market_monitor as mm
    got, want = mm.combined_dict(row), ref.combinations(_as_dict(row))
    assert _equal(_leaves(got), _leaves(want)), (where, got, want)


def check_row(row, host, minute0, s, t, W, where):
    from ai_crypto_trader_b200 import _lib
    want = ref.row_at(host, minute0, s, t, W)
    assert int(row["valid"]) == want["valid"], (where, s, t)
    if not want["valid"]:
        assert all(math.isnan(float(row[k])) for k in _lib.MM_SNAPSHOT_FIELDS + _lib.MM_COMBINED_FIELDS), (where, t)
        assert int(row["trend"]) == 255 and int(row["computed"]) == 0, (where, t)
        return
    for k in _lib.MM_SNAPSHOT_FIELDS:
        if k == "avg_volume":
            assert float(row[k]) == pytest.approx(want[k], rel=1e-12), (where, s, t, k)
        else:
            assert _bits_equal(row[k], want[k]), (where, s, t, k, float(row[k]), want[k])
    assert _lib.MM_TRENDS[int(row["trend"])] == want["trend"], (where, s, t)
    assert int(row["present"]) == want["present"] and int(row["opportunity"]) == want["opportunity"], (where, s, t)
    check_combination_half(row, f"{where} s={s} t={t}")


def _first_valid(minute0, W, N):
    from market_monitor_ref import completed_kline
    return next((t for t in range(N) if t - W + 1 >= 0 and completed_kline(t, minute0, 3) - W + 1 >= 0 and
                 completed_kline(t, minute0, 5) - W + 1 >= 0 and completed_kline(t, minute0, 15) >= 0), N)


@pytest.mark.parametrize("W", [1, 13, 14, 15, 26, 27, 50, 100])
@pytest.mark.parametrize("offset", [0, 7])
def test_rows_bit_equal_to_restatement(torch_cuda, W, offset):
    from ai_crypto_trader_b200 import market_monitor as mm
    minute0 = MINUTE0 + offset
    N = 5 * W + 400 + 11                     # 11: the last 3-, 5- and 15-minute buckets are partial
    market = _synth(2, N, minute0, seed=W + offset)
    table = mm.market_update_history(market, W).table()
    host = market.ohlcv.cpu().numpy()
    first = _first_valid(minute0, W, N)
    rng = np.random.default_rng(W * 10 + offset)
    picks = sorted({first - 1, first, first + 1, N - 2, N - 1, *rng.integers(first, N, 16).tolist()} - {-1})
    for s in range(2):
        for t in picks:
            check_row(table[s, t], host, minute0, s, t, W, f"W={W} minute0+{offset}")
    assert (table["valid"][:, :first] == 0).all() and (table["valid"][:, first:] == 1).all()


def test_combinations_kernel_and_dropin_match_the_reference(torch_cuda):
    from ai_crypto_trader_b200 import market_monitor as mm
    for d, want in zip(DICTS, FIXTURE["combined"]):
        got = mm.calculate_indicator_combinations(dict(d))
        assert _equal(_leaves(got), want), (d, _leaves(got), want)
    # one batched kernel call over every dict with its required fields gives the same halves
    ok = [d for d, w in zip(DICTS, FIXTURE["combined"]) if isinstance(w, list)]
    rows = mm.combine_rows(np.stack([mm.snapshot_row(d) for d in ok]))
    for d, row in zip(ok, rows):
        assert _equal(_leaves(mm.combined_dict(row)), _leaves(ref.combinations(dict(d)))), d


def test_labels_equal_the_rows(torch_cuda):
    from ai_crypto_trader_b200 import _lib, market_monitor as mm
    market = _synth(3, 4000, MINUTE0 + 4, seed=8)
    table = mm.market_update_history(market, 100).table()
    for f, (name, names) in enumerate(_lib.MM_LABEL_FIELDS):
        labels, got_names = mm.monitor_labels(market, name, 100)
        assert got_names == names
        col = table["trend"] if f == 0 else table[_lib.MM_CODE_FIELDS[f - 1]]
        want = np.where(table["valid"] == 1, col, 255).astype(np.uint8)
        assert np.array_equal(labels.cpu().numpy(), want), name
        assert (labels.cpu().numpy()[table["valid"] == 1] < len(names)).all(), name
    # rows and labels from one launch
    rows, labels = mm._run(market, mm.monitor_params(100, 6), True, True)
    t2 = mm.rows_table(rows)
    assert np.array_equal(labels.cpu().numpy(), np.where(t2["valid"] == 1, t2["regime"], 255).astype(np.uint8))
    h = mm.market_update_history(market, 100, rows=False)
    assert h.rows is None and np.array_equal(h.labels.cpu().numpy(), np.where(table["valid"] == 1, table["trend"], 255))


def test_market_update_dicts(torch_cuda):
    from ai_crypto_trader_b200 import market_monitor as mm
    from ai_crypto_trader_b200 import volume_profile as vp
    market = _synth(2, 3000, MINUTE0 + 2, seed=5)
    h = mm.market_update_history(market, 100, config={"trading_params": {"min_volume_usdc": 0}})
    table = h.table()
    vph = vp.volume_profile_history(market)
    up = mm.market_update(h, 1, 2999, volume_profile=vph)
    assert up["symbol"] == market.symbols[1] and up["current_price"] == float(table["current_price"][1, 2999])
    assert up["combined_indicators"] == mm.combined_dict(table[1, 2999])
    j = ref.completed_kline(2999, market.minute0, 5)
    assert up["volume_profile"] == vp.monitor_summary(vph.table(), 1, j)
    assert mm.market_update(h, 0, 10) is None
    assert (table["opportunity"][table["valid"] == 1] ==
            (np.abs(table["price_change_1m"]) >= 0.5)[table["valid"] == 1]).all()


def test_class_stats_by_trend(torch_cuda):
    """class_stats with the trend labels (3 classes; 255 belongs to none) equals the oracle's records split by label."""
    from ai_crypto_trader_b200 import market_monitor as mm
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    x = synth.synth_ohlcv(2, 20_000)
    market = MarketData(x, minute0=MINUTE0 + 3, bar_minutes=1)
    periods = (5, 9, 14, 21)
    sweep = PopulationSweep(market, rsi_periods=periods, mode="fused")
    bank_h = sweep.bank.cpu().numpy()
    pop = synth.random_population(12, seed=4)
    for p in pop:
        p["rsi_period"] = periods[int(p["rsi_period"]) % len(periods)]
    labels, names = mm.monitor_labels(market, "trend")
    _, views = sweep.class_stats(pop, labels, len(names))
    lab = labels.cpu().numpy()
    cfg = sim_oracle.config_of(market.minute0, 1)
    _, evs, pns = sim_oracle.population(x[3], bank_h, sweep.period_row, pop, cfg, event_cap=market.N + 2)
    check_classes(views, evs, pns, lab, len(names), cfg, "labels")
    n_records = sum(int(v["n_records"].sum()) for v in views)
    assert n_records > 100


def test_configs1_history(torch_cuda):
    from ai_crypto_trader_b200 import _lib, market_monitor as mm
    market = _synth(10, 1_000_000)
    h = mm.market_update_history(market, 100)
    table = h.table()
    host = market.ohlcv.cpu().numpy()
    first = _first_valid(MINUTE0, 100, market.N)
    assert (table["valid"][:, :first] == 0).all() and (table["valid"][:, first:] == 1).all()
    rng = np.random.default_rng(2024)
    for s, t in zip(rng.integers(0, 10, 2000).tolist(), rng.integers(first - 2, market.N, 2000).tolist()):
        check_row(table[s, t], host, MINUTE0, s, t, 100, "configs[1]")
    v = table[:, first:]
    assert (v["trend"] < 3).all() and (v["computed"] == (1 << 15) - 1).all()
    for f, names in zip(_lib.MM_CODE_FIELDS, [n for _, n in _lib.MM_LABEL_FIELDS[1:]]):
        assert (v[f] < len(names)).all(), f
    assert (v["reversal_signals"] < 256).all() and np.isin(v["breakout_direction"], (-1, 0, 1)).all()
