"""Volume profile on the GPU (csrc/volume_profile.cu):

* rows, bins and frame-clock labels of b200bt_volume_profile bit-equal to tests/volume_profile_ref.py on 1- and 5-minute
  markets resampled to 5- and 15-minute frames, for B in {1, 2, 20, 64} and W in {1, 20, 100, 1000};
* the VolumeProfileAnalyzer drop-in against the reference's own dicts (tests/golden/volume_profile_reference.json);
* base-clock labels (volume_profile_labels) against the restatement, with bars before the first frame and flat frames;
* PopulationSweep.class_stats with those labels against tests/regime_ref.py on the C oracle's records;
* the configs[1] market (10 symbols x 1M 1-minute bars, 5-minute frames): a seeded sample of frames bit-equal, and the
  profile's invariants on every frame."""
import numpy as np
import pytest

import volume_profile_ref as ref
from gpu_fixtures import torch_cuda
from test_gpu_regime import check_classes
from test_volume_profile_host import CASES, IDS, _close, frame_of

pytestmark = pytest.mark.gpu

MINUTE0 = 28_401_120


def _synth(torch, S, N, bar_minutes=1, seed=1234, minute0=MINUTE0):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    return MarketData(synth.synth_ohlcv(S, N, seed_base=seed), minute0=minute0, bar_minutes=bar_minutes)


def assert_rows_equal(got, want, where):
    """Every field bit for bit (NaN equals NaN)."""
    for name in got.dtype.names:
        g, w = got[name], want[name]
        if g.dtype.kind == "f":
            same = (g.view(np.uint64) == w.view(np.uint64)) | (np.isnan(g) & np.isnan(w))
        else:
            same = g == w
        assert same.all(), (where, name, np.argwhere(~same)[:3].tolist(), g[~same][:3], w[~same][:3])


def _run(torch, fm, W, B, rows=True, bins=True):
    from ai_crypto_trader_b200 import volume_profile as vp
    r, b, lab = vp._run(fm.ohlcv, vp.vp_params(W, B), rows, bins, fm.device)
    return vp.rows_table(r), b.cpu().numpy(), lab.cpu().numpy()


@pytest.mark.parametrize("bar_minutes, timeframe", [(1, 5), (1, 15), (5, 5), (5, 15)])
def test_rows_bins_labels_bit_equal(torch_cuda, bar_minutes, timeframe):
    from ai_crypto_trader_b200 import volume_profile as vp
    M = 1200
    market = _synth(torch_cuda, 2, M * timeframe // bar_minutes + 3, bar_minutes, minute0=MINUTE0 + 2 * bar_minutes)
    fm = vp._frame_market(market, timeframe)
    host = fm.ohlcv.cpu().numpy()
    rng = np.random.default_rng(bar_minutes * 100 + timeframe)
    for W in (1, 20, 100, 1000):
        for B in (1, 2, 20, 64):
            rows, bins, labels = _run(torch_cuda, fm, W, B)
            pick = [(s, int(t)) for s in range(fm.S) for t in rng.choice(fm.N, 12 if W == 1000 else 24, replace=False)]
            pick += [(0, W - 2), (0, W - 1), (1, fm.N - 1)]
            pick = [(s, t) for s, t in pick if 0 <= t < fm.N]
            wr, wb, wl = ref.frames_at(host, pick, W, B)
            s_idx, t_idx = np.array(pick).T
            where = f"{bar_minutes}m bars, {timeframe}m frames, W={W}, B={B}"
            assert_rows_equal(rows[s_idx, t_idx], wr, where)
            assert np.array_equal(bins[s_idx, t_idx], wb), where
            assert np.array_equal(labels[s_idx, t_idx], wl), where
            assert (labels[:, :W - 1] == 255).all() and (rows["n_bars"][:, :W - 1] == 0).all(), where
            assert (labels[:, W - 1:] < 6).all(), where                 # synthetic bars are never flat


def test_history_api_and_history_rows(torch_cuda):
    """volume_profile_history: the resampled clock, rows on request, labels-only runs giving the same labels."""
    from ai_crypto_trader_b200 import indicators as ind
    from ai_crypto_trader_b200 import volume_profile as vp
    market = _synth(torch_cuda, 3, 3000)
    h = vp.volume_profile_history(market)
    assert h.market.bar_minutes == 5 and h.market.N == ind.resample(market, 5).N
    table = h.table()
    assert table.shape == (3, h.market.N)
    lab_only = vp.volume_profile_history(market, rows=False)
    assert lab_only.rows is None and torch_cuda.equal(lab_only.labels, h.labels)
    assert np.array_equal(table["signal"], h.labels.cpu().numpy().astype(np.int32))
    with pytest.raises(ValueError):
        vp.volume_profile_history(_synth(torch_cuda, 1, 100, bar_minutes=5), timeframe_minutes=7)
    summary = vp.monitor_summary(table, 1, h.market.N - 1)
    assert summary["signal"] == vp.SIGNALS[table["signal"][1, -1]] and summary["poc"] == table["poc"][1, -1]
    assert vp.monitor_summary(table, 0, 50) is None


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_dropin_matches_reference(torch_cuda, case):
    from ai_crypto_trader_b200 import volume_profile as vp
    an = vp.VolumeProfileAnalyzer(num_bins=case["num_bins"])
    strip = lambda d: {k: v for k, v in d.items() if k not in ("timestamp", "histogram_base64")}
    got, want = strip(an.analyze_volume_profile(frame_of(case))), dict(case["profile"])
    if case["tie_at_cut"]:
        for k in ("value_area_high", "value_area_low", "summary"):
            got.pop(k), want.pop(k)
        got["signals"] = {k: v for k, v in got["signals"].items() if k not in ("value_area", "overall")}
        want["signals"] = {k: v for k, v in want["signals"].items() if k not in ("value_area", "overall")}
    assert got == want
    assert strip(an.analyze_volume_delta(frame_of(case))) == case["delta"]
    got, want = strip(an.detect_volume_anomalies(frame_of(case))), case["anomalies"]
    assert got.keys() == want.keys()
    if got.get("anomalies_detected"):
        for k in ("total_anomalies", "recent_anomaly_percentage"):
            assert got[k] == want[k]
        for a, b in zip(got["recent_anomalies"] + [got["strongest_anomaly"]],
                        want["recent_anomalies"] + [want["strongest_anomaly"]]):
            assert a.keys() == b.keys() and all(a[k] == b[k] or _close(a[k], b[k], 1e-12) for k in a), (a, b)
        assert len(got["recent_anomalies"]) == len(want["recent_anomalies"])
    else:
        assert got == want
    # the module-level functions are the same analysis
    assert strip(vp.analyze_volume_delta(frame_of(case))) == case["delta"]


def test_dropin_without_timestamps_fails_as_the_reference(torch_cuda):
    from ai_crypto_trader_b200 import volume_profile as vp
    case = next(c for c in CASES if c["name"] == "walk_300_20")
    got = vp.detect_volume_anomalies(frame_of(case).drop(columns="timestamp"))
    assert set(got) == {"error"} and "timestamp" in got["error"]


def _flat_market(torch, S=2, N=4000, bar_minutes=1):
    """Synthetic bars with a flat stretch (every price equal) on symbol 1, long enough for flat 5-minute frames."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    x = synth.synth_ohlcv(S, N)
    x[:4, 1, 1500:2300] = x[3, 1, 1500]
    return MarketData(x, minute0=MINUTE0 + 3, bar_minutes=bar_minutes), x


def test_base_clock_labels(torch_cuda):
    from ai_crypto_trader_b200 import volume_profile as vp
    market, _ = _flat_market(torch_cuda)
    W = 100
    labels = vp.volume_profile_labels(market, 5, W).cpu().numpy()
    fm = vp._frame_market(market, 5)
    _, _, frame_labels = ref.history(fm.ohlcv.cpu().numpy(), W)
    want = ref.base_labels(frame_labels, market.minute0, market.bar_minutes, market.N, fm.minute0, 5)
    assert np.array_equal(labels, want)
    assert (labels[:, :W * 5 - 4] == 255).all() and (labels[0, W * 5 - 4] < 6)   # before the first full frame
    assert (frame_labels[1] == 255).sum() > W - 1 and (labels[1, 2005:2295] == 255).all()   # flat frames
    assert set(np.unique(labels[0, W * 5:])) <= set(range(6))


def test_class_stats_by_zone(torch_cuda):
    """class_stats with the zone labels (6 classes; 255 belongs to none) equals the oracle's records split by label."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200 import volume_profile as vp
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    market, x = _flat_market(torch_cuda, S=2, N=20_000)
    periods = (5, 9, 14, 21)
    sweep = PopulationSweep(market, rsi_periods=periods, mode="fused")
    bank_h = sweep.bank.cpu().numpy()
    pop = synth.random_population(12, seed=4)
    for p in pop:
        p["rsi_period"] = periods[int(p["rsi_period"]) % len(periods)]
    labels = vp.volume_profile_labels(market)
    _, views = sweep.class_stats(pop, labels, 6)
    lab = labels.cpu().numpy()
    cfg = sim_oracle.config_of(market.minute0, 1)
    _, evs, pns = sim_oracle.population(x[3], bank_h, sweep.period_row, pop, cfg, event_cap=market.N + 2)
    check_classes(views, evs, pns, lab, 6, cfg, "labels")
    n_records = sum(int(v["n_records"].sum()) for v in views)
    assert n_records > 100


def test_configs1_history(torch_cuda):
    """10 symbols x 1M 1-minute bars, 100-bar 5-minute frames: a seeded sample of 2 400 frames bit-equal, and on every
    frame min <= VAL <= VAH <= max (the POC may fall outside the value area when the largest bin is tied)."""
    from ai_crypto_trader_b200 import volume_profile as vp
    market = _synth(torch_cuda, 10, 1_000_000)
    h = vp.volume_profile_history(market)
    table = h.table()
    host = h.market.ohlcv.cpu().numpy()
    rng = np.random.default_rng(99)
    pick = [(int(s), int(t)) for s, t in zip(rng.integers(0, 10, 2400), rng.integers(99, h.market.N, 2400))]
    want, _, wl = ref.frames_at(host, pick, 100)
    s_idx, t_idx = np.array(pick).T
    assert_rows_equal(table[s_idx, t_idx], want, "configs[1]")
    assert np.array_equal(h.labels.cpu().numpy()[s_idx, t_idx], wl)
    f = table[:, 99:]
    ok = f["valid"] == 1
    assert ok.mean() > 0.99
    assert (f["price_min"][ok] <= f["value_area_low"][ok]).all() and (f["value_area_low"][ok] <= f["value_area_high"][ok]).all()
    assert (f["value_area_high"][ok] <= f["price_max"][ok]).all()
    assert (f["value_area_low_bin"][ok] <= f["value_area_high_bin"][ok]).all()
    assert (f["total_anomalies"] <= 100 - 19).all() and (f["anomaly_status"] == 1).all()
