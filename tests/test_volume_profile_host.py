"""Volume profile without a GPU: numpy's pairwise order, tests/volume_profile_ref.py against the reference's own
VolumeProfileAnalyzer (tests/golden/volume_profile_reference.json, tests/golden/make_volume_profile.py), and the host's
assembly of the reference's dicts, summary strings and the monitor's block from rows."""
import json
from pathlib import Path

import numpy as np
import pytest

import volume_profile_ref as ref

GOLDEN = Path(__file__).resolve().parent / "golden" / "volume_profile_reference.json"
FIXTURE = json.loads(GOLDEN.read_text())
CASES = FIXTURE["cases"]
IDS = [c["name"] for c in CASES]


def frame_of(case):
    import pandas as pd
    o, h, l, c, v = (np.asarray(x, dtype=np.float64) / FIXTURE["tick"] for x in case["bars"])
    ts = pd.date_range(case["start"], periods=len(c), freq="5min")
    return pd.DataFrame({"timestamp": ts, "open": o, "high": h, "low": l, "close": c, "volume": v})


def ref_frame(case):
    df = frame_of(case)
    return ref.frame(*(df[k].to_numpy() for k in ("open", "high", "low", "close", "volume")), num_bins=case["num_bins"])


def _strip(d):
    return {k: v for k, v in d.items() if k not in ("timestamp", "histogram_base64")}


def _call(fn, *args):
    try:
        return _strip(fn(*args))
    except Exception as e:                                     # the analyzer's error convention
        return {"error": str(e)}


def _close(got, want, rel):
    """Equal, or within `rel` for the anomaly pass's rolling mean / std values."""
    return got == want or abs(got - want) <= rel * abs(want)


def test_pairwise_sum_is_numpy_order():
    rng = np.random.default_rng(7)
    for n in list(range(0, 300)) + [1000, 1023, 1024, 1025, 4097]:
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 8, n)
        assert ref.pairwise_sum(x) == np.sum(x), n


def test_price_levels_are_linspace_formula():
    rng = np.random.default_rng(3)
    for _ in range(500):
        lo = float(np.float32(rng.uniform(1e-4, 1e5)))
        hi = float(np.float32(lo * rng.uniform(1.0001, 3)))
        B = int(rng.integers(1, 65))
        step = (hi - lo) / B
        edges = [i * step + lo for i in range(B)] + [hi]
        assert np.array_equal(ref.price_levels(lo, hi, B), [(edges[i] + edges[i + 1]) / 2 for i in range(B)])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_matches_reference(case):
    """Every field of the reference's dicts from the restatement's row, through the host's assembly."""
    from ai_crypto_trader_b200 import volume_profile as vp
    row, bins = ref_frame(case)
    df = frame_of(case)
    want = case["profile"]
    if "error" in want:
        assert not row["valid"] and want["error"] == vp._FLAT_FRAME_ERROR
    else:
        got = _call(vp.profile_result, row, bins)
        if case["tie_at_cut"]:                              # the platform's argsort decides the value area there
            for k in ("value_area_high", "value_area_low"):
                got.pop(k), want.pop(k)
            got["signals"].pop("value_area"), want["signals"].pop("value_area")
            got.pop("summary"), want.pop("summary")
            got["signals"].pop("overall"), want["signals"].pop("overall")
        assert got == want
    assert _call(vp.delta_result, row) == case["delta"]
    want = case["anomalies"]
    if "error" in want:
        assert not row["anomaly_status"] and want["error"] == f"Insufficient data for window size 20"
        return
    got = _call(vp.anomaly_result, row, df)
    assert got.keys() == want.keys()
    if got["anomalies_detected"]:
        assert got["total_anomalies"] == want["total_anomalies"]
        assert got["recent_anomaly_percentage"] == want["recent_anomaly_percentage"]
        assert got.get("message") == want.get("message")
        for a, b in zip(got["recent_anomalies"] + [got["strongest_anomaly"]],
                        want["recent_anomalies"] + [want["strongest_anomaly"]]):
            assert a.keys() == b.keys()
            for k in a:
                assert a[k] == b[k] or _close(a[k], b[k], 1e-12), (k, a[k], b[k])
        assert len(got["recent_anomalies"]) == len(want["recent_anomalies"])
    else:
        assert got == want


def test_fixture_covers_the_issue_cases():
    names = set(IDS)
    assert {f"walk_{W}_20" for W in (1, 5, 19, 20, 39, 40, 100, 300)} <= names
    assert {"flat", "one_candle_spans_all", "constant_volume", "sell_only", "zero_volume",
            "close_on_single_bin_midpoint"} <= names
    assert sum(c["tie_at_cut"] for c in CASES) >= 3
    mid = next(c for c in CASES if c["name"] == "close_on_single_bin_midpoint")
    assert mid["profile"]["signals"]["value_area"] == "inside_value_area_middle"
    assert mid["profile"]["value_area_low"] == mid["profile"]["value_area_high"]
    assert next(c for c in CASES if c["name"] == "sell_only")["delta"] == {"error": "float division by zero"}
    assert next(c for c in CASES if c["name"] == "zero_volume")["delta"]["buy_sell_ratio"] == float("inf")


def test_monitor_summary_keys():
    """The optional keys of the monitor's block (:492-512), from restatement rows."""
    from ai_crypto_trader_b200 import volume_profile as vp
    rows = {}
    for case in CASES:
        rows[case["name"]] = ref_frame(case)[0]
    table = np.stack([rows[k] for k in ("flat", "sell_only", "walk_300_20", "constant_volume")])[:, None]
    assert vp.monitor_summary(table, 0, 0) is None                                     # flat: no block
    sell = vp.monitor_summary(table, 1, 0)
    assert "volume_pressure" not in sell and "volume_divergence" not in sell             # the delta pass failed
    full = vp.monitor_summary(table, 2, 0)
    want = next(c for c in CASES if c["name"] == "walk_300_20")
    assert full["poc"] == want["profile"]["poc"] and full["summary"] == want["profile"]["summary"]
    assert full["signal"] == want["profile"]["signals"]["overall"]
    assert full["volume_pressure"] == want["delta"]["signals"]["overall_pressure"]
    assert ("volume_divergence" in full) == (want["delta"]["signals"]["divergence"] != "no_divergence")
    assert full["volume_anomalies"] is True
    assert full["recent_anomaly_percentage"] == want["anomalies"]["recent_anomaly_percentage"]
    quiet = vp.monitor_summary(table, 3, 0)
    assert "volume_anomalies" not in quiet and "recent_anomaly_percentage" not in quiet
    empty = ref.empty_row()
    assert vp.monitor_summary(np.array([[empty]]), 0, 0) is None                        # no frame


def test_base_labels_follow_completed_bars():
    """A 1-minute bar carries the label of the last 5-minute frame completed by its end."""
    frame = np.array([[0, 1, 2, 3]], dtype=np.uint8)
    got = ref.base_labels(frame, 28_401_120 + 3, 1, 18, 28_401_120, 5)
    assert got[0].tolist() == [255, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 2, 2, 2, 2, 2, 3, 3]


def test_dropin_window_below_two_and_errors():
    """The drop-in's answers that need no kernel: missing columns, short frames, windows below 2."""
    from ai_crypto_trader_b200 import volume_profile as vp
    df = frame_of(CASES[6])
    an = vp.VolumeProfileAnalyzer()
    assert an.analyze_volume_profile(df.drop(columns="high")) == {"error": "Missing required column: high"}
    assert an.analyze_volume_delta(df.drop(columns="open")) == {"error": "Missing required column: open"}
    assert an.detect_volume_anomalies(df.drop(columns="volume")) == {"error": "Missing required column: volume"}
    assert an.detect_volume_anomalies(df, window=len(df) + 1) == {
        "error": f"Insufficient data for window size {len(df) + 1}"}
    for w in (0, 1):
        got = an.detect_volume_anomalies(df, window=w)
        assert got["anomalies_detected"] is False and got["message"] == "No volume anomalies detected"
    assert an.detect_volume_anomalies(df, window=-1) == {"error": "window must be an integer 0 or greater"}
    assert an.analyze_volume_profile(df.iloc[:0]) == {"error": vp._EMPTY_FRAME_ERROR}
