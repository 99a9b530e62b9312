"""The multi-timeframe oracle `oracle/indicators_ref.rsi_rows_on_timeframe` against an independent pandas statement of the
same rule (CPU only).  It is what tests/test_gpu_timeframes.py and test_multi_timeframe_bank_and_sweep hold the device bank
(b200bt_resample -> b200bt_rsi_bank -> b200bt_align) to, so its bucket and "last completed bar" rules are pinned here by
other means than the floor-division formula it shares with align_kernel:

  buckets    pandas' Series.resample(f"{k}min", origin="epoch").last() on the bar START times.  The contract is epoch
             alignment: bucket b covers the minutes [b k, (b + 1) k) from 1970-01-01 00:00 UTC, not from the first day of
             the series (pandas' default origin="start_day"; the two differ for a k that does not divide 1440).
  completed  searchsorted(bucket_end, bar_start + bar_minutes, side="right") - 1: the last bucket that has ended by the
             time bar t has closed (NaN before the first one).

The grid covers the bar clocks 1 / 3 / 5 / 7 minutes, k = bar x {1, 2, 3, 12}, a daily bucket and a k that does not divide
1440, first bars on and off both grids, and series from one bar to a few thousand, including those ending one bar short of,
on, and one bar past a bucket boundary."""
import numpy as np
import pandas as pd
import pytest

from ai_crypto_trader_b200.synth import EPOCH_2024_MINUTES
from oracle import indicators_ref

PERIODS = (2, 5, 14)
DAY0 = EPOCH_2024_MINUTES                     # a UTC midnight: the offsets below are minutes into that day


def timeframes_of(bar):
    """k for a bar clock: bar x {1, 2, 3, 12}, the daily bucket (the multiple of bar nearest 1440 from above when bar does
    not divide it) and one more k that does not divide 1440."""
    daily = 1440 if 1440 % bar == 0 else -(-1440 // bar) * bar
    other = {1: 7, 3: 21, 5: 2880, 7: 7 * 300}[bar]
    return sorted({bar, 2 * bar, 3 * bar, 12 * bar, daily, other})


def grid_cases(long_n=3001):
    """(bar_minutes, k, minute0, n) of the grid above (shared with tests/test_gpu_timeframes.py)."""
    out = []
    for bar in (1, 3, 5, 7):
        for k in timeframes_of(bar):
            per = k // bar
            for off in sorted({0, 1, bar - 1, k - 1, 1439}):
                for n in sorted({1, per - 1, per, per + 1, 3 * per + 2, long_n} - {0}):
                    out.append((bar, k, DAY0 + off, n))
    return out


def close_series(n, seed):
    rng = np.random.default_rng(seed)
    return (100.0 * np.exp(np.cumsum(rng.normal(0.0, 0.002, n)))).astype(np.float32)


def pandas_rows(close32, minute0, k, periods, bar_minutes):
    """The independent statement: pandas resample on bar start times (origin="epoch"), RSI on that clock, and the last
    bucket that has ended when bar t closes."""
    n = len(close32)
    start = minute0 + np.arange(n, dtype=np.int64) * bar_minutes
    s = pd.Series(close32, index=pd.to_datetime(start * 60, unit="s"))
    r = s.resample(f"{k}min", origin="epoch").last()
    assert not r.isna().any()                            # k >= bar_minutes: no empty bucket between two bars
    rows = indicators_ref.rsi_bank(r.to_numpy(dtype=np.float32), periods)
    bucket_end = r.index.values.astype("datetime64[m]").astype(np.int64) + k
    j = np.searchsorted(bucket_end, start + bar_minutes, side="right") - 1
    out = rows[:, np.maximum(j, 0)]
    out[:, j < 0] = np.nan
    return out


def _identical(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_grid_covers_what_the_kernels_branch_on():
    cases = grid_cases()
    assert len(cases) > 500
    assert any(k % 1440 and 1440 % k for _, k, _, _ in cases)                       # k that does not divide 1440
    assert any((m0 - DAY0) % bar for bar, _, m0, _ in cases)                        # first bar off the bar grid
    assert any(k // bar > n for bar, k, _, n in cases)                              # series shorter than one bucket
    assert any(k == 1440 for _, k, _, _ in cases)


@pytest.mark.parametrize("bar", [1, 3, 5, 7])
def test_rsi_rows_on_timeframe_equal_pandas_epoch_resample(bar):
    """Bit for bit, NaN positions included, over the whole grid of this bar clock."""
    cases = [c for c in grid_cases() if c[0] == bar]
    base = close_series(max(n for *_, n in cases), seed=bar)
    for _, k, minute0, n in cases:
        close = base[:n]
        got = indicators_ref.rsi_rows_on_timeframe(close, minute0, k, PERIODS, bar_minutes=bar)
        want = pandas_rows(close, minute0, k, PERIODS, bar)
        assert got.shape == (len(PERIODS), n)
        assert _identical(got, want), (bar, k, minute0 - DAY0, n)


def test_buckets_are_aligned_to_the_epoch_not_to_the_first_day():
    """k = 7 from a midnight: the first bucket starts at the epoch-aligned minute floor(minute0 / 7) * 7, which is not the
    first bar; pandas' default origin (the first day's midnight) would close the first bucket on another bar."""
    bar, k, minute0, n = 1, 7, DAY0, 200
    assert minute0 % k != 0
    first_end = (minute0 // k + 1) * k                   # end of the bucket the first bar falls in
    t_close = first_end - minute0 - 1                    # the bar that completes it
    rows = indicators_ref.rsi_rows_on_timeframe(close_series(n, seed=11), minute0, k, PERIODS, bar_minutes=bar)
    assert np.isnan(rows[:, :t_close]).all() and not np.isnan(rows[:, t_close:]).any()
    assert t_close != k - 1                              # origin="start_day" would close it on bar k - 1
    s = pd.Series(np.zeros(n), index=pd.to_datetime((minute0 + np.arange(n)) * 60, unit="s"))
    assert s.resample("7min").last().index[0] != s.resample("7min", origin="epoch").last().index[0]


@pytest.mark.parametrize("bar,k", [(1, 5), (1, 1440), (3, 36), (5, 2880), (7, 14), (7, 2100)])
def test_no_look_ahead(bar, k):
    """Rows up to bar t do not depend on any close after t: replacing every later close leaves them bit-identical.

    This holds from the end of the warm-up on: the NaN policy of the reference's analyzer (ffill, then bfill) back-fills the
    first max(PERIODS) - 1 buckets of the derived clock with the first defined RSI, so a bar inside the warm-up shows a
    value of a later bucket, as the base-clock bank does on its own clock."""
    rng = np.random.default_rng(bar * 10_000 + k)
    per = k // bar
    minute0 = DAY0 + int(rng.integers(0, 1440))
    first = -((minute0 - (minute0 // k + 1) * k) // bar) - 1     # the bar that completes the first bucket
    warm = first + (max(PERIODS) - 1) * per                      # ... and the one completing the first defined bucket
    n = warm + 6 * per + 50
    close = close_series(n, seed=k)
    full = indicators_ref.rsi_rows_on_timeframe(close, minute0, k, PERIODS, bar_minutes=bar)
    for t in rng.integers(warm, n - 2 * per, size=8):           # (a whole bucket completes after t)
        other = close.copy()
        other[t + 1:] = (other[t + 1:] * rng.uniform(0.5, 2.0, n - t - 1)).astype(np.float32)
        cut = indicators_ref.rsi_rows_on_timeframe(other, minute0, k, PERIODS, bar_minutes=bar)
        assert _identical(cut[:, :t + 1], full[:, :t + 1]), (bar, k, int(t))
        assert not _identical(cut, full)                 # the change is visible once a later bucket completes
    other = close.copy()
    other[warm - 1:] *= np.float32(1.5)                          # inside the warm-up: the back-fill reads ahead
    cut = indicators_ref.rsi_rows_on_timeframe(other, minute0, k, PERIODS, bar_minutes=bar)
    assert not _identical(cut[-1, first:warm - 1], full[-1, first:warm - 1])


@pytest.mark.parametrize("bar,k,offset", [(1, 5, 1), (5, 60, 25), (7, 21, 3), (1, 1440, 600)])
def test_known_answers_head_and_unfinished_tail(bar, k, offset):
    """Everything before the first completed bucket is NaN, the bar that completes it shows it, and the bars of a bucket
    the series ends inside show the last completed bucket, whatever their closes."""
    minute0 = DAY0 + offset
    per = k // bar
    end0 = (minute0 // k + 1) * k                                # epoch minute at which the first bucket ends
    first = -((minute0 - end0) // bar) - 1                       # the bar that closes at or after it: ceil(...) - 1
    assert minute0 + first * bar < end0 <= minute0 + (first + 1) * bar
    n = first + 1 + 20 * per + per // 2 + 1                     # 20 whole buckets after it, then half a bucket
    close = close_series(n, seed=offset)
    close[n - (per // 2 + 1):] *= np.float32(3.0)                # a jump inside the unfinished bucket
    rows = indicators_ref.rsi_rows_on_timeframe(close, minute0, k, PERIODS, bar_minutes=bar)
    assert np.isnan(rows[:, :first]).all(), (bar, k, offset)
    assert not np.isnan(rows[:, first:]).any()
    # the 21 completed buckets end on bars first, first + per, ...; their closes are those bars' closes
    ends = first + per * np.arange(21)
    done = indicators_ref.rsi_bank(close[ends], PERIODS)
    assert (rows[:, ends[-1]:] == done[:, -1:]).all()            # the unfinished bucket never shows
    for i, e in enumerate(ends):
        assert (rows[:, e:e + per] == done[:, i:i + 1]).all(), (bar, k, offset, i)
