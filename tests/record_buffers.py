"""Synthetic event buffers for the passes that read a sweep's trade records (b200bt_book_metrics, b200bt_daily_pnl,
b200bt_class_stats, b200bt_trade_pnl; csrc/sweep_dev.cuh read_lane / record_batch), a float64 host pricer of their
records, and the existing references fed with them.

A buffer is built directly, not swept, so that its records can sit exactly on the seams of the readers (32-record
batches, book windows, class stagings, calendar days).  It keeps the invariants the readers assume (include/b200bt.h):

* a lane's records alternate entry, exit, entry, exit: an even count, entries at even indices; an exit's SELL bit is the
  opposite of its entry's (a long trip is entered with 0 and closed with SELL, a short one entered with SELL);
* bars are below N and strictly increasing within a lane, except that the last bar N - 1 may hold an entry followed by
  its force-close;
* lane_stats[i][s].n_records is the only field the readers take from the stats (every other field is NaN here);
  n_records > event_cap marks a lane whose records the buffer lost;
* the slots of a lane from n_records up to event_cap hold POISON, a long exit on bar 0: a reader that went past
  n_records would price and count it.  Padding of the price rows (ld_price > N) holds finite junk for the same reason.
"""
from __future__ import annotations

import numpy as np

import book_ref
import cscv_ref
import regime_ref
import trade_mc_ref

BAR_MASK = 0x3FFFFFFF
EXIT = 0x40000000
SELL = 0x80000000
POISON = EXIT | SELL              # a long trip's exit on bar 0
PAD_PRICE = 3.0e4                 # finite junk in the padding of the price rows
STATS_WORDS = 20                  # b200bt_lane_stats: 20 x 8 bytes
INDIV_DTYPE = np.dtype([("rsi_row", "<i4"), ("rsi_lo", "<f4"), ("rsi_hi", "<f4"), ("reserved", "<i4"),
                        ("take_profit", "<f8"), ("stop_loss", "<f8"), ("position_size", "<f8")])


# ---- lanes ---------------------------------------------------------------------------------------------------------
def lane_words(bars, shorts=None) -> np.ndarray:
    """uint32 event words of the trips whose entry / exit bars are bars[2k], bars[2k + 1]; shorts[k]: trip k is short."""
    bars = np.asarray(bars, dtype=np.int64)
    assert len(bars) % 2 == 0
    shorts = np.zeros(len(bars) // 2, dtype=bool) if shorts is None else np.asarray(shorts, dtype=bool)
    w = bars.astype(np.uint64)
    w[0::2] |= np.where(shorts, SELL, 0).astype(np.uint64)
    w[1::2] |= EXIT | np.where(shorts, 0, SELL).astype(np.uint64)
    return w.astype(np.uint32)


def random_bars(rng, n: int, N: int, lo: int = 0, hi: int | None = None, last_pair: bool = False) -> np.ndarray:
    """n sorted distinct bars drawn from [lo, hi) (hi <= N - 1 when last_pair); with last_pair the last two records are the
    entry and force-close on bar N - 1."""
    hi = (N - 1 if last_pair else N) if hi is None else hi
    k = n - 2 if last_pair else n
    assert 0 <= k <= hi - lo and n % 2 == 0
    bars = np.sort(rng.choice(np.arange(lo, hi), size=k, replace=False))
    if last_pair:
        assert hi <= N - 1
        bars = np.concatenate([bars, [N - 1, N - 1]])
    return bars.astype(np.int64)


def random_lane(rng, n: int, N: int, **kw) -> np.ndarray:
    """Event words of n records on random distinct bars (random_bars), each trip long or short at random."""
    return lane_words(random_bars(rng, n, N, **kw), rng.random(n // 2) < 0.5)


def check_lane(words, N: int, complete: bool = True) -> None:
    """Raise ValueError unless `words` keep the readers' invariants on a series of N bars.  complete=False checks the
    prefix a lost lane leaves in the buffer (its count may be odd)."""
    w = np.asarray(words, dtype=np.uint32).astype(np.int64)
    n = len(w)
    if complete and n % 2:
        raise ValueError(f"odd record count {n}")
    bars, exit_, sell = w & BAR_MASK, (w & EXIT) != 0, (w & SELL) != 0
    if np.any(exit_[0::2]):
        raise ValueError(f"an exit at an entry index: {np.nonzero(exit_[0::2])[0][:4] * 2}")
    if not np.all(exit_[1::2]):
        raise ValueError(f"an entry at an exit index: {np.nonzero(~exit_[1::2])[0][:4] * 2 + 1}")
    m = n // 2
    if np.any(sell[0:2 * m:2] == sell[1:2 * m:2]):
        raise ValueError("an exit on the same side as its entry")
    if n and (bars.max() >= N):
        raise ValueError(f"bar {int(bars.max())} not below N = {N}")
    step = np.diff(bars)
    same = np.nonzero(step == 0)[0]
    if np.any(step < 0):
        raise ValueError(f"bars go back at record {int(np.nonzero(step < 0)[0][0]) + 1}")
    for j in same.tolist():      # two records on one bar: only the last bar's entry and its force-close
        if not (bars[j] == N - 1 and j % 2 == 0 and j + 2 == n):
            raise ValueError(f"records {j} and {j + 1} share bar {int(bars[j])}")


def check_buffer(events, n_records, N: int) -> None:
    """check_lane on every lane of events [pop][S][cap] with lane_stats n_records [pop][S], and POISON past each lane's
    records; a lane with n_records > cap is lost and only its prefix is checked."""
    events = np.asarray(events, dtype=np.uint32)
    cap = events.shape[-1]
    for idx in np.ndindex(*events.shape[:-1]):
        n = int(n_records[idx])
        ev = events[idx]
        if n > cap:
            check_lane(ev, N, complete=False)
            continue
        check_lane(ev[:n], N)
        if np.any(ev[n:] != POISON):
            raise ValueError(f"lane {idx}: slots past n_records = {n} are not POISON")


# ---- host pricer ---------------------------------------------------------------------------------------------------
def price_lane(words, close_row, size: float) -> np.ndarray:
    """float64 pnl of every record (record_pnl in csrc/sweep_dev.cuh, strategy_evaluation.py:796-867): an entry costs
    -size * 0.001; an exit earns size / entry * move - size * 0.002 with move = close - entry for a long trip and
    entry - close for a short one, the fp32 closes widened to float64.  Every operation is one correctly rounded
    numpy operation, as the kernels' _rn intrinsics and oracle/sim_oracle.c are."""
    w = np.asarray(words, dtype=np.uint32).astype(np.int64)
    size = np.float64(size)
    px = np.asarray(close_row, dtype=np.float32)[w & BAR_MASK].astype(np.float64)
    pnl = np.full(len(w), -(size * np.float64(0.001)))
    e, x = px[0::2][:len(w) // 2], px[1::2]
    short = (w[0::2][:len(x)] & SELL) != 0
    move = np.where(short, e - x, x - e)
    pnl[1::2] = (size / e) * move - size * np.float64(0.002)
    return pnl


# ---- device inputs -------------------------------------------------------------------------------------------------
def close_rows(rng, S: int, N: int, scale: float = 1.0) -> np.ndarray:
    """float32 [S][N] positive random-walk closes around 100 * scale (scale a power of two keeps them exact)."""
    steps = rng.normal(0.0, 0.002, (S, N))
    base = rng.uniform(50.0, 200.0, (S, 1))
    return (base * np.exp(np.cumsum(steps, axis=1))).astype(np.float32) * np.float32(scale)


def padded_rows(close, ld: int) -> np.ndarray:
    """[S][ld] float32 holding `close` in its first N columns and PAD_PRICE after them."""
    S, N = close.shape
    out = np.full((S, ld), PAD_PRICE, dtype=np.float32)
    out[:, :N] = close
    return out


def pack(lanes, event_cap: int, n_records=None):
    """lanes [pop][S] of word arrays -> (events uint32 [pop][S][event_cap] with POISON past each lane's records,
    lane_stats float64 [pop][S][20] with n_records set and every other field NaN).  n_records [pop][S] overrides the
    counts (a count above event_cap marks a lost lane: its first event_cap words are stored)."""
    pop, S = len(lanes), len(lanes[0])
    events = np.full((pop, S, event_cap), POISON, dtype=np.uint32)
    stats = np.full((pop, S, STATS_WORDS), np.nan)
    for i in range(pop):
        for s in range(S):
            w = np.asarray(lanes[i][s], dtype=np.uint32)
            k = min(len(w), event_cap)
            events[i, s, :k] = w[:k]
            stats[i, s, 0] = len(w) if n_records is None else n_records[i][s]
    return events, stats


def individuals(sizes) -> np.ndarray:
    """b200bt_individual [pop] with the given position sizes (the readers take nothing else from an individual)."""
    out = np.zeros(len(sizes), dtype=INDIV_DTYPE)
    out["rsi_row"], out["rsi_lo"], out["rsi_hi"] = 0, 30.0, 70.0
    out["take_profit"], out["stop_loss"] = 0.03, 0.02
    out["position_size"] = np.asarray(sizes, dtype=np.float64)
    return out


# ---- references ----------------------------------------------------------------------------------------------------
def book(words, pnls, cfg) -> dict:
    """book_ref.book of one individual's lanes, with the equal-days rule of the metrics step (regime_ref._equal_days on
    the merged list): days whose sums are all equal have exactly zero variance on the device, where np.std can leave a
    residue.  Entries alone on their days (each -fee) make such days common in these buffers."""
    out = book_ref.book(list(words), list(pnls), cfg)
    m = book_ref.merged(list(words), list(pnls))
    ev = np.array([r[2] for r in m], dtype=np.uint32)
    pn = np.array([r[3] for r in m], dtype=np.float64)
    return regime_ref._equal_days(out, ev, pn, cfg)


def classes(words, pnl, labels_row, R: int, cfg) -> list:
    """regime_ref.class_stats of one lane."""
    return regime_ref.class_stats(words, pnl, labels_row, R, cfg)


def day_row(words, pnl, cfg, N: int, D: int) -> np.ndarray:
    """cscv_ref.lane_rows of one lane, widened with zero columns to D >= the series' calendar span."""
    row = cscv_ref.lane_rows(words, pnl, cfg, N)
    assert D >= len(row)
    return np.concatenate([row, np.zeros(D - len(row))])


def trips(pnl):
    """trade_mc_ref.trips_from_records of one lane: (fee, trip pnl)."""
    return trade_mc_ref.trips_from_records([{"pnl": p} for p in np.asarray(pnl, dtype=np.float64).tolist()])
