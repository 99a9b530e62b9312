"""The passes over a sweep's trade records at their seams, called through the C ABI on synthetic event buffers
(tests/record_buffers.py) and compared with the float64 references: tests/book_ref.py for b200bt_book_metrics,
tests/cscv_ref.py for b200bt_daily_pnl, tests/regime_ref.py for b200bt_class_stats, tests/trade_mc_ref.py for
b200bt_trade_pnl.

Every case runs all four passes on the same buffer.  The cases put records on the readers' seams: 32-record batches that
carry, close or split calendar days; the book's staged windows (K records per symbol, 1024 bars, one 64-bit symbol mask
per bar, the last bar's entry and force-close); the class stagings; n_records at and past event_cap; padded price rows,
wide day rows and price scales.  Each case asserts that it lands on its seams, from a host model of the kernel's
schedule (book windows, class fills, day batches).  The case builders are pure NumPy, so that
tests/test_record_buffers_host.py checks every buffer built here against the readers' invariants without a GPU.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, field

import numpy as np
import pytest

import cscv_ref
import record_buffers as rb
import trade_mc_ref
from gpu_fixtures import torch_cuda
from oracle import sim_oracle

pytestmark = pytest.mark.gpu

# ---- seams of the readers, copied from csrc/ ------------------------------------------------------------------------
BATCH = 32               # sweep_dev.cuh:185 record_batch: records [base, base + 32), one per lane of a warp
BK_CAP = 512             # book.cu:24 BK_CAP: records staged and merged per window
BK_BARS = 1024           # book.cu:25 BK_BARS: bars per window
BK_MAX_SYMBOLS = 64      # book.cu:26 BK_MAX_SYMBOLS: one 64-bit symbol mask per bar
CL_MAX = 8               # regime.cu:25 CL_MAX: classes per call
CL_STAGE = 64            # regime.cu:26 CL_STAGE: staged records per class


def book_k(S):
    """Records staged per symbol and window (book.cu:73)."""
    return BK_CAP // S


# Books are held to sim_oracle.assert_lanes as in test_gpu_book.py, classes to it without an absolute floor as in
# test_gpu_regime.py.  Day rows: test_gpu_overfitting.py holds them to rel 1e-12.  The device sums a day in warp-tree
# order within each batch of 32, the reference in record order; both are within n * eps * sum |pnl| of the exact sum, and
# these buffers put up to 1024 records of both signs into one day, so the 1e-12 is taken relative to the day's sum of
# |pnl|, not to the sum itself (which can be much smaller).
ROW_REL = 1e-12

EPOCH = 28_401_120                       # 2024-01-01T00:00Z in minutes
MINUTE0 = EPOCH + 777                    # bar 0 is not on a midnight
FIELDS = sim_oracle.STATS_FIELDS


# ---- cases ---------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    close: np.ndarray                 # float32 [S][N]
    lanes: list                       # [pop][S] event words
    sizes: list                       # position size per individual
    cfg: object                       # sim_oracle.Config
    event_cap: int = 0                # 0: the longest lane + 7 (every lane ends in POISON)
    ld_price: int = 0                 # 0: N
    n_records: list | None = None     # [pop][S] overriding the counts (lost lanes)
    labels: np.ndarray | None = None  # uint8 [S][N]; None: every bar in class 0
    R: int = 1
    D: int = 0                        # 0: the calendar span of the series
    seams: dict = field(default_factory=dict)

    def __post_init__(self):
        self.S, self.N = self.close.shape
        self.pop = len(self.lanes)
        self.lanes = [[np.asarray(w, dtype=np.uint32) for w in row] for row in self.lanes]
        self.event_cap = self.event_cap or max(len(w) for row in self.lanes for w in row) + 7
        self.ld_price = self.ld_price or self.N
        self.D = self.D or cscv_ref.calendar(self.cfg, self.N)[1]
        if self.labels is None:
            self.labels = np.zeros((self.S, self.N), dtype=np.uint8)
        if self.n_records is None:
            self.n_records = [[len(w) for w in row] for row in self.lanes]

    def lost(self, i, s):
        return self.n_records[i][s] > self.event_cap

    def pnl(self, i, s):
        return rb.price_lane(self.lanes[i][s], self.close[s], self.sizes[i])


def _cfg(bar_minutes, minute0=MINUTE0, gap=None):
    cfg = sim_oracle.config_of(minute0, bar_minutes)
    if gap is not None:
        cfg.gap_bar, cfg.gap_minutes = gap
    return cfg


def lane_by_days(rng, plan, cfg, N, total):
    """Event words of `total` records: plan[d] records on distinct bars of calendar day d (from the series' first day),
    the rest on random bars after the planned days."""
    day = cscv_ref.day_of(np.arange(N), cfg) - cscv_ref.day_of(np.array([0]), cfg)[0]
    bars = [np.sort(rng.choice(np.nonzero(day == d)[0], size=c, replace=False)) for d, c in enumerate(plan)]
    after = int(np.nonzero(day == len(plan))[0][0])
    bars.append(rb.random_bars(rng, total - sum(plan), N, lo=after))
    return rb.lane_words(np.concatenate(bars), rng.random(total // 2) < 0.5)


# n_records of the lanes of a batch case: empty, inside one batch, one short of / on / one past a batch, two batches
N_RECORDS = (0, 2, 30, 32, 34, 62, 64, 66, 1024)
DAY_PLAN = (5, 27, 64, 160, 31, 1, 0, 0, 10)  # days of 5; 27 closing on record 31; 64 over 2 batches; 160 over 5
CLOCKS = {1: 12 * 1440, 5: 14 * 288, 7: 16 * 206, 1440: 4096}     # bar_minutes: N


def day_seams(words, cfg):
    """Batch seams of b200bt_daily_pnl on one lane: per calendar day the batches it touches and whether it ends on the
    last record of a batch; per batch its distinct days and whether any day between them is empty."""
    w = np.asarray(words, dtype=np.int64)
    days = cscv_ref.day_of(w & rb.BAR_MASK, cfg)
    idx = np.arange(len(w))
    spans, ends_on_seam = set(), False
    for d in np.unique(days):
        j = idx[days == d]
        spans.add(len(np.unique(j // BATCH)))
        ends_on_seam |= j[-1] % BATCH == BATCH - 1 and j[-1] + 1 < len(w)
    full_batches_of_days = any(len(np.unique(days[b:b + BATCH])) == BATCH and np.all(np.diff(days[b:b + BATCH]) > 1)
                               for b in range(0, len(w) - BATCH + 1, BATCH))
    return spans, ends_on_seam, full_batches_of_days


def batch_case(bar_minutes, scale=1.0, glued=False):
    rng = np.random.default_rng(bar_minutes)
    N = CLOCKS[bar_minutes]
    cfg = _cfg(bar_minutes)
    if bar_minutes == 1440:
        planned = rb.lane_words(np.arange(0, 2048, 2), rng.random(512) < 0.5)     # one day per record, a day between
    else:
        planned = lane_by_days(rng, DAY_PLAN, cfg, N, 1024)
    lanes = [[planned if s == len(N_RECORDS) - 1 else rb.random_lane(rng, n, N, last_pair=n > 0 and s % 2 == 1)
              for s, n in enumerate(N_RECORDS)],
             [rb.random_lane(rng, N_RECORDS[(s + 3) % len(N_RECORDS)], N, last_pair=s % 3 == 0 and N_RECORDS[(s + 3) % 9] > 0)
              for s in range(len(N_RECORDS))]]
    seams = {}
    spans, on_seam, full = day_seams(planned, cfg)
    if bar_minutes == 1440:
        seams["32 days in one batch, an empty day between each"] = full
    else:
        seams["days over 1, 2 and 5 batches"] = {1, 2, 5} <= spans
        seams["a day closing on record 31 of its batch"] = on_seam
    seams["every n_records of N_RECORDS"] = sorted(len(w) for w in lanes[0]) == sorted(N_RECORDS)
    gap, D = None, 0
    if glued:
        j = 40                                        # records 32..39 before the seam, 40.. after: inside batch 1
        gap = (int(planned[j] & rb.BAR_MASK), 2 * 1440 + 17)
        seams["the gap inside a batch"] = j % BATCH != 0 and int(planned[j - 1] & rb.BAR_MASK) < gap[0]
        cfg = _cfg(bar_minutes, gap=gap)
        D = cscv_ref.calendar(cfg, N)[1] + 5          # columns past the calendar span stay 0
    seams["bar 0 not on a midnight"] = MINUTE0 % 1440 != 0
    close = rb.close_rows(np.random.default_rng(100 + bar_minutes), len(N_RECORDS), N, scale)
    return Case(close, lanes, [2000.0, 777.25], cfg, ld_price=N + 13, D=D, seams=seams)


def book_windows(lanes, N):
    """The window schedule of book_kernel (book.cu:79-165) on one individual's lanes (sorted bar arrays): per window
    b0, B, the symbol bounding it by its K-th staged record (or None), and the symbols whose first record in the window
    is an exit whose entry an earlier window consumed."""
    S = len(lanes)
    K = book_k(S)
    cur = [0] * S
    out = []
    while True:
        staged = [b[c:c + K] for b, c in zip(lanes, cur)]
        firsts = [int(st[0]) for st in staged if len(st)]
        if not firsts:
            return out
        b0 = min(firsts)
        kth = {s: int(st[K - 1]) for s, st in enumerate(staged) if len(st) == K}
        B = min(list(kth.values()) + [b0 + BK_BARS])
        bound = min(kth, key=kth.get) if kth and min(kth.values()) < b0 + BK_BARS else None
        take = [int(np.sum(st < B)) for st in staged]
        carried = [s for s in range(S) if take[s] and cur[s] % 2 == 1]
        out.append(dict(b0=b0, B=B, bound=bound, carried=carried, n=sum(take),
                        last=[s for s in range(S) if take[s] and int(staged[s][take[s] - 1]) == N - 1]))
        cur = [c + t for c, t in zip(cur, take)]


def _bars(words):
    return (np.asarray(words, dtype=np.int64) & rb.BAR_MASK)


def book_case(S):
    """Dense symbols 0 and 1 (consecutive bars, symbol 1 one bar behind: they bound windows by their K-th record, and
    symbol 0 is left with an exit whose entry an earlier window consumed whatever the parity of K), sparse symbols,
    empty symbols and symbols with the last bar's entry and force-close."""
    rng = np.random.default_rng(S)
    N = 6000
    K = book_k(S)
    n0 = min(3 * K + 6, 1600) // 2 * 2
    lanes = []
    for i in range(2):
        row = [rb.lane_words(np.arange(100 + i + s, 100 + i + s + n0), rng.random(n0 // 2) < 0.5) for s in range(min(S, 2))]
        for s in range(2, S):
            n = 0 if s % 4 == 3 else 2 * int(rng.integers(1, 20))
            row.append(rb.random_lane(rng, n, N, last_pair=n > 0 and s % 5 == 2))
        lanes.append(row)
    wins = book_windows([_bars(w) for w in lanes[0]], N)
    seams = {"K = BK_CAP / S": K == BK_CAP // S and S <= BK_MAX_SYMBOLS,
             "a window bounded by a dense symbol's K-th record": any(w["bound"] in (0, 1) for w in wins),
             "an exit whose entry an earlier window consumed": any(w["carried"] for w in wins),
             "more than one window": len(wins) > 1}
    if S >= 4:
        seams["empty symbols next to dense ones"] = any(len(w) == 0 for w in lanes[0])
    if S >= 3:
        seams["the last bar's entry and force-close"] = any(w["last"] for w in wins)
    close = rb.close_rows(np.random.default_rng(200 + S), S, N)
    return Case(close, lanes, [1500.0, 250.5], _cfg(1), seams=seams)


def book_spacing_case():
    """Windows bounded by exactly b0 + BK_BARS with a record on that bar, and stretches of more than BK_BARS empty bars."""
    N = 9000
    bars = [[0, BK_BARS, BK_BARS + 6, 4000, 4000 + BK_BARS, 4000 + BK_BARS + 1],
            [2, 3, 5000 + 2 * BK_BARS, 8000, N - 1, N - 1],     # the last two: the entry and force-close on N - 1
            []]
    lanes = [[rb.lane_words(b, [k % 2 == 1 for k in range(len(b) // 2)]) for b in bars]]
    wins = book_windows([np.asarray(b, dtype=np.int64) for b in bars], N)
    merged = np.sort(np.concatenate([np.asarray(b) for b in bars]))
    seams = {"a window bounded by b0 + BK_BARS with a record on B":
             any(w["B"] == w["b0"] + BK_BARS and w["B"] in merged for w in wins),
             "more than BK_BARS empty bars between records": np.max(np.diff(merged)) > BK_BARS}
    close = rb.close_rows(np.random.default_rng(300), 3, N)
    return Case(close, lanes, [1000.0], _cfg(1), seams=seams)


def book_full_mask_case():
    """All 64 symbols with a record on one bar (bit 63 of the mask) and an entry and force-close on the last bar; in
    individual 0 every symbol has exactly K = 8 records, so the last bar is a window's first bar, in individual 1 it is
    inside the first window."""
    S, N, shared = BK_MAX_SYMBOLS, 900, 450
    rng = np.random.default_rng(64)
    lanes = []
    for n_rand in (5, 1):
        row = []
        for s in range(S):
            pool = np.setdiff1d(np.arange(N - 1), [shared])
            b = np.sort(np.concatenate([rng.choice(pool, size=n_rand, replace=False), [shared]]))
            row.append(rb.lane_words(np.concatenate([b, [N - 1, N - 1]]), rng.random((n_rand + 3) // 2) < 0.5))
        lanes.append(row)
    w0 = book_windows([_bars(w) for w in lanes[0]], N)
    w1 = book_windows([_bars(w) for w in lanes[1]], N)
    seams = {"every symbol on one bar": all(shared in _bars(w) for row in lanes for w in row),
             "K records per symbol": all(len(w) == book_k(S) for w in lanes[0]),
             "the last bar is a window's first bar, all 64 symbols on it":
             any(w["b0"] == N - 1 and len(w["last"]) == S and w["n"] == 2 * S for w in w0),
             "the last bar inside a window, all 64 symbols on it":
             any(w["b0"] < N - 1 and len(w["last"]) == S for w in w1)}
    close = rb.close_rows(np.random.default_rng(400), S, N)
    return Case(close, lanes, [2000.0, 1000.0], _cfg(5), seams=seams)


def class_fills(labels, R):
    """The largest fill of each class staging of class_stats_kernel (regime.cu:202-232) over a lane's record labels."""
    fill, peak = [0] * R, [0] * R
    for b in range(0, len(labels), BATCH):
        for c in range(R):
            f = fill[c] + int(np.sum(labels[b:b + BATCH] == c))
            peak[c] = max(peak[c], f)
            fill[c] = f - BATCH if f >= BATCH else f
    return peak


def class_case(R):
    """Symbol 0: every record in class R - 1.  Symbol 1: the class changes on every record, entries in class 0 and
    exits cycling through the other classes (an entry and its exit in different classes; class 0 fills its staging
    faster than the others).  Symbol 2: class 0 gets 31 records of the first batch and all 32 of the second (a staging
    of 63), then random labels that include labels >= R, which belong to no class."""
    rng = np.random.default_rng(R)
    N = 5000
    lanes = [[rb.random_lane(rng, n, N, last_pair=k == 0) for k, n in enumerate((300, 322, 400))],
             [rb.random_lane(rng, n, N) for n in (66, 2, 128)]]
    labels = np.full((3, N), 255, dtype=np.uint8)
    labels[0] = R - 1
    for i in (1, 0):                                    # individual 0's labels win on bars both lanes use
        j1 = np.arange(len(lanes[i][1]))
        labels[1, _bars(lanes[i][1])] = np.where(j1 % 2 == 0, 0, 1 + (j1 // 2) % max(R - 1, 1)) % R
        lab2 = rng.integers(0, R + 2, len(lanes[i][2])).astype(np.uint8)
        if i == 0:
            lab2[:64] = 0
            lab2[31] = R                                # record 31 in no class: 31 + 32 staged records of class 0
        labels[2, _bars(lanes[i][2])] = lab2
    alt, lab2 = labels[1, _bars(lanes[0][1])], labels[2, _bars(lanes[0][2])]
    seams = {"R <= CL_MAX": R <= CL_MAX,
             "every record of a lane in one class": bool(np.all(labels[0, _bars(lanes[0][0])] == R - 1)),
             "a staging of CL_STAGE - 1 records": max(class_fills(lab2, R)) == CL_STAGE - 1,
             "records in no class": bool(np.any(lab2 >= R))}
    if R > 1:
        seams["the class changes on every record"] = bool(np.all(np.diff(alt.astype(int)) != 0))
        seams["entries and exits in different classes"] = bool(np.all(alt[0::2] != alt[1::2]))
    if R > 2:
        seams["stagings fill at different rates"] = len(set(np.bincount(alt, minlength=R).tolist())) > 1
    close = rb.close_rows(np.random.default_rng(500 + R), 3, N)
    return Case(close, lanes, [1200.0, 3000.0], _cfg(7), labels=labels, R=R, seams=seams)


CAP = 64


def limits_case():
    """n_records == event_cap (read), event_cap + 1 (lost) in an otherwise valid individual, and an individual whose
    lanes all fit."""
    rng = np.random.default_rng(7)
    N = 3000
    lanes = [[rb.random_lane(rng, CAP, N), rb.random_lane(rng, 2, N), np.zeros(0, np.uint32)],
             [rb.random_lane(rng, 10, N), rb.random_lane(rng, CAP + 2, N), rb.random_lane(rng, 40, N, last_pair=True)],
             [rb.random_lane(rng, 34, N), rb.random_lane(rng, 0, N), rb.random_lane(rng, CAP - 2, N)]]
    n_records = [[len(w) for w in row] for row in lanes]
    n_records[1][1] = CAP + 1
    seams = {"n_records == event_cap": n_records[0][0] == CAP,
             "n_records == event_cap + 1": n_records[1][1] == CAP + 1}
    close = rb.close_rows(np.random.default_rng(600), 3, N)
    return Case(close, lanes, [2000.0, 1000.0, 500.0], _cfg(1), event_cap=CAP, n_records=n_records, seams=seams)


CASES = {
    **{f"batches, {m}-minute bars": (lambda m=m: batch_case(m)) for m in CLOCKS},
    "batches, glued series, wide day rows": lambda: batch_case(1, glued=True),
    **{f"book, S = {S}": (lambda S=S: book_case(S)) for S in (1, 2, 3, 7, 31, 32, 33, 63, 64)},
    "book, window bounded by BK_BARS": book_spacing_case,
    "book, all 64 symbols on one bar and the last bar": book_full_mask_case,
    **{f"classes, R = {R}": (lambda R=R: class_case(R)) for R in range(1, CL_MAX + 1)},
    "lost lanes at event_cap": limits_case,
}
SCALES = (2.0 ** -12, 2.0 ** 10)


# ---- device calls --------------------------------------------------------------------------------------------------
def run(torch, case):
    """All four passes on the case's buffer -> host arrays."""
    from ai_crypto_trader_b200 import _lib
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pop, S, N, D, R = case.pop, case.S, case.N, case.D, case.R
    events, stats = rb.pack(case.lanes, case.event_cap, case.n_records)
    price = dev(rb.padded_rows(case.close, case.ld_price))
    indiv = dev(rb.individuals(case.sizes).view(np.uint8))
    events, stats, labels = dev(events), dev(stats), dev(case.labels)
    c = case.cfg
    cfg = _lib.SweepConfig(c.initial_capital, c.minute0, c.bar_minutes, c.primary, c.secondary_mask, 0, c.gap_bar,
                           c.gap_minutes)
    f64 = dict(dtype=torch.float64, device="cuda")
    book, fit = torch.full((pop, 20), 7.0, **f64), torch.full((pop,), 7.0, **f64)
    lane_pnl, book_pnl = torch.full((pop, S, D), 7.0, **f64), torch.full((pop, D), 7.0, **f64)
    cls = torch.full((R, pop, S, 20), 7.0, **f64)
    ld_trip = max(1, (case.event_cap + 1) // 2)
    trip = torch.full((pop * S, ld_trip), math.nan, **f64)
    n_trips = torch.zeros(pop * S, dtype=torch.int32, device="cuda")
    fee = torch.zeros(pop * S, **f64)
    common = (price.data_ptr(), case.ld_price, S, N, indiv.data_ptr(), pop)
    buf = (stats.data_ptr(), events.data_ptr(), case.event_cap)
    st = _lib.current_stream()
    _lib.call("b200bt_book_metrics", *common, ctypes.byref(cfg), *buf, book.data_ptr(), fit.data_ptr(), st)
    _lib.call("b200bt_daily_pnl", *common, ctypes.byref(cfg), *buf, lane_pnl.data_ptr(), D, book_pnl.data_ptr(), st)
    _lib.call("b200bt_class_stats", *common, ctypes.byref(cfg), *buf, labels.data_ptr(), N, R, cls.data_ptr(), st)
    _lib.call("b200bt_trade_pnl", *common, *buf, trip.data_ptr(), ld_trip, n_trips.data_ptr(), fee.data_ptr(), st)
    torch.cuda.synchronize()
    host = lambda t: t.cpu().numpy()
    return dict(book=host(book), fitness=host(fit), lane_pnl=host(lane_pnl), book_pnl=host(book_pnl), classes=host(cls),
                trip=host(trip).reshape(pop, S, ld_trip), n_trips=host(n_trips).reshape(pop, S),
                fee=host(fee).reshape(pop, S))


def _fields(row):
    row = np.ascontiguousarray(row, dtype=np.float64)
    d = {f: float(row[k]) for k, f in enumerate(FIELDS[:-1])}
    d["trade_hash"] = int(row.view(np.uint64)[19])
    return d


def _is_lost(row, where):
    g = _fields(row)
    assert g["n_records"] == -1.0 and math.isnan(g["score"]), where
    assert all(g[f] == 0.0 for f in FIELDS[1:-1] if f != "score") and g["trade_hash"] == 0, where


def _row_scale(words, pnl, cfg, N, D):
    """float64 [D]: each day's sum of |pnl| (the scale of ROW_REL)."""
    return rb.day_row(words, np.abs(pnl), cfg, N, D)


def check(case, out, where):
    """Every output of `run` against the references."""
    pop, S, N, D = case.pop, case.S, case.N, case.D
    for i in range(pop):
        lost = [case.lost(i, s) for s in range(S)]
        pnls = [None if lost[s] else case.pnl(i, s) for s in range(S)]
        # book
        if any(lost):
            _is_lost(out["book"][i], f"{where} book {i}")
            assert math.isnan(out["fitness"][i])
        else:
            want = rb.book(case.lanes[i], pnls, case.cfg)
            sim_oracle.assert_lanes(_fields(out["book"][i]), want, f"{where} book {i}")
            assert out["fitness"][i] == out["book"][i][12] or np.isnan(out["fitness"][i]) and np.isnan(out["book"][i][12])
        # day rows, the book row as their sum over symbols in order
        rows = out["lane_pnl"][i]
        np.testing.assert_array_equal(out["book_pnl"][i], cscv_ref.book_row(list(rows)), err_msg=f"{where} book row {i}")
        for s in range(S):
            w = f"{where} lane ({i}, {s})"
            if lost[s]:
                assert np.all(np.isnan(rows[s])), w
                continue
            want = rb.day_row(case.lanes[i][s], pnls[s], case.cfg, N, D)
            np.testing.assert_array_equal(rows[s] == 0, want == 0, err_msg=f"{w}: days without records")
            scale = _row_scale(case.lanes[i][s], pnls[s], case.cfg, N, D)
            assert np.all(np.abs(rows[s] - want) <= ROW_REL * scale), (w, np.max(np.abs(rows[s] - want) / np.maximum(scale, 1e-300)))
        # class stats
        for s in range(S):
            if lost[s]:
                for r in range(case.R):
                    _is_lost(out["classes"][r, i, s], f"{where} lane ({i}, {s}) class {r}")
                continue
            want = rb.classes(case.lanes[i][s], pnls[s], case.labels[s], case.R, case.cfg)
            for r in range(case.R):
                sim_oracle.assert_lanes(_fields(out["classes"][r, i, s]), want[r], f"{where} lane ({i}, {s}) class {r}",
                                        atol=0)
        # trip pnl, and the day row's sum against the net profit of the trips
        for s in range(S):
            w = f"{where} lane ({i}, {s})"
            assert out["fee"][i, s] == case.sizes[i] * 0.001, w
            if lost[s]:
                assert out["n_trips"][i, s] == -1, w
                continue
            T = len(case.lanes[i][s]) // 2
            fee, trips = rb.trips(pnls[s])
            assert out["n_trips"][i, s] == T, w
            assert np.array_equal(out["trip"][i, s, :T], trips), w
            assert T == 0 or out["fee"][i, s] == fee, w
            net = trade_mc_ref.net_profit(out["fee"][i, s], out["trip"][i, s, :T])
            assert abs(rows[s].sum() - net) <= ROW_REL * np.abs(pnls[s]).sum(), w


# ---- tests ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_passes_match_the_references(torch_cuda, name):
    case = CASES[name]()
    assert case.seams and all(case.seams.values()), {k: v for k, v in case.seams.items() if not v}
    check(case, run(torch_cuda, case), name)


def test_single_symbol_book_is_its_one_class(torch_cuda):
    """A book of one symbol is that lane's class_stats with R = 1 and every record in class 0."""
    case = book_case(1)
    out = run(torch_cuda, case)
    for i in range(case.pop):
        book, cls = _fields(out["book"][i]), out["classes"][0, i, 0]
        sim_oracle.assert_lanes(_fields(cls), book, f"individual {i}", atol=0)


def test_price_scales_leave_every_output_unchanged(torch_cuda):
    """Closes scaled by 2^-12 and 2^10: each pass still matches its reference, and since a record's pnl depends on the
    closes only through move / entry, every output is bit-identical to the unscaled run."""
    base = run(torch_cuda, batch_case(7))
    for scale in SCALES:
        case = batch_case(7, scale=scale)
        assert np.all(np.isfinite(case.close)) and case.close.min() > 0
        out = run(torch_cuda, case)
        check(case, out, f"scale {scale}")
        for k in base:
            assert np.array_equal(np.asarray(out[k]).view(np.uint8), np.asarray(base[k]).view(np.uint8)), (scale, k)
