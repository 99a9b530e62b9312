"""Walk-forward evaluation at its limits (csrc/walk_forward.cu): segment lanes against the C oracle run once per segment
(tests/test_gpu_walk_forward.py's _oracle: the oracle on each segment's slice, words shifted to global bars, records scored
as one list by tests/book_ref.book), built so that each case reaches the edge it is named for:

* segment lengths around the 512-bar cp.async groups and the 64-bar windows, starts at every residue mod 4, and the
  16-byte / 4-byte choice of GroupRing on both sides, also with the price and RSI rows aligned differently;
* segments that fire on every bar (batches at every fill level, a full event queue at the segment's end), hundreds of
  segments in one lane, and event buffers of exactly n_records, n_records - 1 and 1 words;
* the per-segment reload of ScanConst, take-profit / stop-loss / size and fees between individuals one field apart;
* the lane grid (ceil(J / 8) * S CTAs) and the table bounds;
* bars just below 2^30 with minute0 as large as the clock check accepts, on 1- and 3-minute bars;
* the calendar of 7- and 1440-minute bars with minute0 off the bar grid;
* b200bt_decode_individuals against decode_population at the edges of its period table and of fp32."""
import ctypes as C

import numpy as np
import pytest

from abi_header import ELIMIT
from gpu_fixtures import torch_cuda  # noqa: F401
from oracle import sim_oracle
from test_gpu_walk_forward import BUSY, _check, _oracle, _run

pytestmark = pytest.mark.gpu

GOALS = {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]}
BAR_MASK, EXIT, SELL = 0x3FFFFFFF, 0x40000000, 0x80000000
# an entry on every flat bar and an exit on the bar after (take-profit / stop-loss of 10^-6): long, and short (RSI is
# never below 0, always above -1); and a rule that never trades
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)
DENSE_SHORT = dict(rsi_period=5, rsi_oversold=0, rsi_overbought=-1, take_profit=0.0001, stop_loss=0.0001)
QUIET = dict(rsi_period=5, rsi_oversold=-1, rsi_overbought=101)
SW_GROUP, SW_EVQ, SW_WARPS = 512, 128, 8          # csrc/sweep_dev.cuh


def _sweep(S, N, seed, minute0=None, bar_minutes=1):
    """(sweep, host close [S][N], host bank [S][P][N]) of a synthetic market."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    ohlcv = synth.synth_ohlcv(S, N, seed_base=seed)
    minute0 = synth.EPOCH_2024_MINUTES + 7 * 60 + 13 if minute0 is None else minute0
    sweep = PopulationSweep(MarketData(ohlcv, minute0=minute0, bar_minutes=bar_minutes), optimization_goals=GOALS,
                            mode="fused")
    return sweep, ohlcv[3].astype(np.float32), sweep.bank.cpu().numpy()


@pytest.fixture(scope="module", params=[6001, 6000], ids=["ld-ragged", "ld-x4"])
def market(torch_cuda, request):
    return _sweep(2, request.param, seed=123)


def _bars(words):
    return (np.asarray(words, dtype=np.uint32) & BAR_MASK).astype(np.int64)


def _vec16(price_ptr, ld_price, rsi_ptr, ld_rsi, P, row, s, a):
    """Whether segment_sweep_kernel streams a segment from bar a of symbol s, RSI row `row`, with 16-byte copies."""
    return ((price_ptr + 4 * (s * ld_price + a)) | (rsi_ptr + 4 * ((s * P + row) * ld_rsi + a))) % 16 == 0


def _sweep_vec16(sweep, params, a, k, s):
    from ai_crypto_trader_b200 import _lib
    m = sweep.market
    row = sweep.period_row[int(params[k].get("rsi_period", 14))]
    return _vec16(m.close.data_ptr(), _lib.ld(m.close), sweep.bank.data_ptr(), _lib.ld(sweep.bank), sweep.bank.shape[1],
                  row, s, a)


def _check_lanes(sweep, close, bank, params, schedules, got, ev, lanes, event_cap, where):
    """Lanes [(j, s)] of a run (stats fields {f: [J][S]}, events [J][S][cap] or None) against the oracle."""
    want, want_ev = [], []
    for j, s in lanes:
        o, w = _oracle(sweep, close, bank, params, schedules[j], s)
        want.append(o)
        want_ev.append([w[:event_cap]])
    sim_oracle.assert_lanes([{f: got[f][j, s] for f in got} for j, s in lanes], want, where)
    if ev is not None:
        sim_oracle.assert_events([[ev[j][s]] for j, s in lanes], want_ev, where)


# -- 1. group and alignment seams -----------------------------------------------------------------------------------------
def test_group_and_alignment_seams(market):
    """Every length around the 64-bar windows and 512-bar groups, from every residue mod 4 and a group-aligned start, alone
    and followed by a segment of the same length (whose start has another residue when the length is odd) on another
    RSI row."""
    sweep, close, bank = market
    N = sweep.market.N
    lengths = (1, 2, 3, 4, 5, 63, 64, 65, 511, 512, 513, 1023, 1024, 1025, 1536)
    starts = (1000, 1001, 1002, 1003, 4 * SW_GROUP)
    params = [dict(BUSY, rsi_period=p) for p in (5, 6, 7, 8)]
    schedules = []
    for L in lengths:
        for a in starts:
            for k in range(len(params)):
                sched = [(a, a + L, k)]
                if a + 2 * L <= N:
                    sched.append((a + L, a + 2 * L, (k + 1) % len(params)))
                schedules.append(sched)
    forms = {}
    for sched in schedules:
        for a, b, k in sched:
            for s in range(sweep.market.S):
                forms.setdefault(b - a, set()).add(_sweep_vec16(sweep, params, a, k, s))
    for L in (511, 512, 513):
        assert forms[L] == {True, False}, (L, forms[L])
    got, _ = _check(sweep, close, bank, params, schedules, event_cap=N + 1)
    assert got["n_records"][[i for i, sc in enumerate(schedules) if sc[0][1] - sc[0][0] >= 512]].min() > 0


# -- 2. price and RSI rows aligned differently ----------------------------------------------------------------------------
def test_price_and_rsi_rows_aligned_differently(market):
    """The bank as a view one float into a wider NaN-padded buffer (ld_rsi = N + 5 != ld_price): segments where only the
    price row or only the RSI row starts on 16 bytes, which must take the 4-byte copies, beside ones where both or
    neither do."""
    import torch
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import _stats_fields, decode_population
    from ai_crypto_trader_b200.walk_forward import segment_tables
    sweep, close, bank = market
    m = sweep.market
    S, P, N = m.S, sweep.bank.shape[1], m.N
    wide = torch.full((S, P, N + 5), float("nan"), dtype=torch.float32, device="cuda")
    view = wide[:, :, 1:N + 1]
    view.copy_(sweep.bank)
    ld_price, ld_rsi = _lib.ld(m.close), _lib.ld(view)
    assert ld_rsi == N + 5 != ld_price
    params = [dict(BUSY, rsi_period=p) for p in (5, 6, 7, 8)]
    rng = np.random.default_rng(21)
    schedules, kinds = [], set()
    for j in range(24):
        sched, a = [], int(rng.integers(0, 40))
        while True:
            L = int(rng.choice([SW_GROUP - 1, SW_GROUP, SW_GROUP + 1, 2 * SW_GROUP + 3, 1500]))
            if a + L > N:
                break
            k = int(rng.integers(len(params)))
            sched.append((a, a + L, k))
            row = sweep.period_row[params[k]["rsi_period"]]
            for s in range(S):
                pa = (m.close.data_ptr() + 4 * (s * ld_price + a)) % 16 == 0
                ra = (view.data_ptr() + 4 * ((s * P + row) * ld_rsi + a)) % 16 == 0
                kinds.add((pa, ra))
            a += L + int(rng.integers(0, 4))
        schedules.append(sched)
    assert kinds >= {(True, False), (False, True)}, kinds
    packed = decode_population(params, sweep.period_row)
    indiv = torch.from_numpy(packed.view(np.uint8).copy()).cuda()
    seg, begin = segment_tables(schedules)
    seg_d, begin_d = torch.from_numpy(seg.view(np.int64)).cuda(), torch.from_numpy(begin).cuda()
    stats = torch.empty((len(schedules), S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device="cuda")
    cap = N + 1
    events = torch.zeros((len(schedules), S, cap), dtype=torch.int32, device="cuda")
    _lib.call("b200bt_sweep_segments", m.close.data_ptr(), ld_price, view.data_ptr(), ld_rsi, P, S, N, indiv.data_ptr(),
              len(packed), seg_d.data_ptr(), begin_d.data_ptr(), len(schedules), C.byref(sweep.cfg), stats.data_ptr(),
              events.data_ptr(), cap, _lib.current_stream())
    got = _stats_fields(stats.cpu().numpy())
    ev = events.cpu().numpy().view(np.uint32)
    lanes = [(j, s) for j in range(len(schedules)) for s in range(S)]
    _check_lanes(sweep, close, bank, params, schedules, got, ev, lanes, cap, "rows aligned differently")


# -- 3. dense segment ends and long schedules -----------------------------------------------------------------------------
def test_dense_segment_ends(market):
    """Adjacent segments of every length 1..130 (across the 32-record batches, the 64-bar windows and the 128-entry queue),
    traded in turn by an every-bar long rule, an every-bar short rule and a rule that never trades, in three rotations."""
    sweep, close, bank = market
    params = [DENSE, DENSE_SHORT, QUIET]
    schedules = []
    for lengths in (range(1, 91), range(91, 131)):
        for rot in range(3):
            sched, a = [], 100
            for i, L in enumerate(lengths):
                sched.append((a, a + L, (i + rot) % 3))
                a += L
            schedules.append(sched)
    assert schedules[-1][-1][1] <= sweep.market.N
    _, want_ev = _check(sweep, close, bank, params, schedules, event_cap=sweep.market.N + 1)
    # records per dense segment: every batch fill level at a segment's end, and segments longer than the queue
    counts, dense_bars = [], 0
    for sched, lanes in zip(schedules, want_ev):
        for ev in lanes:
            bars = _bars(ev)
            for a, b, k in sched:
                n = int(np.searchsorted(bars, b) - np.searchsorted(bars, a))
                if k == 2:
                    assert n == 0
                else:
                    counts.append(n)
                    dense_bars += b - a
    # records come in (entry, exit) pairs and a segment's queue starts empty: its last batch holds n % 32 of them
    assert sum(counts) >= 0.9 * dense_bars
    assert {n % 32 for n in counts} == set(range(0, 32, 2)) and max(counts) > SW_EVQ


def _long_schedule(rng, N, n_params):
    """Adjacent segments of 7..40 bars covering [0, N), individuals drawn at random."""
    lengths = rng.integers(7, 34, size=N // 20).tolist()
    diff = N - sum(lengths)
    while diff:
        i = int(rng.integers(len(lengths)))
        step = max(7 - lengths[i], min(40 - lengths[i], diff))
        lengths[i] += step
        diff -= step
    bounds = np.concatenate([[0], np.cumsum(lengths)])
    return [(int(a), int(b), int(rng.integers(n_params))) for a, b in zip(bounds[:-1], bounds[1:])]


def test_hundreds_of_segments_in_one_lane(market):
    """One lane of >= 300 adjacent segments of 7..40 bars over the whole series: the hash, the days and the equity / peak /
    drawdown carry across every boundary.  Event buffers of exactly n_records words, one word short, and one word."""
    from ai_crypto_trader_b200 import synth
    sweep, close, bank = market
    N = sweep.market.N
    params = [DENSE, DENSE_SHORT, QUIET, dict(BUSY)] + synth.random_population(4, seed=8)
    sched = _long_schedule(np.random.default_rng(3), N, len(params))
    assert len(sched) >= 300 and sched[0][0] == 0 and sched[-1][1] == N
    assert all(7 <= b - a <= 40 for a, b, _ in sched) and all(x[1] == y[0] for x, y in zip(sched, sched[1:]))
    counts = [len(_oracle(sweep, close, bank, params, sched, s)[1]) for s in range(sweep.market.S)]
    n = min(counts)
    assert n > 1000
    for cap in (n, n - 1, 1):
        got, _ = _check(sweep, close, bank, params, [sched], event_cap=cap)
        assert got["n_records"][0].tolist() == counts
    assert got["n_days"][0].min() >= 4


# -- 4. the per-segment reload --------------------------------------------------------------------------------------------
RELOAD_BASE = dict(rsi_period=7, rsi_oversold=35, rsi_overbought=65, take_profit=1, stop_loss=1, max_position_size=5)
RELOAD_VARIANTS = {"rsi_row": dict(rsi_period=9), "rsi_lo": dict(rsi_oversold=38), "rsi_hi": dict(rsi_overbought=62),
                   "take_profit": dict(take_profit=0.4), "stop_loss": dict(stop_loss=0.3),
                   "position_size": dict(max_position_size=15)}


def test_per_segment_reload(market):
    """Schedules whose segments alternate between individuals one decoded field apart, with the odd one first, last or
    every other: a field kept from the previous segment, or from the schedule's first (init_acc), changes the lane."""
    from ai_crypto_trader_b200.sweep import decode_population
    sweep, close, bank = market
    params = [dict(RELOAD_BASE)] + [dict(RELOAD_BASE, **v) for v in RELOAD_VARIANTS.values()]
    packed = decode_population(params, sweep.period_row)
    for i, field in enumerate(RELOAD_VARIANTS, start=1):
        differ = [f for f in packed.dtype.names if packed[f][0] != packed[f][i]]
        assert differ == [field], (field, differ)
    cuts = [(50 + 400 * q, 450 + 400 * q) for q in range(8)]
    schedules = [[(a, b, 0) for a, b in cuts]]
    for i in range(1, len(params)):
        schedules.append([(a, b, i if q % 2 == 0 else 0) for q, (a, b) in enumerate(cuts)])
        schedules.append([(a, b, 0 if q % 2 == 0 else i) for q, (a, b) in enumerate(cuts)])
        schedules.append([(a, b, i if q == 0 else 0) for q, (a, b) in enumerate(cuts)])
        schedules.append([(a, b, i if q == len(cuts) - 1 else 0) for q, (a, b) in enumerate(cuts)])
    got, _ = _check(sweep, close, bank, params, schedules, event_cap=sweep.market.N + 1)
    base = [(got["net_profit"][0, s], got["trade_hash"][0, s]) for s in range(sweep.market.S)]
    for j in range(1, len(schedules)):
        assert any((got["net_profit"][j, s], got["trade_hash"][j, s]) != base[s] for s in range(sweep.market.S)), j


# -- 5. lane grid ---------------------------------------------------------------------------------------------------------
def _random_schedules(rng, N, J, n_params):
    out = []
    for _ in range(J):
        k = int(rng.integers(1, 6))
        cuts = np.sort(rng.choice(np.arange(1, N), size=2 * k, replace=False))
        out.append([(int(cuts[2 * i]), int(cuts[2 * i + 1]), int(rng.integers(n_params))) for i in range(k)])
    return out


@pytest.mark.parametrize("S", [1, 3, 11])
def test_lane_grid(torch_cuda, S):
    """J in {1, 7, 8, 9, 1025} schedules on S symbols (ceil(J / 8) * S CTAs, symbol = CTA % S): every lane of the small
    grids and a seeded sample of the large one against the oracle; one schedule repeated at several j gives bit-identical
    lanes; a schedule at the table bounds (end == N, the last individual, the bank's last row) is valid."""
    from ai_crypto_trader_b200 import synth
    N = 2500
    sweep, close, bank = _sweep(S, N, seed=40 + S)
    P = sweep.bank.shape[1]
    params = synth.random_population(5, seed=S) + [dict(BUSY), dict(BUSY, rsi_period=max(sweep.period_row))]
    assert sweep.period_row[params[-1]["rsi_period"]] == P - 1
    bound = [(7, 300, 5), (N - 700, N, len(params) - 1)]
    repeated = [(100, 900, 5), (900, 1700, 2), (1800, 2400, 5)]
    rng = np.random.default_rng(S)
    for J in (1, 7, 8, 9, 1025):
        schedules = _random_schedules(rng, N, J, len(params))
        schedules[J - 1] = bound
        rep = sorted({0, 7, 8, J - 2} & set(range(J - 1)))
        for j in rep:
            schedules[j] = repeated
        got, ev = _run(sweep, params, schedules, event_cap=N + 1)
        if J <= 9:
            lanes = [(j, s) for j in range(J) for s in range(S)]
        else:
            pick = np.random.default_rng(J + S).choice(J * S, size=48, replace=False)
            lanes = sorted({(int(x) // S, int(x) % S) for x in pick} | {(J - 1, s) for s in range(S)} |
                           {(j, s) for j in rep for s in range(S)})
        _check_lanes(sweep, close, bank, params, schedules, got, ev, lanes, N + 1, f"J={J} S={S}")
        assert np.all(got["n_records"][J - 1] >= 0)
        for j in rep[1:]:
            for f in got:
                np.testing.assert_array_equal(got[f][j].view(np.uint64), got[f][rep[0]].view(np.uint64),
                                              err_msg=f"{f}: schedule at j={j} vs j={rep[0]}, J={J} S={S}")
            np.testing.assert_array_equal(ev[j], ev[rep[0]])


# -- 6. the top of the bar range ------------------------------------------------------------------------------------------
class _Tail:
    """Host rows [..][n] of bars [lo, lo + n) of a longer series, sliced by global bar: x[s, a:b] / x[s, row, a:b]."""

    def __init__(self, lo, rows):
        self.lo, self.rows = lo, rows

    def __getitem__(self, key):
        *head, sl = key
        assert sl.start >= self.lo and sl.stop <= self.lo + self.rows.shape[-1], (sl, self.lo)
        return self.rows[tuple(head)][sl.start - self.lo:sl.stop - self.lo]


def test_top_of_the_bar_range(torch_cuda):
    """N = 2^30 - 1 bars (S = 1, P = 1) with minute0 as large as the clock check accepts, on 1- and 3-minute bars (the
    latter takes minute0 + bar * bar_minutes to within 1444 of 2^32).  The rows are NaN but for the last 5000 bars, where a
    synthetic close and its RSI row sit; segments lie there, one of them ending on bar N - 1.  Event words carry bars above
    2^29 with their EXIT / SELL bits intact."""
    import types

    import torch
    from ai_crypto_trader_b200 import _lib, synth
    from ai_crypto_trader_b200.sweep import _stats_fields, decode_population
    from ai_crypto_trader_b200.walk_forward import segment_tables
    from oracle import indicators_ref
    free, _ = torch.cuda.mem_get_info()
    if free < 10 * 2 ** 30:
        pytest.skip(f"two 2^30-bar fp32 rows need ~8.6 GB; {free / 2 ** 30:.1f} GiB of device memory is free (< 10 GiB)")
    N, T = 2 ** 30 - 1, 5000
    lo = N - T
    close = synth.synth_ohlcv(1, T, seed_base=31)[3].astype(np.float32)              # [1][T]
    rsi = indicators_ref.rsi_bank(close[0], [5])                                        # [1][T]
    params = [DENSE, DENSE_SHORT, dict(BUSY), QUIET]
    schedules = [
        [(N - 300, N, 0)],                                                              # dense, up to the last bar
        [(N - 300, N - 1, 1), (N - 1, N, 0)],                                           # dense short, then the last bar alone
        [(lo + 10, lo + 1700, 2), (lo + 1700, lo + 2213, 0), (lo + 2300, lo + 2301, 1), (lo + 3000, N, 2)],
        [(lo + 5 + 37 * q, lo + 5 + 37 * (q + 1), q % 4) for q in range(130)],
    ]
    packed = decode_population(params, {5: 0})
    indiv = torch.from_numpy(packed.view(np.uint8).copy()).cuda()
    seg, begin = segment_tables(schedules)
    seg_d, begin_d = torch.from_numpy(seg.view(np.int64)).cuda(), torch.from_numpy(begin).cuda()
    J, cap = len(schedules), 2 * T
    stats = torch.empty((J, 1, _lib.LANE_STATS_WORDS), dtype=torch.float64, device="cuda")
    events = torch.zeros((J, 1, cap), dtype=torch.int32, device="cuda")
    price = row = None
    try:
        price = torch.full((N,), float("nan"), dtype=torch.float32, device="cuda")
        row = torch.full((N,), float("nan"), dtype=torch.float32, device="cuda")
        price[lo:] = torch.from_numpy(close[0]).cuda()
        row[lo:] = torch.from_numpy(rsi[0]).cuda()
        for bar_minutes in (1, 3):
            minute0 = (1 << 32) - 1441 - N * bar_minutes
            ref_cfg = sim_oracle.config_of(minute0, bar_minutes, GOALS)

            def launch(m0):
                cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=m0, bar_minutes=bar_minutes,
                                       primary=ref_cfg.primary, secondary_mask=ref_cfg.secondary_mask, variant=0)
                _lib.call("b200bt_sweep_segments", price.data_ptr(), N, row.data_ptr(), N, 1, 1, N, indiv.data_ptr(),
                          len(packed), seg_d.data_ptr(), begin_d.data_ptr(), J, C.byref(cfg), stats.data_ptr(),
                          events.data_ptr(), cap, _lib.current_stream())

            with pytest.raises(_lib.B200btError) as e:
                launch(minute0 + 1)
            assert e.value.status == ELIMIT
            events.zero_()
            launch(minute0)
            got = _stats_fields(stats.cpu().numpy())
            ev = events.cpu().numpy().view(np.uint32)
            sweep = types.SimpleNamespace(market=types.SimpleNamespace(minute0=minute0, bar_minutes=bar_minutes),
                                          period_row={5: 0})
            host_close, host_bank = _Tail(lo, close), _Tail(lo, rsi[None])
            _check_lanes(sweep, host_close, host_bank, params, schedules, got, ev, [(j, 0) for j in range(J)], cap,
                         f"top of the bar range, {bar_minutes}-minute bars")
            words = [_oracle(sweep, host_close, host_bank, params, sc, 0)[1] for sc in schedules]
            assert len(words[0]) >= 290 and len(words[1]) >= 290
            assert _bars(words[0])[-1] == N - 1 and _bars(words[1])[-1] == N - 1
            for w in words:
                assert np.all(_bars(w) > 2 ** 29)
            allw = np.concatenate(words)
            kinds = {(bool(x & EXIT), bool(x & SELL)) for x in allw.tolist()}
            assert kinds == {(False, False), (False, True), (True, False), (True, True)}, kinds
    finally:
        del price, row
        torch.cuda.empty_cache()


# -- 7. calendar ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bar_minutes", [7, 1440])
def test_calendar(torch_cuda, bar_minutes):
    """Segments days apart with no trade between them, segments that start on a day's first bar (on a 7-minute clock also
    exactly at midnight) or end on the bar before one, on a clock whose minute0 is not a multiple of the bar."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.walk_forward import first_bar_of_day
    N = 6000 if bar_minutes == 7 else 600
    minute0 = synth.EPOCH_2024_MINUTES + 2 * 1440 + (4 if bar_minutes == 7 else 611)
    assert minute0 % bar_minutes != 0
    sweep, close, bank = _sweep(2, N, seed=60 + bar_minutes, minute0=minute0, bar_minutes=bar_minutes)
    d0 = minute0 // 1440
    first = [first_bar_of_day(d, minute0, bar_minutes) for d in range(d0, d0 + N * bar_minutes // 1440 + 2)]
    first = [t for t in first if 0 < t < N]
    params = [DENSE, DENSE_SHORT, dict(BUSY), QUIET]
    w = 40 if bar_minutes == 7 else 2
    inside = lambda sched: [(a, b, k) for a, b, k in sched if 0 <= a and b <= N]
    schedules = [
        [(first[d], first[d] + w, d % 2) for d in range(1, len(first), 4)],                   # from a day's first bar
        [(first[d] - w, first[d], 2 - d % 3) for d in range(1, len(first), 3)],               # up to the bar before one
        [(first[d], first[d + 1], 2) for d in range(0, len(first) - 1, 5)],                   # whole days, 4 quiet ones between
        [(first[d] - w, first[d] + w, (d % 2) * 2) for d in range(1, len(first), 6)],         # across midnight
    ]
    if bar_minutes == 7:
        midnight = [t for t in range(N) if (minute0 + t * bar_minutes) % 1440 == 0]
        assert len(midnight) >= 3 and set(midnight) <= set(first)
        schedules.append([(t, t + w, 0) for t in midnight])
        schedules.append([(t - w, t, 1) for t in midnight])
    schedules = [inside(sched) for sched in schedules]
    for sched in schedules:
        assert all(x[1] <= y[0] for x, y in zip(sched, sched[1:])) and sched[-1][1] <= N, sched
    got, _ = _check(sweep, close, bank, params, schedules, event_cap=N + 1)
    assert got["n_days"].min() >= 3
    # days without trades between the segments: fewer trade days than the schedule spans
    span = [(minute0 + sc[-1][1] * bar_minutes) // 1440 - (minute0 + sc[0][0] * bar_minutes) // 1440 for sc in schedules]
    assert np.all(got["n_days"].max(axis=1) < np.array(span))


# -- 8. decode at its limits ----------------------------------------------------------------------------------------------
DECODE_FIELDS = ("rsi_row", "rsi_lo", "rsi_hi", "reserved", "take_profit", "stop_loss", "position_size")
F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.nextafter(np.float32(0), np.float32(1)))
EDGE_PERIODS = [0, -0.5, -0.0, 14.999, 255, 255.999, 256, 1e9, -1, np.nan, np.inf, -np.inf, 3, 1e300, 127.5, 5]
EDGE_THRESHOLDS = [np.inf, -np.inf, 1e39, -1e39, -0.0, 0.0, np.nan, 1e-310, -1e-310, 1e-40, -1e-40, F32_TINY,
                   F32_TINY / 2, F32_MAX, F32_MAX * (1 + 2 ** -25), -F32_MAX * (1 + 2 ** -25), F32_MAX * (1 + 2 ** -24),
                   30.0, np.nextafter(30.0, 99), np.nextafter(70.0, 0), 33.3]
EDGE_EXITS = [-0.0, 0.0, np.nan, np.inf, -np.inf, 5e-324, 1e308, -3.0, 0.7, 1.0]
EDGE_SIZES = [np.nan, 20.0, np.nextafter(20.0, np.inf), -5.0, np.inf, -np.inf, 1e-320, -0.0, 19.999999, 5.0]


def _period_table(rng):
    """A full 256-entry period -> row table: distinct rows, period 3 and a few others not in the bank (-1)."""
    table = rng.permutation(256).astype(np.int32) * 3 + 7
    table[[3, 100, 254]] = -1
    return table


def _decode_device(matrix, cols, table):
    import torch
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import INDIVIDUAL_DTYPE
    dev = torch.from_numpy(np.ascontiguousarray(matrix, dtype=np.float64)).cuda()
    out = torch.zeros(len(matrix) * C.sizeof(_lib.Individual), dtype=torch.uint8, device="cuda")
    _lib.call("b200bt_decode_individuals", dev.data_ptr(), matrix.shape[1], len(matrix), (C.c_int * 6)(*cols),
              (C.c_int32 * len(table))(*[int(x) for x in table]), len(table), out.data_ptr(), _lib.current_stream())
    return out.cpu().numpy().view(INDIVIDUAL_DTYPE)


def _assert_decoded(got, matrix, cols, table):
    """Row by row against decode_population: every field byte for byte, except that a field decode_population gives as
    NaN must be a NaN (of any payload); a row decode_population refuses (period outside the bank) has rsi_row -1 and the
    other fields of the same row with a period in the bank."""
    from ai_crypto_trader_b200.sweep import decode_population
    from ai_crypto_trader_b200.walk_forward import DECODE_GENES
    period_row = {p: int(r) for p, r in enumerate(table) if r >= 0}
    valid = next(iter(period_row))
    for i, row in enumerate(matrix):
        p = {g: float(row[c]) for g, c in zip(DECODE_GENES, cols) if c >= 0}
        try:
            want = decode_population([p], period_row)[0]
            refused = False
        except KeyError:
            want = decode_population([dict(p, rsi_period=valid)], period_row)[0]
            refused = True
        g = got[i]
        for f in DECODE_FIELDS:
            a, b = np.asarray(g[f]), np.asarray(want[f])
            if f == "rsi_row" and refused:
                assert int(a) == -1, (i, p)
            elif b.dtype.kind == "f" and np.isnan(b):
                assert np.isnan(a), (i, f, p, a)
            else:
                assert a.tobytes() == b.tobytes(), (i, f, p, a, b)


@pytest.mark.filterwarnings("ignore::RuntimeWarning")        # NumPy on the edge genes: NaN casts, fp32 overflow
@pytest.mark.parametrize("n", [1, 127, 128, 129, 257])
def test_decode_at_its_limits(torch_cuda, n):
    """Edge genes (periods on and off the 256-entry table, truncated; thresholds at +-inf, beyond fp32, -0.0, subnormal,
    NaN; exits at -0.0 and NaN; sizes NaN, 20, just above 20, negative) in gene columns scattered over a 41-wide row, the
    other columns junk, across the 128-thread block seams."""
    rng = np.random.default_rng(n)
    table = _period_table(rng)
    ld = 41
    cols = [37, 2, 19, 40, 0, 23]
    M = rng.uniform(-1e6, 1e6, size=(n, ld))
    M[:, ::3] = np.nan
    edges = [EDGE_PERIODS, EDGE_THRESHOLDS, EDGE_THRESHOLDS[::-1], EDGE_EXITS, EDGE_EXITS[::-1], EDGE_SIZES]
    for c, e in zip(cols, edges):
        M[:, c] = [e[(i * 11 + c) % len(e)] for i in range(n)]      # 11: prime to every list's length
    M[0, cols] = [255, 30.0, 70.0, 3, 2, 5]                   # the table's last row
    if n > 1:
        M[n - 1, cols] = [255.999, np.nan, -0.0, np.nan, -0.0, np.nextafter(20.0, np.inf)]
    got = _decode_device(M, cols, table)
    assert got["rsi_row"][0] == table[255]
    _assert_decoded(got, M, cols, table)
    if n >= 128:
        # every edge of each gene appears, and every period of the table decodes to its row
        for c, e in zip(cols, edges):
            assert len(np.unique(M[:, c].view(np.uint64))) >= len(e) - 1
        P = np.tile(M[:1], (256, 1))
        P[:, cols[0]] = np.arange(256) + rng.uniform(0, 1, 256) * (np.arange(256) % 2)
        dec = _decode_device(P, cols, table)
        np.testing.assert_array_equal(dec["rsi_row"], table)


def test_decode_periods_and_table_size(torch_cuda):
    """Truncation (14.999 -> 14, -0.5 -> period 0), periods 256 and 1e9 outside a full table, absent gene columns
    (decode_population's defaults), and n_period_row = 257 refused with ELIMIT."""
    import torch
    from ai_crypto_trader_b200 import _lib
    table = _period_table(np.random.default_rng(1))
    cols = [0, 1, 2, 3, 4, 5]
    M = np.array([[14.999, 30, 70, 3, 2, 5], [-0.5, 30, 70, 3, 2, 5], [256, 30, 70, 3, 2, 5], [1e9, 30, 70, 3, 2, 5],
                  [255, 30, 70, 3, 2, 5], [0.999, 30, 70, 3, 2, 5]], dtype=np.float64)
    got = _decode_device(M, cols, table)
    assert got["rsi_row"].tolist() == [table[14], table[0], -1, -1, table[255], table[0]]
    _assert_decoded(got, M, cols, table)
    # absent genes: only the period column present
    got = _decode_device(M[:, :1], [0, -1, -1, -1, -1, -1], table)
    _assert_decoded(got, M[:, :1], [0, -1, -1, -1, -1, -1], table)
    # a short table: a period past its end decodes to -1
    got = _decode_device(M, cols, table[:15])
    assert got["rsi_row"].tolist() == [table[14], table[0], -1, -1, -1, table[0]]
    dev = torch.zeros(6, dtype=torch.float64, device="cuda")
    out = torch.zeros(C.sizeof(_lib.Individual), dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.B200btError) as e:
        _lib.call("b200bt_decode_individuals", dev.data_ptr(), 6, 1, (C.c_int * 6)(*cols), (C.c_int32 * 257)(*range(257)),
                  257, out.data_ptr(), _lib.current_stream())
    assert e.value.status == ELIMIT
