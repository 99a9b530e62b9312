"""The multi-timeframe RSI bank on every bar clock (BASELINE configs[3]: PopulationSweep(timeframes=...), gene
`rsi_timeframe`), built as b200bt_resample -> b200bt_rsi_bank -> b200bt_align, against independent statements:

1. b200bt_resample against pandas' resample(f"{k}min", origin="epoch") by bar start (first / max / min / last bit-equal,
   volume within 1 ulp of the exact sum rounded to fp32), and b200bt_align against searchsorted on pandas' bucket ends,
   over the grid of tests/test_oracle_indicators.py: bar clocks 1 / 3 / 5 / 7, k = bar x {1, 2, 3, 12}, daily buckets, a k
   that does not divide 1440, first bars off both grids, N from one bar to a few thousand; and one 262 147-bar series.
2. The bank of PopulationSweep(timeframes=...) on a 5-minute clock (5, 15, 60, 1440; the daily block's NaN head covers
   more than two 128-bar tiles of the scan) and on a 7-minute clock (7, 14, 56) starting off the 7-minute grid, against
   oracle/indicators_ref.rsi_rows_on_timeframe; its lanes against the C oracle fed those rows, through the fused, chunked
   and thread-per-lane schedules (the last one swept twice, so that its zone map is built and used).
3. The zone map (b200bt_zone_map, and the rows b200bt_rsi_bank_zones writes with a bank) against a NumPy restatement of
   the layout in csrc/common.cuh, on a single-clock bank and on the NaN-headed multi-timeframe bank.
4. A MarketData built from pinned memory whose close copies arrive late: resample and multi_timeframe_indicators wait
   for them.
5. set_gap refuses a gap on a multi-timeframe sweep."""
import math
import warnings
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest

from gpu_fixtures import torch_cuda
from test_oracle_indicators import DAY0, grid_cases

pytestmark = pytest.mark.gpu

S = 3
SCHEDULES = {
    "fused": dict(mode="fused"),
    "chunked": dict(mode="chunked", chunk_options=dict(target_events=300, max_chunks=64, warm=256, pool_scale=4.0)),
    "tiled": dict(mode="tiled", chunk_options=dict(chunks=16, warm=1024, pool_scale=4.0)),
}


# -- 1. resample and align -----------------------------------------------------------------------------------------------
def pandas_bars(ohlcv, minute0, bar, k):
    """pandas' epoch-aligned k-minute bars of ohlcv [5][S][n] -> ([5][S][M] float32, bucket end minutes [M]).  Volume:
    math.fsum of the bucket rounded once to fp32."""
    _, n_sym, n = ohlcv.shape
    start = minute0 + np.arange(n, dtype=np.int64) * bar
    frame = pd.DataFrame(ohlcv.reshape(5 * n_sym, n).T, index=pd.to_datetime(start * 60, unit="s"))
    r = frame.resample(f"{k}min", origin="epoch")
    aggs = (r.first(), r.max(), r.min(), r.last())
    begins = aggs[3].index.values.astype("datetime64[m]").astype(np.int64)
    out = np.empty((5, n_sym, len(begins)), dtype=np.float32)
    for f, agg in enumerate(aggs):
        out[f] = agg.to_numpy(dtype=np.float32)[:, f * n_sym:(f + 1) * n_sym].T
    cuts = np.flatnonzero(np.diff(np.searchsorted(begins, start, side="right"))) + 1
    for s in range(n_sym):
        out[4, s] = [math.fsum(g) for g in np.split(ohlcv[4, s].astype(np.float64), cuts)]
    return out, begins + k


def _check_resample_and_align(torch, ohlcv, minute0, bar, k):
    from ai_crypto_trader_b200 import _lib, indicators as ind
    from ai_crypto_trader_b200.sweep import MarketData
    n = ohlcv.shape[2]
    where = (bar, k, minute0 - DAY0, n)
    want, ends = pandas_bars(ohlcv, minute0, bar, k)
    M = want.shape[2]
    market = MarketData(ohlcv, minute0=minute0, bar_minutes=bar)
    hi = ind.resample(market, k)
    assert (hi.N, hi.minute0, hi.bar_minutes) == (M, int(ends[0]) - k, k), where
    got = hi.ohlcv.cpu().numpy()
    assert np.array_equal(got[:4].view(np.uint32), want[:4].view(np.uint32)), where
    assert (np.abs(got[4] - want[4]) <= np.spacing(np.abs(want[4]))).all(), where
    # align: a distinct value per higher-timeframe bar, so that any other bucket shows
    src = (np.arange(M)[None, :] + 1 + 1_000_003 * np.arange(S)[:, None]).astype(np.float32)
    al = ind.align_to_base(torch.from_numpy(src).cuda(), SimpleNamespace(N=n, minute0=minute0, bar_minutes=bar), k)
    j = np.searchsorted(ends, minute0 + (np.arange(n, dtype=np.int64) + 1) * bar, side="right") - 1
    ref = np.where(j >= 0, src[:, np.maximum(j, 0)], np.float32(np.nan)).astype(np.float32)
    assert np.array_equal(al.cpu().numpy(), ref, equal_nan=True), where
    assert int(_lib.load().b200bt_resample_bars(n, minute0, bar, k)) == M
    return M == 1, bool(j[0] < 0), bool(j[-1] < M - 1)


@pytest.mark.parametrize("bar", [1, 3, 5, 7])
def test_resample_and_align_on_the_grid(torch_cuda, bar):
    from ai_crypto_trader_b200 import synth
    cases = [c for c in grid_cases() if c[0] == bar]
    data = synth.synth_ohlcv(S, max(n for *_, n in cases), first_symbol=10 + bar)
    seen = np.zeros(3, dtype=bool)
    for _, k, minute0, n in cases:
        seen |= _check_resample_and_align(torch_cuda, data[:, :, :n], minute0, bar, k)
    assert seen.all()            # M = 1, bars before the first completed bucket, bars after the last one


@pytest.mark.parametrize("bar,k,offset", [(1, 1440, 1439), (1, 7, 3), (5, 60, 1)])
def test_resample_and_align_long_series(torch_cuda, bar, k, offset):
    from ai_crypto_trader_b200 import synth
    data = synth.synth_ohlcv(S, 262_147, first_symbol=20)
    _check_resample_and_align(torch_cuda, data, DAY0 + offset, bar, k)


# -- 2. the bank and its lanes -------------------------------------------------------------------------------------------
BANK_CASES = {
    # minute0 = 00:05: the daily block is NaN until the bar closing at midnight, 286 five-minute bars (> 2 tiles of 128)
    "5min": dict(bar=5, timeframes=(5, 15, 60, 1440), minute0=DAY0 + 5, n=60_001, daily_head=286),
    "7min": dict(bar=7, timeframes=(7, 14, 56), minute0=DAY0 + 3, n=45_001, daily_head=None),
}
PERIODS = (5, 9, 14, 21, 30)
DENSE_AFTER_HEAD = dict(rsi_oversold=99, rsi_overbought=101, take_profit=0.05, stop_loss=0.05)


def _population(n_tf, pop=120, seed=31):
    import random
    from ai_crypto_trader_b200 import synth
    population = synth.random_population(pop, seed=seed)
    rnd = random.Random(seed)
    for p in population:
        p["rsi_period"] = rnd.choice(PERIODS)
        p["rsi_timeframe"] = rnd.randrange(n_tf)
    last = n_tf - 1
    for i, period in enumerate(PERIODS):           # every period of the top block fires on its first defined bar
        population[i].update(DENSE_AFTER_HEAD, rsi_period=period, rsi_timeframe=last)
    population[len(PERIODS)].update(rsi_oversold=35, rsi_overbought=65, rsi_period=5, take_profit=1, stop_loss=1,
                                    rsi_timeframe=last)
    for t in range(n_tf):
        population[len(PERIODS) + 1 + t].update(DENSE_AFTER_HEAD, rsi_period=14, rsi_timeframe=t)
    return population


@pytest.fixture(scope="module", params=sorted(BANK_CASES))
def mtf(request, torch_cuda):
    """One multi-timeframe case: data, oracle rows per (symbol, block) and the oracle lanes."""
    from ai_crypto_trader_b200 import synth
    from oracle import indicators_ref, sim_oracle
    c = SimpleNamespace(name=request.param, **BANK_CASES[request.param])
    c.S = 2
    c.ohlcv = synth.synth_ohlcv(c.S, c.n, first_symbol=30)
    c.rows = np.empty((c.S, len(c.timeframes) * len(PERIODS), c.n), dtype=np.float32)
    P = len(PERIODS)
    for s in range(c.S):
        c.rows[s, :P] = indicators_ref.rsi_bank(c.ohlcv[3, s], PERIODS)
        for i, k in enumerate(c.timeframes[1:], start=1):
            c.rows[s, i * P:(i + 1) * P] = indicators_ref.rsi_rows_on_timeframe(c.ohlcv[3, s], c.minute0, k, PERIODS,
                                                                                bar_minutes=c.bar)
    c.population = _population(len(c.timeframes))
    row_of = lambda p: p["rsi_timeframe"] * P + PERIODS.index(p["rsi_period"])
    c.want, _, _ = sim_oracle.population(c.ohlcv[3], c.rows, row_of, c.population, sim_oracle.config_of(c.minute0, c.bar))
    return c


def _market(c):
    from ai_crypto_trader_b200.sweep import MarketData
    return MarketData(c.ohlcv, minute0=c.minute0, bar_minutes=c.bar)


def test_multi_timeframe_bank_rows(mtf):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    c = mtf
    sweep = PopulationSweep(_market(c), rsi_periods=PERIODS, timeframes=c.timeframes, mode="fused")
    bank = sweep.bank.cpu().numpy()
    assert bank.shape == c.rows.shape
    P = len(PERIODS)
    for s in range(c.S):
        for i, k in enumerate(c.timeframes):
            got, ref = bank[s, i * P:(i + 1) * P], c.rows[s, i * P:(i + 1) * P]
            assert np.array_equal(np.isnan(got), np.isnan(ref)), (c.name, s, k)
            neq = (got != ref) & ~np.isnan(ref)
            assert int(neq.sum()) <= max(2, int(2e-6 * ref.size)), (c.name, s, k, int(neq.sum()))   # double-rounding ties
    if c.daily_head is not None:
        head = np.isnan(bank[:, -P:]).all(axis=(0, 1))
        assert head[:c.daily_head].all() and not head[c.daily_head:].any()
        assert c.daily_head > 2 * 128


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
def test_multi_timeframe_lanes_against_the_c_oracle(mtf, schedule):
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    c = mtf
    opt = SCHEDULES[schedule]
    sweep = PopulationSweep(_market(c), rsi_periods=PERIODS, timeframes=c.timeframes, mode=opt["mode"],
                            chunk_options=opt.get("chunk_options"))
    zones_passed = []
    amortised = sweep._zones_if_amortised

    def spy():
        z = amortised()
        zones_passed.append(z is not None)
        return z
    sweep._zones_if_amortised = spy
    for _ in range(2 if schedule == "tiled" else 1):
        fit = sweep.evaluate(c.population)
    sim_oracle.assert_lanes(sweep.lane_stats(), c.want, f"{c.name} {schedule}")
    np.testing.assert_allclose(fit, c.want["score"].mean(axis=1), rtol=1e-9, atol=1e-11, equal_nan=True)
    plans = sweep._last_plans
    if schedule == "fused":
        assert not plans
    elif schedule == "chunked":
        assert len(plans) == 1 and int(plans[0].n_chunks.max()) >= 8, plans
        assert sweep.last_invalid_lanes < len(c.population) * c.S
    else:
        assert len(plans) == 1 and plans[0].K == 16
        assert zones_passed == [False, True] and sweep._zones is not None      # built on the second sweep and used
        assert sweep.last_invalid_lanes == 0
    # the lanes that buy on the top block's first defined bar trade
    top = [i for i, p in enumerate(c.population) if p["rsi_timeframe"] == len(c.timeframes) - 1]
    assert (c.want["n_records"][top[:len(PERIODS)]] > 0).all()


def test_set_gap_is_refused_on_a_multi_timeframe_sweep(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(1, 3000), minute0=DAY0 + 2, bar_minutes=1)
    multi = PopulationSweep(market, rsi_periods=(14,), timeframes=(1, 5))
    with pytest.raises(ValueError, match="gap"):
        multi.set_gap(1000, 1440)
    multi.set_gap(0, 0)                                   # no gap: nothing to refuse
    single = PopulationSweep(market, rsi_periods=(14,))
    single.set_gap(1000, 1440)
    assert (single.cfg.gap_bar, single.cfg.gap_minutes) == (1000, 1440)


# -- 3. zone map ---------------------------------------------------------------------------------------------------------
def zone_map_ref(price, bank):
    """The layout of csrc/common.cuh restated: coarse (min, max) per 32-bar block [S][P + 1][stride] then fine per 4-bar
    group [S][P + 1][fine_stride], row 0 = price, NaNs ignored, all-NaN groups and padding (NaN, NaN).  stride =
    ceil(N / 32) rounded up to even, fine_stride = 32 groups per started 128-bar tile."""
    n_sym, P, n = bank.shape
    rows = np.concatenate([price[:, None, :], bank], axis=1)
    stride = -(-n // 32) + (-(-n // 32)) % 2
    fine_stride = -(-n // 128) * 32

    def ranges(width, count):
        pad = np.full((n_sym, P + 1, count * width), np.nan, dtype=np.float32)
        pad[:, :, :n] = rows
        g = pad.reshape(n_sym, P + 1, count, width)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)      # all-NaN groups
            return np.stack([np.nanmin(g, axis=-1), np.nanmax(g, axis=-1)], axis=-1)
    return np.concatenate([ranges(32, stride).ravel(), ranges(4, fine_stride).ravel()])


def _same_zones(got, want, where):
    assert got.shape == want.shape, where
    assert np.array_equal(np.isnan(got), np.isnan(want)), (where, np.flatnonzero(np.isnan(got) != np.isnan(want))[:8])
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok], want[ok]), (where, np.flatnonzero(got[ok] != want[ok])[:8])


@pytest.mark.parametrize("n_bars", [5, 127, 4096, 70_001, 262_177])
def test_zone_map_against_the_layout(torch_cuda, n_bars):
    torch = torch_cuda
    from ai_crypto_trader_b200 import _lib, synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    ohlcv = synth.synth_ohlcv(3, n_bars, first_symbol=40)
    # single clock from a pinned source: the bank's zone rows come out of b200bt_rsi_bank_zones, one call per symbol
    single = PopulationSweep(MarketData(torch.from_numpy(ohlcv).pin_memory()), rsi_periods=(2, 5, 14, 30))
    # 5-minute clock with a daily block: whole blocks and groups of NaN at the head of the aligned rows
    multi = PopulationSweep(MarketData(ohlcv[:, :2], minute0=DAY0 + 5, bar_minutes=5), rsi_periods=(5, 14),
                            timeframes=(5, 60, 1440))
    for name, sweep in (("single", single), ("multi", multi)):
        m = sweep.market
        want = zone_map_ref(m.close.cpu().numpy(), sweep.bank.cpu().numpy())
        assert int(_lib.load().b200bt_zone_map_floats(sweep.bank.shape[1], m.S, m.N)) == want.size
        if name == "single":
            _same_zones(sweep._zones.cpu().numpy(), want, (name, "rsi_bank_zones", n_bars))
            sweep._zones = None
        else:
            assert sweep._zones is None
            if n_bars > 288:
                assert np.isnan(sweep.bank[:, -2:, :256].cpu().numpy()).all()
        _same_zones(sweep.zone_map().cpu().numpy(), want, (name, "zone_map", n_bars))


# -- 4. pinned source ----------------------------------------------------------------------------------------------------
def test_pinned_source_resample_waits_for_the_close_copies(torch_cuda):
    """MarketData from pinned memory uploads the close prices in quarter copies on side streams.  resample() reads the
    whole [5][S][N] array on the current stream: it must wait for those copies.  The copy streams are held back by a
    ~10 ms device sleep queued before the copies, so a resample that does not wait reads the close row before it lands.

    On the H100 the deferred open / high / low / volume copies that reading `ohlcv` issues happen to be executed after
    the held-back close copies, which orders a resample behind them even without the join; CUDA promises no such order,
    so the test also asserts that reading `ohlcv` (and materialise()) joined the close copies.

    The pageable reference runs first: it leaves every buffer the late runs allocate in the caching allocator, so no
    cudaMalloc (an implicit synchronisation of all streams) falls between the copies and the kernels that read them.  The
    late market's buffer is then refilled with NaN, and the data has its own seed: a read that overtakes the copies cannot
    match by chance."""
    torch = torch_cuda
    from ai_crypto_trader_b200 import indicators as ind, synth
    from ai_crypto_trader_b200.sweep import MarketData, _copy_stream
    n_sym, N, k = 4, 40_000, 15
    ohlcv = synth.synth_ohlcv(n_sym, N, seed_base=7_771)
    dev = torch.device("cuda", 0)
    ref = MarketData(ohlcv, minute0=DAY0 + 7)
    want_bars = ind.resample(ref, k).ohlcv.cpu()
    want_mtf = ind.multi_timeframe_indicators(ref)
    del ref
    host = torch.from_numpy(ohlcv).pin_memory()          # (page-locking synchronises too: done before the copies)

    def late_market():
        stale = torch.full((5, n_sym, N), float("nan"), dtype=torch.float32, device=dev)
        del stale                                         # (the caching allocator hands this block out next)
        torch.cuda.synchronize()
        for i in range(1, 5):
            with torch.cuda.stream(_copy_stream(dev, i)):
                torch.cuda._sleep(20_000_000)
        market = MarketData(host, minute0=DAY0 + 7)
        assert market._close_parts                        # the close rows are still in flight
        return market

    late = late_market()
    got_bars = ind.resample(late, k).ohlcv.cpu()
    assert not late._close_parts                          # the current stream has joined every quarter copy
    del late
    late = late_market()
    got_mtf = ind.multi_timeframe_indicators(late)
    assert not late._close_parts
    del late
    torch.cuda.synchronize()
    assert torch.equal(got_bars, want_bars)
    assert got_mtf == want_mtf, {key: (got_mtf[key], want_mtf[key]) for key in want_mtf if got_mtf[key] != want_mtf[key]}
    whole = MarketData(host, minute0=DAY0 + 7).materialise()
    assert not whole._close_parts and whole._pending_host is None
