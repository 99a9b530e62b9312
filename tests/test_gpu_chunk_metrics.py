"""Trade metrics of the time-chunked sweep (chunk_partial_kernel) at the edges of its 128-record step, against the fused
sweep's record-by-record form.

The metrics pass walks a chunk's records 128 at a time, four per lane, and closes calendar days in the lane that holds
their last record.  Symbol 0 is built so that one lane's chunks hold 1, 127, 128, 129, 255, 256 and 257 records (step
and pool-block boundaries, odd counts), most chunks opening on an exit (a position carried in) and some on an entry.
Each chunk has a window of alternating prices in which a long lane with a 0.0001 % take-profit / stop-loss and an
oversold level of 99 records an event on every bar; outside the windows the price is constant and the lane holds its
position, or, where the window ends in a steady rise that lifts the RSI above 99, stays flat.  The calendar is varied
by the bar length: one bar per day (every record its own day, entries are negative days in every lane of a step), 1440
bars per day (a first chunk inside one day, days spanning several steps) and 7-minute bars."""
import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

K, CHUNK = 12, 1024               # tiled chunks: chunk c is bars [1024 c, 1024 (c + 1)) (group aligned)
N = K * CHUNK
STEP = 128                        # records per step of the metrics pass
# per chunk: length of the alternating window (-1: one down tick, then flat), and whether it ends in a rise (flat after)
WINDOW = [20, -1, 96, 97, 128, 224, 225, 256, 32, 169, 300, 61]
RISE = [1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 0]
EDGES = {1, 127, 128, 129, 255, 256, 257}
LONG = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)


def _close():
    from ai_crypto_trader_b200 import synth
    rng = np.random.default_rng(7)
    c = np.full(N, 100.0)
    for k, L in enumerate(WINDOW):
        a = k * CHUNK + 16
        level = c[k * CHUNK - 1] if k else 100.0
        if L < 0:
            c[a:] = level - 0.05
            continue
        t = np.arange(a, a + L)
        c[t] = 100.0 + np.where(t % 2 == 0, 0.5, -0.5) + rng.uniform(-0.2, 0.2, L)
        c[a + L:] = c[a + L - 1] + 0.05 * np.minimum(np.arange(1, N - a - L + 1), 40) if RISE[k] else 100.0
    return np.stack([c, synth.synth_symbol(2, N)["close"]]).astype(np.float32)


def _population():
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(40, seed=5)
    pop[0].update(LONG)
    pop[1].update(LONG, rsi_oversold=-1, rsi_overbought=1)     # the short mirror: trades wherever the price moves
    pop[2].update(LONG, take_profit=0.3, stop_loss=0.3)         # fewer, larger trades
    return pop


def _chunk_counts(events, n):
    bars = events[:n] & 0x3FFFFFFF
    return np.bincount(bars // CHUNK, minlength=K)


@pytest.mark.parametrize("bar_minutes", [1440, 1, 7])
@pytest.mark.parametrize("warm", [2048, 64])
def test_chunk_metrics_match_fused_at_step_edges(torch_cuda, bar_minutes, warm):
    torch = torch_cuda
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    close = _close()
    market = MarketData.from_close(torch.from_numpy(close).cuda(), minute0=0, bar_minutes=bar_minutes)
    population = _population()
    cap = N + 1
    tiled = PopulationSweep(market, event_cap=cap, mode="tiled", chunk_options=dict(chunks=K, warm=warm))
    fused = PopulationSweep(market, event_cap=cap, mode="fused")
    f_f = fused.evaluate(population)
    st_f, ev_f = fused.lane_stats(), fused.events()
    f_t = tiled.evaluate(population)
    st_t, ev_t = tiled.lane_stats(), tiled.events()
    assert tiled.plan(population)[0].K == K and tiled.last_invalid_lanes == 0

    # the shapes the lanes were built for
    n0 = int(st_f["n_records"][0, 0])
    ev0 = ev_f[0, 0, :n0]
    counts = _chunk_counts(ev0, n0)
    hist = {int(c): int((counts == c).sum()) for c in np.unique(counts)}
    print(f"records per chunk of the built lane (bar_minutes {bar_minutes}): {counts.tolist()}; histogram {hist}")
    assert EDGES <= set(hist), hist
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    first_is_exit = [bool(ev0[s] & 0x40000000) for s, c in zip(starts, counts) if c]
    assert any(first_is_exit) and not all(first_is_exit)
    day = (ev0 & 0x3FFFFFFF).astype(np.int64) * bar_minutes // 1440
    lane_in_step = np.concatenate([(np.arange(c) % STEP) // 4 for c in counts])
    last_of_step = np.concatenate([(np.arange(c) % STEP == STEP - 1) | (np.arange(c) == c - 1) for c in counts])
    if bar_minutes == 1440:
        # every record is a day of its own; entries (the fee alone) are negative days in the first and last lane of steps
        assert len(np.unique(day)) == n0
        entry = (ev0 & 0x40000000) == 0
        assert np.any(entry & (lane_in_step == 0) & ~last_of_step) and np.any(entry & (lane_in_step == 31) & ~last_of_step)
    if bar_minutes == 1:
        assert counts[0] > 0 and day[counts[0] - 1] == day[0]                   # a chunk inside one day
        chunk_of = (ev0 & 0x3FFFFFFF) // CHUNK
        per_day = np.unique(chunk_of.astype(np.int64) * 1_000_000 + day, return_counts=True)[1]
        assert per_day.max() > 2 * STEP                                          # a day across three steps of one chunk

    sim_oracle.assert_lanes(st_t, st_f, "tiled against fused")
    live = np.arange(cap)[None, None, :] < st_f["n_records"][:, :, None]
    np.testing.assert_array_equal(ev_t[live], ev_f[live])
    worst = 0.0
    for f in sim_oracle.CLOSE_FIELDS:
        a, b = np.asarray(st_t[f], dtype=np.float64), np.asarray(st_f[f], dtype=np.float64)
        both = np.isfinite(a) & np.isfinite(b)
        worst = max(worst, float(np.max(np.abs(a - b)[both] / np.maximum(np.abs(b[both]), 1e-300), initial=0.0)))
    np.testing.assert_allclose(f_t, f_f, rtol=1e-9, atol=1e-11, equal_nan=True)
    print(f"largest relative difference of a float64 statistic: {worst:.2e}")
    assert st_f["n_negative_days"][0, 0] > 0
