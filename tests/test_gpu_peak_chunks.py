"""Max drawdown of the time-chunked sweeps: a chunk below the equity peak it inherits takes its drawdown from three
per-chunk sums, only a chunk that sets a new peak is replayed record by record (chunk_peak_kernel).  Lanes built to hit
each case -- a lane that sets a new peak in nearly every chunk, a lane whose first record lies in a later chunk (E0 = P0 =
initial capital) after chunks without records, a lane whose equity never moves (E0 + largest prefix == P0 in every chunk)
-- against the fused kernel and the C oracle, through both time-chunked schedules."""
import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

N = 140_000
QUIET = 30_000          # constant price before this bar: RSI stays at 100, the long-only lanes do not trade


def _close():
    """Symbol 0: flat, then a 10-bar sawtooth 100 -> 95 -> 100 on which a long entry below RSI 35 meets a 1 % take profit
    on the way up every cycle (every exit a win: the equity sets a new peak in every chunk it trades in).  Symbol 1: the
    synthetic market."""
    from ai_crypto_trader_b200 import synth
    t = np.arange(N)
    saw = np.array([100, 99, 98, 97, 96, 95, 96, 97, 98, 99], dtype=np.float64)[t % 10]
    return np.stack([np.where(t < QUIET, 100.0, saw), synth.synth_symbol(1, N)["close"]]).astype(np.float32)


def _population():
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(30, seed=11)
    winner = dict(pop[0], rsi_period=5, rsi_oversold=35, rsi_overbought=101, take_profit=1, stop_loss=5)
    flat = dict(winner, max_position_size=0)          # no fees, no PnL: every chunk's equity ties its inherited peak
    return [winner, flat] + pop


def _check_vs_oracle(sweep, population, close):
    from ai_crypto_trader_b200 import synth
    from oracle import indicators_ref, sim_oracle
    bank = np.stack([indicators_ref.rsi_bank(close[s], sweep.periods) for s in range(close.shape[0])])
    want, _, _ = sim_oracle.population(close, bank, sweep.period_row, population,
                                       sim_oracle.config_of(synth.EPOCH_2024_MINUTES, 1))
    sim_oracle.assert_lanes(sweep.lane_stats(), want, "lanes")


@pytest.mark.parametrize("mode,opts", [
    ("tiled", dict(warm=2048, chunks=6)),
    ("tiled", dict(warm=0, chunks=12, max_repair_rounds=64)),            # wrong boundaries: the overlapped repair and the fix-up pass
    ("tiled", dict(warm=2048, chunks=6, pool_blocks=8)),                 # full pool: flagged lanes re-run by the fused kernel
    ("chunked", dict(target_events=300, warm=1024, max_chunks=64)),
    ("chunked", dict(target_events=300, warm=0, max_chunks=64, max_repair_rounds=64)),
])
def test_chunk_drawdown_matches_fused_and_oracle(torch_cuda, mode, opts):
    torch = torch_cuda
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    close = _close()
    market = MarketData.from_close(torch.from_numpy(close).cuda())
    population = _population()
    sweep = PopulationSweep(market, mode=mode, chunk_options=opts)
    fused = PopulationSweep(market, mode="fused")
    f = sweep.evaluate(population)
    peaks, invalid = sweep.last_peak_chunks, sweep.last_invalid_lanes
    f_f = fused.evaluate(population)
    plan = sweep.plan_tiles(population, **opts) if mode == "tiled" else sweep.plan_chunks(population, **opts)
    k_winner = plan.K if mode == "tiled" else int(plan.n_chunks[0])
    assert k_winner >= 6
    if "pool_blocks" in opts:
        assert sweep.last_pool_overflow and invalid > 0 and peaks >= 0
    else:
        # the winner's lane on symbol 0 sets a new peak in every chunk it trades in (all but the quiet first one or two)
        assert peaks >= k_winner // 2, (peaks, k_winner)
    np.testing.assert_array_equal(sweep.lane_stats()["trade_hash"], fused.lane_stats()["trade_hash"])
    np.testing.assert_array_equal(sweep.lane_stats()["n_records"], fused.lane_stats()["n_records"])
    np.testing.assert_allclose(sweep.lane_stats()["max_drawdown"], fused.lane_stats()["max_drawdown"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(f, f_f, rtol=1e-9, atol=1e-11, equal_nan=True)
    _check_vs_oracle(sweep, population, close)
    st = sweep.lane_stats()
    assert st["n_records"][0, 0] > 0 and st["n_wins"][0, 0] == st["n_records"][0, 0] // 2      # the winner wins every trade
    assert st["max_drawdown"][1, 0] == 0.0 and st["net_profit"][1, 0] == 0.0                     # the flat lane
