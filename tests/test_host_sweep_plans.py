"""Event-pool learning of the population sweep (PopulationSweep._pool_options) and the flag read-out it shares with the
last_* diagnostics, on the host: the flags a sweep leaves in pinned memory are stood in for by CPU int32[5] rows."""
import types

import numpy as np
import pytest
import torch

from ai_crypto_trader_b200 import sweep as sw
from ai_crypto_trader_b200 import synth

S = 2


class _Stream:
    syncs = 0

    def synchronize(self):
        _Stream.syncs += 1


@pytest.fixture
def host_sweep(monkeypatch):
    """A PopulationSweep over a placeholder bank on the CPU; stream synchronisations are counted."""
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
    monkeypatch.setattr(sw, "_flag_slot", lambda: torch.zeros(5, dtype=torch.int32))
    monkeypatch.setattr(sw, "_sm_count", lambda device: 132)
    _Stream.syncs = 0
    market = types.SimpleNamespace(S=S, N=200_000, device=torch.device("cpu"), minute0=synth.EPOCH_2024_MINUTES, bar_minutes=1)
    sweep = sw.PopulationSweep.__new__(sw.PopulationSweep)
    sweep._setup(market, list(range(5, 31)), None, 10000.0, 0, "tiled", dict(warm=2048, chunks=6), False, (),
                 bank=torch.empty(0))
    return sweep


def _swept(n_seg, pred_blocks, overflow=0, used=0, invalid=0, stalls=0, peaks=0):
    """A plan as the flag read-out sees it after its sweep: `used` pool blocks beyond the 2 * n_seg * S floor."""
    flags = torch.tensor([overflow, invalid, 2 * n_seg * S + used, stalls, peaks], dtype=torch.int32)
    return types.SimpleNamespace(n_seg=n_seg, pred_blocks=pred_blocks, overflow=flags)


def test_pool_factor_follows_use_and_quadruples_after_an_overflow(host_sweep):
    opts = {"pool_blocks": 77}
    host_sweep._pool_options(opts)                        # nothing swept yet: no synchronisation, the model as is
    assert opts == {"pool_blocks": 77} and host_sweep._pool_factor == 1.0 and _Stream.syncs == 0

    host_sweep._last_plans = [_swept(10, 100.0, used=500), _swept(20, 150.0, used=250)]
    opts = {}
    host_sweep._pool_options(opts)                        # 750 blocks used for 250 predicted
    assert _Stream.syncs == 1
    learnt = host_sweep._pool_factor
    assert learnt == max(1.0, 1.2 * 750 / 250.0) and learnt > 3
    assert opts == {"pool_scale": learnt * 1.5}

    host_sweep._last_plans = [_swept(10, 100.0, used=10), _swept(20, 150.0, overflow=1, used=3)]
    opts = {"pool_blocks": 77, "pool_scale": 2.0}
    host_sweep._pool_options(opts)                        # an overflow: x4, and a fixed pool size no longer holds
    assert host_sweep._pool_factor == 4.0 * learnt
    assert opts == {"pool_scale": 4.0 * learnt * 2.0}

    host_sweep._last_plans = [_swept(10, 100.0, used=20)]
    opts = {}
    host_sweep._pool_options(opts)                        # fewer blocks than predicted: never below the model
    assert host_sweep._pool_factor == 1.0 and opts == {}

    host_sweep._last_plans = [_swept(10, 0.0, used=20)]
    host_sweep._pool_factor = 2.0
    host_sweep._pool_options({})                          # nothing predicted: keep what was learnt
    assert host_sweep._pool_factor == 2.0


def test_last_flags_sum_over_the_slices(host_sweep):
    host_sweep._last_plans = [_swept(4, 1.0, invalid=3, stalls=1, peaks=7), _swept(4, 1.0, overflow=1, invalid=2, peaks=5)]
    assert host_sweep.last_invalid_lanes == 5 and host_sweep.last_scan_stalls == 1 and host_sweep.last_peak_chunks == 12
    assert host_sweep.last_pool_overflow is True
    host_sweep._last_plans = [_swept(4, 1.0), _swept(4, 1.0)]
    assert host_sweep.last_pool_overflow is False and host_sweep.last_invalid_lanes == 0
    assert _Stream.syncs == 6                             # every read-out waits for the stream


def test_next_plan_pool_grows_by_the_learnt_factor(host_sweep, native_lib):
    pop = synth.random_population(64, seed=4)
    first = host_sweep.plan(pop)
    assert len(first) == 1 and type(first[0]).__name__ == "TilePlan" and first[0].workspace.numel() >= first[0].ws_bytes
    p = first[0]
    used = int(2 * p.pred_blocks)
    p.overflow[2] = 2 * p.n_seg * S + used
    host_sweep._last_plans = first
    again = host_sweep.plan(pop)[0]
    factor = 1.2 * used / p.pred_blocks
    assert host_sweep._pool_factor == factor
    assert again.pool_blocks == int(factor * 1.5 * again.pred_blocks) + 2 * again.n_seg * S + 1024
    assert again.pool_blocks > p.pool_blocks and np.array_equal(again.slots, p.slots)
