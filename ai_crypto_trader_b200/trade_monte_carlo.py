"""Trade-sequence Monte-Carlo of backtested strategies on the GPU.

The engine scores a strategy by what it earned on ONE history: one trade sequence per (individual, symbol) lane.  How much
of that lane's return and drawdown came from the order in which its trades happened to arrive is answered by resampling
the lane's own round trips many times and reading the spread of final equity and maximum drawdown (the reference's open
item "BACK-04: Add Monte Carlo simulations", BACKLOG.md:194).

  * round-trip PnL of a sweep's lanes: PopulationSweep.trade_pnl (kernel b200bt_trade_pnl, bit-identical to the pnl of
    StrategyEvaluationSystem._simulate_trades' records);
  * the paths: TradeMonteCarlo.simulate (kernel b200bt_trade_mc: bootstrap, block bootstrap or keyed shuffle of the
    round trips, float64 equity walk in calculate_metrics' record order, strategy_evaluation.py:119-139);
  * the statistics: monte_carlo.risk_statistics (the statistics block of run_monte_carlo_simulation,
    monte_carlo_service.py:305-336) on one lane with equity for price and mdd_percentiles=(95,), and
    monte_carlo.statistics_blocks(..., "equity") for the result blocks.

StrategyEvaluationSystem.monte_carlo_trades / monte_carlo_population are the user-facing calls.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from .monte_carlo import PathEngine


def _host(x, dtype) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x).reshape(-1), dtype=dtype)


class TradeMonteCarlo:
    """Monte-Carlo over the round trips of backtested lanes (one instance per GPU)."""

    def __init__(self, device: Optional[torch.device] = None):
        self.engine = PathEngine(device)
        self.device = self.engine.device

    def simulate(self, trip_pnl: torch.Tensor, n_trips, fee, n_paths: int, method: str = "bootstrap",
                 block_len: int = 1, initial_capital: float = 10000.0, seed: int = 2024, path_offset: int = 0,
                 lane_ids=None):
        """trip_pnl: device float64 [..., T_max], one row per lane (e.g. [pop][S][T_max] from PopulationSweep.trade_pnl);
        n_trips, fee (and lane_ids, the Philox lane id of every row, default the row index): one entry per lane, host or
        device.  -> (finals, maxdd): device fp32 [L][n_paths], final equity and maximum drawdown of every path."""
        if method not in _lib.TRADE_MC_METHODS:
            raise ValueError(f"unknown simulation method {method!r} (one of {sorted(_lib.TRADE_MC_METHODS)})")
        trips = trip_pnl.reshape(-1, trip_pnl.shape[-1])
        if trips.dtype != torch.float64 or not trips.is_cuda or trips.stride(-1) != 1:
            raise ValueError("trip_pnl must be a device float64 tensor with unit stride in its last axis")
        L = int(trips.shape[0])
        nt, fe = _host(n_trips, np.int32), _host(fee, np.float64)
        ids = None if lane_ids is None else _host(lane_ids, np.uint32)
        if len(nt) != L or len(fe) != L or (ids is not None and len(ids) != L):
            raise ValueError(f"{L} lanes of trip PnL, but {len(nt)} trip counts and {len(fe)} fees")
        finals = torch.empty((L, int(n_paths)), dtype=torch.float32, device=self.device)
        maxdd = torch.empty_like(finals)
        with torch.cuda.device(self.device):
            _lib.call("b200bt_trade_mc", trips.data_ptr(), _lib.ld(trips), nt.ctypes.data_as(C.POINTER(C.c_int32)),
                      fe.ctypes.data_as(C.POINTER(C.c_double)),
                      None if ids is None else ids.ctypes.data_as(C.POINTER(C.c_uint32)), L,
                      _lib.TRADE_MC_METHODS[method], int(block_len), float(initial_capital), int(n_paths),
                      int(seed) & (2**64 - 1), int(path_offset), finals.data_ptr(), maxdd.data_ptr(),
                      _lib.current_stream())
        return finals, maxdd
