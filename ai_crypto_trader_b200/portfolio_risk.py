"""Portfolio risk numerics on the GPU engine (SURVEY 8-f4).

Reference: services/portfolio_risk_service.py (class PortfolioRiskService)
  calculate_var                :217-246   historical VaR        -> exact order statistics (b200bt_select)
  calculate_conditional_var    :248-284   expected shortfall    -> b200bt_tail_stats
  calculate_asset_correlation  :286-326   returns.corr()        -> b200bt_correlation
  calculate_portfolio_var      :328-396   diversification formula (host; S x S is tiny)
Kept: method names, argument meaning, the "log and return 0.0 / fallback" error convention.  Out of scope: the
Redis / Binance plumbing around them.  Returns are fp32 device rows (float64 arithmetic inside the kernels), so
VaR / CVaR agree with the float64 reference to ~1e-6 relative, the correlation to ~1e-7 absolute.
"""
from __future__ import annotations

import logging
from functools import partial
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .monte_carlo import PathEngine, _lerp, percentile_points

logger = logging.getLogger("b200bt.portfolio_risk")


class ReturnBank:
    """Device-resident simple returns of S assets: fp32 [S][N], NaN where undefined (bar 0, missing data)."""

    def __init__(self, symbols: Sequence[str], returns: torch.Tensor):
        if not (returns.dim() == 2 and returns.dtype == torch.float32 and returns.is_cuda and len(symbols) == returns.shape[0]):
            raise ValueError(f"returns must be a device float32 tensor with one row per symbol ({len(symbols)})")
        self.symbols = list(symbols)
        self.returns = returns.contiguous()
        self.row = {s: i for i, s in enumerate(self.symbols)}

    @classmethod
    def from_close(cls, symbols: Sequence[str], close, device=None) -> "ReturnBank":
        """close: [S][N] host array or device tensor (fp32 values) -> pct_change rows (:208)."""
        dev = torch.device(device or "cuda")
        c = close if isinstance(close, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(close, dtype=np.float32))
        c = c.to(dev, dtype=torch.float32).contiguous()
        out = torch.empty_like(c)
        S, N = c.shape
        with torch.cuda.device(dev):
            _lib.call("b200bt_pct_change", c.data_ptr(), _lib.ld(c), S, N, out.data_ptr(), _lib.ld(out), _lib.current_stream())
        return cls(symbols, out)


class PortfolioRiskService:
    """Compute surface of the reference's PortfolioRiskService on device return rows."""

    def __init__(self, bank: Optional[ReturnBank] = None, risk_config: Optional[Dict] = None, device=None):
        self.bank = bank
        self.device = torch.device(device or (bank.returns.device if bank is not None else "cuda"))
        self.risk_config = risk_config or {}
        self.asset_correlations: Dict[str, Dict[str, float]] = {}
        self._engine = PathEngine(self.device)
        self._ws: Optional[torch.Tensor] = None

    # -- helpers ------------------------------------------------------------------------------------
    def _as_device(self, returns) -> torch.Tensor:
        if isinstance(returns, str):
            returns = self.bank.returns[self.bank.row[returns]]
        if isinstance(returns, torch.Tensor):
            x = returns.to(self.device, dtype=torch.float32)
        else:
            x = torch.from_numpy(np.ascontiguousarray(np.asarray(returns, dtype=np.float32))).to(self.device)
        x = x.contiguous()
        return x[~torch.isnan(x)] if bool(torch.isnan(x).any()) else x       # returns.dropna() (:232,:264)

    def _workspace(self, need: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=self.device)
        return self._ws

    def _percentile(self, x: torch.Tensor, q: float) -> float:
        [(lo, hi, g)] = percentile_points(partial(self._engine.select, x), int(x.numel()), [q])
        return _lerp(lo, hi, g)

    def _tail(self, x: torch.Tensor, threshold: float) -> np.ndarray:
        n = int(x.numel())
        need = int(_lib.load().b200bt_tail_stats_workspace_bytes(n))
        ws = self._workspace(need)
        out = torch.empty(4, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("b200bt_tail_stats", x.data_ptr(), n, float(threshold), out.data_ptr(), ws.data_ptr(), need,
                      _lib.current_stream())
        return out.cpu().numpy()

    # -- reference surface ----------------------------------------------------------------------------
    def calculate_var(self, returns, confidence_level: float = 0.95, value: float = 1.0) -> float:
        try:
            x = self._as_device(returns)
            if x.numel() < 2:
                logger.warning("Not enough data points to calculate VaR")
                return 0.0
            return abs(self._percentile(x, 100 * (1 - confidence_level)) * value)
        except Exception as e:      # reference convention (:244-246)
            logger.error("Error calculating VaR: %s", e)
            return 0.0

    def calculate_conditional_var(self, returns, confidence_level: float = 0.95, value: float = 1.0) -> float:
        try:
            x = self._as_device(returns)
            if x.numel() < 2:
                logger.warning("Not enough data points to calculate CVaR")
                return 0.0
            q = self._percentile(x, 100 * (1 - confidence_level))
            t = self._tail(x, q)
            return abs(t[0] / t[1] * value)
        except Exception as e:
            logger.error("Error calculating CVaR: %s", e)
            return 0.0

    def correlation_matrix(self, rows: Optional[Sequence[int]] = None) -> np.ndarray:
        x = self.bank.returns if rows is None else self.bank.returns[list(rows)].contiguous()
        S, N = x.shape
        need = int(_lib.load().b200bt_correlation_workspace_bytes(S, N))
        ws = self._workspace(need)
        out = torch.empty((S, S), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("b200bt_correlation", x.data_ptr(), _lib.ld(x), S, N, out.data_ptr(), ws.data_ptr(), need,
                      _lib.current_stream())
        return out.cpu().numpy()

    def calculate_asset_correlation(self, symbols: List[str]) -> Dict[str, Dict[str, float]]:
        try:
            known = [s for s in symbols if self.bank is not None and s in self.bank.row]
            c = self.correlation_matrix([self.bank.row[s] for s in known]) if known else np.zeros((0, 0))
            pos = {s: i for i, s in enumerate(known)}
            return {a: {b: (float(c[pos[a], pos[b]]) if a in pos and b in pos else 0.0) for b in symbols} for a in symbols}
        except Exception as e:      # (:324-326)
            logger.error("Error calculating asset correlations: %s", e)
            return {a: {b: 0.0 for b in symbols} for a in symbols}

    def calculate_portfolio_var(self, holdings: Dict, var_estimates: Dict) -> float:
        try:
            assets = [a for a in holdings["assets"] if a in var_estimates and a != "USDC"]
            if not assets:
                return 0.0
            values = np.array([holdings["assets"][a]["value_usdc"] for a in assets], dtype=np.float64)
            total = values.sum()
            if total == 0:
                return 0.0
            w = values / total
            v = np.array([var_estimates[a] for a in assets], dtype=np.float64)
            c = np.array([[self.asset_correlations.get(a, {}).get(b, 0.0) for b in assets] for a in assets])
            if not np.all(np.linalg.eigvals(c) > 0):
                logger.warning("Correlation matrix is not positive definite, using identity matrix")
                c = np.eye(len(assets))
            return float(np.sqrt(w @ (np.outer(v, v) * c) @ w) * holdings["total_value"])
        except Exception as e:      # (:394-396)
            logger.error("Error calculating portfolio VaR: %s", e)
            return sum(var_estimates.get(a, 0) for a in holdings["assets"] if a != "USDC")
