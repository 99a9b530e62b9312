"""Backtest overfitting of a searched population: how much of the best backtest's performance is the search itself.

Host side of `b200bt_cscv` (include/b200bt.h):

* `cscv(pnl, n_blocks)` -- the Probability of Backtest Overfitting by combinatorially symmetric cross-validation
  (Bailey, Borwein, Lopez de Prado, Zhu 2015, "The Probability of Backtest Overfitting").  The kernel gives, for every
  split of the B time blocks into two halves, the in-sample winner and the integer rank counts of its out-of-sample
  Sharpe; the relative rank, its logit and the summary statistics are formed here.
* `deflated_sharpe(moments, n_trials)` -- the Deflated Sharpe Ratio (Bailey, Lopez de Prado 2014, "The Deflated Sharpe
  Ratio"): the probability that a trial's true Sharpe exceeds the expected maximum of `n_trials` unskilled trials.

The per-day rows come from `PopulationSweep.daily_pnl`; StrategyEvaluationSystem.backtest_overfitting chains the two.
"""
from __future__ import annotations

import math
from statistics import NormalDist
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib

EULER_GAMMA = 0.5772156649015329


def cscv(pnl: torch.Tensor, n_blocks: int = 16) -> Dict:
    """CSCV of the N trials in the rows of `pnl` (device float64 [N][T], one per-period return per column, the same
    periods for every trial).  Returns numpy arrays per combination c (itertools.combinations(range(B), B // 2) order:
    in-sample set J_c, out-of-sample its complement):
      sel, is_sr, oos_sr, n_below, n_tied   the kernel's outputs (include/b200bt.h)
      omega   (n_below + 1 + n_tied / 2) / (N + 1), the selected trial's average relative rank out of sample
      logit   ln(omega / (1 - omega))
    per trial: mu, m2, m3, m4 (full-sample central moments of the kept days), sharpe (annualised, all kept days);
    and pbo = mean(logit <= 0), prob_oos_loss = mean(oos_sr < 0), degradation {slope, intercept, r2} of the least-squares
    fit oos_sr ~ slope * is_sr + intercept, n_trials, n_blocks, n_combinations, block_days, dropped_days."""
    if not (isinstance(pnl, torch.Tensor) and pnl.is_cuda and pnl.dtype == torch.float64 and pnl.dim() == 2):
        raise ValueError("cscv needs a device float64 matrix [N][T]")
    N, T = int(pnl.shape[0]), int(pnl.shape[1])
    B = int(n_blocks)
    lib = _lib.load()
    ws_bytes = int(lib.b200bt_cscv_workspace_bytes(N, T, B))
    if ws_bytes <= 0:
        raise ValueError(f"cscv: N = {N} trials, T = {T} days and B = {B} blocks are outside the limits "
                         "(N >= 2, B even, 2 <= B <= 20, T // B >= 2)")
    if not bool(torch.isfinite(pnl).all()):
        raise ValueError("cscv: the rows hold NaN or inf (lost records? sweep again with a larger event cap)")
    dev = pnl.device
    C = math.comb(B, B // 2)
    pnl = pnl if pnl.stride(1) == 1 else pnl.contiguous()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    i32 = lambda n: torch.empty(n, dtype=torch.int32, device=dev)
    f64 = lambda n: torch.empty(n, dtype=torch.float64, device=dev)
    sel, n_below, n_tied = i32(C), i32(C), i32(C)
    is_sr, oos_sr = f64(C), f64(C)
    mu, m2, m3, m4, sr = f64(N), f64(N), f64(N), f64(N), f64(N)
    with torch.cuda.device(dev):
        _lib.call("b200bt_cscv", pnl.data_ptr(), _lib.ld(pnl), N, T, B, ws.data_ptr(), ws_bytes, sel.data_ptr(),
                  is_sr.data_ptr(), oos_sr.data_ptr(), n_below.data_ptr(), n_tied.data_ptr(), mu.data_ptr(), m2.data_ptr(),
                  m3.data_ptr(), m4.data_ptr(), sr.data_ptr(), _lib.current_stream())
    out = {k: v.cpu().numpy() for k, v in dict(sel=sel, is_sr=is_sr, oos_sr=oos_sr, n_below=n_below, n_tied=n_tied, mu=mu,
                                               m2=m2, m3=m3, m4=m4, sharpe=sr).items()}
    L = T // B
    out.update(summarize(out["is_sr"], out["oos_sr"], out["n_below"], out["n_tied"], N),
               n_trials=N, n_blocks=B, n_combinations=C, block_days=L, dropped_days=T - B * L)
    return out


def summarize(is_sr: np.ndarray, oos_sr: np.ndarray, n_below: np.ndarray, n_tied: np.ndarray, n_trials: int) -> Dict:
    """omega, logit, pbo, prob_oos_loss and the degradation fit from the per-combination outputs."""
    omega = (n_below.astype(np.float64) + 1.0 + n_tied.astype(np.float64) / 2.0) / (n_trials + 1.0)
    logit = np.log(omega / (1.0 - omega))
    x, y = np.asarray(is_sr, dtype=np.float64), np.asarray(oos_sr, dtype=np.float64)
    dx, dy = x - x.mean(), y - y.mean()
    sxx, syy, sxy = float(dx @ dx), float(dy @ dy), float(dx @ dy)
    slope = sxy / sxx if sxx > 0 else math.nan
    intercept = float(y.mean() - slope * x.mean()) if sxx > 0 else math.nan
    r2 = sxy * sxy / (sxx * syy) if sxx > 0 and syy > 0 else math.nan
    return dict(omega=omega, logit=logit, pbo=float(np.mean(logit <= 0)), prob_oos_loss=float(np.mean(y < 0)),
                degradation=dict(slope=slope, intercept=intercept, r2=r2))


def deflated_sharpe(moments: Dict, n_trials: int, n_days: Optional[int] = None) -> np.ndarray:
    """Deflated Sharpe Ratio of every trial.  `moments`: per-trial arrays mu, m2, m3, m4, full-sample central moments of
    `n_days` kept days (a cscv() result: n_days defaults to its n_blocks * block_days).  With the daily (non-annualised)
    SR_n = mu / sqrt(m2), skew = m3 / m2^1.5, kurt = m4 / m2^2 (not excess):
      SR0 = sqrt(Var[SR_n]) * ((1 - g) * Phi^-1(1 - 1/N) + g * Phi^-1(1 - 1/(N e))),  g = Euler-Mascheroni, N = n_trials
      DSR = Phi((SR - SR0) * sqrt(n_days - 1) / sqrt(1 - skew * SR + (kurt - 1) / 4 * SR^2))
    Var[SR_n] is the population variance (ddof 0) across the trials given.  A trial of zero variance, or whose
    denominator is not positive, gets NaN."""
    N = int(n_trials)
    if n_days is None:
        n_days = int(moments["n_blocks"]) * int(moments["block_days"])
    if N < 2:
        raise ValueError("deflated_sharpe needs at least 2 trials")
    mu = np.asarray(moments["mu"], dtype=np.float64)
    m2 = np.asarray(moments["m2"], dtype=np.float64)
    m3 = np.asarray(moments["m3"], dtype=np.float64)
    m4 = np.asarray(moments["m4"], dtype=np.float64)
    ok = m2 > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        sr = np.where(ok, mu / np.sqrt(m2), 0.0)
        skew = np.where(ok, m3 / m2 ** 1.5, np.nan)
        kurt = np.where(ok, m4 / (m2 * m2), np.nan)
        nd = NormalDist()
        sr0 = math.sqrt(float(np.var(sr))) * ((1 - EULER_GAMMA) * nd.inv_cdf(1 - 1 / N)
                                              + EULER_GAMMA * nd.inv_cdf(1 - 1 / (N * math.e)))
        den = 1 - skew * sr + (kurt - 1) / 4 * sr * sr
        z = (sr - sr0) * math.sqrt(n_days - 1) / np.sqrt(den)
    out = np.full(len(mu), np.nan)
    for i in np.nonzero(ok & (den > 0))[0]:
        out[i] = 0.5 * math.erfc(-float(z[i]) / math.sqrt(2.0))
    return out
