"""Backtest overfitting of a searched population: how much of the best backtest's performance is the search itself.

Host side of `b200bt_cscv`, `b200bt_spa_moments` and `b200bt_spa_bootstrap` (include/b200bt.h):

* `cscv(pnl, n_blocks)` -- the Probability of Backtest Overfitting by combinatorially symmetric cross-validation
  (Bailey, Borwein, Lopez de Prado, Zhu 2015, "The Probability of Backtest Overfitting").  The kernel gives, for every
  split of the B time blocks into two halves, the in-sample winner and the integer rank counts of its out-of-sample
  Sharpe; the relative rank, its logit and the summary statistics are formed here.
* `deflated_sharpe(moments, n_trials)` -- the Deflated Sharpe Ratio (Bailey, Lopez de Prado 2014, "The Deflated Sharpe
  Ratio"): the probability that a trial's true Sharpe exceeds the expected maximum of `n_trials` unskilled trials.
* `spa(rows, benchmark)` -- the data-snooping tests of the best of N trials against a benchmark on the stationary
  bootstrap: White's Reality Check, Hansen's SPA and Romano and Wolf's StepM.
* `mcs(rows)` -- Hansen, Lunde and Nason's Model Confidence Set: the trials that cannot be told apart from the best, with
  a p-value for each (b200bt_boot_means, b200bt_mcs_*).
* `optimal_block_length(rows)` -- Politis and White's automatic block length (Patton, Politis and White's correction)
  from the rows' autocovariances (b200bt_autocov).

The per-day rows come from `PopulationSweep.daily_pnl`; StrategyEvaluationSystem.backtest_overfitting chains them with
CSCV and the deflated Sharpe ratio, StrategyEvaluationSystem.data_snooping with `spa`,
StrategyEvaluationSystem.model_confidence_set with `mcs`.
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


SPA_MAX_OUT_BYTES = 1 << 28


def spa_q32(block_len: float) -> int:
    """round(2^32 / block_len) in [1, 2^32]: the restart threshold of the stationary bootstrap's index stream."""
    if not (block_len >= 1.0 and math.isfinite(block_len)):
        raise ValueError(f"spa: block_len = {block_len} must be a finite number >= 1")
    return min(1 << 32, max(1, round(2.0 ** 32 / float(block_len))))


def spa_shifts(mean: np.ndarray, omega: np.ndarray, n_days: int):
    """(shift, scale) rows [4][N] of the first bootstrap launch: Reality Check (shift mean, scale sqrt(T)), then SPA
    lower / consistent / upper (shifts max(mean, 0), mean * 1{mean > -omega sqrt(2 ln ln T / T)}, mean; scale
    sqrt(T) / omega).  Trials without a positive variance estimate (omega NaN) are excluded from SPA (shift +inf)."""
    rt = math.sqrt(n_days)
    ok = np.isfinite(omega)
    thr = math.sqrt(max(0.0, 2.0 * math.log(math.log(n_days)) / n_days)) if n_days > 2 else 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        scale_t = np.where(ok, rt / omega, 0.0)
        consistent = np.where(mean > -omega * thr, mean, 0.0)
    shift = np.stack([mean, np.maximum(mean, 0.0), consistent, mean])
    shift[1:, ~ok] = np.inf
    scale = np.stack([np.full(len(mean), rt), scale_t, scale_t, scale_t])
    return shift, scale


def spa_summary(mean: np.ndarray, omega: np.ndarray, n_days: int, out: np.ndarray, stepm_rows, alpha: float) -> Dict:
    """Statistics and p-values from the bootstrap maxima.  out: [4][B], the rows of spa_shifts; stepm_rows(active)
    returns the [B] maxima of (m* - mean) * sqrt(T) / omega over the boolean mask `active` (a further launch); the first
    StepM step reads the SPA-upper row instead."""
    B = out.shape[1]
    rt = math.sqrt(n_days)
    ok = np.isfinite(omega)
    with np.errstate(invalid="ignore", divide="ignore"):
        t_stat = np.where(ok, rt * mean / omega, np.nan)
    V = float(np.max(rt * mean))
    rc = dict(stat=V, pvalue=float(np.count_nonzero(out[0] > V)) / B)
    if ok.any():
        t_spa = max(0.0, float(np.max(t_stat[ok])))
        p = [float(np.count_nonzero(np.maximum(0.0, out[j]) > t_spa)) / B for j in (1, 2, 3)]
    else:
        t_spa, p = math.nan, [math.nan] * 3
    spa = dict(stat=t_spa, pvalue_lower=p[0], pvalue_consistent=p[1], pvalue_upper=p[2])
    rejected = np.zeros(len(mean), dtype=bool)
    crit = []
    rank = max(1, math.ceil((1.0 - alpha) * B))
    active = ok.copy()
    row = out[3]
    while active.any():
        c = float(np.sort(row)[rank - 1])
        crit.append(c)
        new = active & (t_stat > c)
        if not new.any():
            break
        rejected |= new
        active &= ~new
        if not active.any():
            break
        row = stepm_rows(active)
    best = None
    if ok.any():
        i = int(np.argmax(np.where(ok, t_stat, -np.inf)))
        best = dict(index=i, t_stat=float(t_stat[i]), mean=float(mean[i]))
    return dict(t_stat=t_stat, reality_check=rc, spa=spa,
                stepm=dict(alpha=alpha, rejected=rejected, critical_values=crit), best=best)


def spa(rows: torch.Tensor, benchmark: Optional[torch.Tensor] = None, n_boot: int = 10_000, block_len=10.0,
        alpha: float = 0.05, seed: int = 0, max_out_bytes: int = SPA_MAX_OUT_BYTES) -> Dict:
    """Data-snooping tests of the N trials in the rows of `rows` (device float64 [N][T], one per-period PnL per column,
    the same periods for every trial) against `benchmark` (a device [T] row; None: flat, zero PnL): is the best trial
    better than the benchmark once the search over N trials is accounted for?

    On the differentials d = rows - benchmark, with the stationary bootstrap of mean block length `block_len`
    (q = 1 / block_len; "auto": optimal_block_length of the differentials) and `n_boot` resamples
    (b200bt_spa_moments, b200bt_spa_bootstrap; include/b200bt.h):
      mean, omega (Hansen's stationary-bootstrap standard deviation, NaN where omega^2 <= 0), t_stat = sqrt(T) mean /
      omega (NaN likewise) per trial;
      reality_check {stat, pvalue}: White's V = max sqrt(T) mean, p = #{b: V*_b > V} / B;
      spa {stat, pvalue_lower, pvalue_consistent, pvalue_upper}: Hansen's T = max(0, max t), p = #{b: T*_b > T} / B
        with T*_b = max(0, max_k (m* - g(mean)) sqrt(T) / omega) for the three recentrings g (NaN with no eligible trial);
      stepm {alpha, rejected [N], critical_values}: Romano and Wolf's studentized StepM at level alpha: each step's
        critical value is the ceil((1 - alpha) B)-th smallest bootstrap maximum over the active (not yet rejected,
        eligible) trials; the active trials with t > c are rejected, until a step rejects nothing;
      best {index, t_stat, mean}: the trial of highest t_stat (the first on ties; None with no eligible trial);
      n_trials, n_days, n_boot, block_len, seed.
    Trials with omega^2 <= 0 (a never-trading row against a flat benchmark) take no part in SPA and StepM.  The
    resamples are split over launches by their global index when the [4][n_boot] maxima exceed `max_out_bytes`; the
    result does not depend on the split."""
    if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype == torch.float64 and rows.dim() == 2):
        raise ValueError("spa needs a device float64 matrix [N][T]")
    N, T = int(rows.shape[0]), int(rows.shape[1])
    B = int(n_boot)
    if N < 1 or B < 1 or not 0.0 < alpha < 1.0:
        raise ValueError(f"spa: N = {N} trials, n_boot = {B} and alpha = {alpha} need N >= 1, n_boot >= 1, 0 < alpha < 1")
    if benchmark is not None:
        if not (isinstance(benchmark, torch.Tensor) and benchmark.device == rows.device and benchmark.numel() == T):
            raise ValueError(f"spa: the benchmark must be a [{T}] row on {rows.device}")
        d = rows - benchmark.reshape(1, T).to(torch.float64)
    else:
        d = rows if rows.stride(1) == 1 else rows.contiguous()
    if not bool(torch.isfinite(d).all()):
        raise ValueError("spa: the rows hold NaN or inf (lost records? sweep again with a larger event cap)")
    if block_len == "auto" and not 2 <= T <= 8192:
        raise ValueError(f"spa: T = {T} days outside [2, 8192]")
    block_len = _block_len(d, block_len)
    q32 = spa_q32(block_len)
    dev = d.device
    per_launch = max(1, int(max_out_bytes) // (4 * 8))
    mean_d = torch.empty(N, dtype=torch.float64, device=dev)
    omega2_d = torch.empty(N, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        st = _lib.current_stream()
        _lib.call("b200bt_spa_moments", d.data_ptr(), _lib.ld(d), N, T, q32 / 2.0 ** 32, mean_d.data_ptr(),
                  omega2_d.data_ptr(), st)
        mean, omega2 = mean_d.cpu().numpy(), omega2_d.cpu().numpy()
        omega = np.where(omega2 > 0, np.sqrt(np.where(omega2 > 0, omega2, 1.0)), np.nan)

        def maxima(shift: np.ndarray, scale: np.ndarray) -> np.ndarray:
            n_stats = shift.shape[0]
            sh = torch.from_numpy(np.ascontiguousarray(shift)).to(dev)
            sc = torch.from_numpy(np.ascontiguousarray(scale)).to(dev)
            res = np.empty((n_stats, B))
            for lo in range(0, B, per_launch):
                n = min(per_launch, B - lo)
                out = torch.empty((n_stats, n), dtype=torch.float64, device=dev)
                _lib.call("b200bt_spa_bootstrap", d.data_ptr(), _lib.ld(d), N, T, q32, n, seed, lo, n_stats,
                          sh.data_ptr(), sc.data_ptr(), out.data_ptr(), st)
                res[:, lo:lo + n] = out.cpu().numpy()
            return res

        shift, scale = spa_shifts(mean, omega, T)
        out = maxima(shift, scale)

        def stepm_rows(active: np.ndarray) -> np.ndarray:
            return maxima(np.where(active, mean, np.inf)[None], scale[1:2])[0]

        res = spa_summary(mean, omega, T, out, stepm_rows, alpha)
    res.update(mean=mean, omega=omega, n_trials=N, n_days=T, n_boot=B, block_len=float(block_len), seed=int(seed))
    return res


# ---- automatic block length and the model confidence set ----------------------------------------------------------

MCS_MAX_BYTES = 8 << 30


def block_length_rule(acov: np.ndarray, n_days: int):
    """Politis and White (2004) optimal mean block length of the stationary bootstrap, with the correction of Patton,
    Politis and White (2009), from each row's autocovariances acov [N][K+1] (R(k) for k = 0..K; lags past K count as 0).
    With T = n_days:
      K_N = max(5, ceil(sqrt(log10 T))), m_max = ceil(sqrt T) + K_N, b_max = ceil(min(3 sqrt T, T / 3));
      rho(k) = R(k) / R(0);
      m_hat = the smallest m >= 0 with |rho(m + j)| < 2 sqrt(log10 T / T) (strict) for every j = 1..K_N, else m_max;
      M = min(2 max(m_hat, 1), m_max);
      lambda(s) = 1 for |s| <= 1/2, 2 (1 - |s|) for 1/2 < |s| <= 1, 0 otherwise;
      g = R(0) + 2 sum_{k=1}^{M} lambda(k / M) R(k);  G = 2 sum_{k=1}^{M} lambda(k / M) k R(k);
      b = (2 G^2 / (2 g^2))^(1/3) T^(1/3), clipped to [1, b_max] (g = 0 gives b_max).
    A row with R(0) = 0 has no estimate (NaN).  Returns (per_row [N], block_len): block_len is the median of the rows
    that have an estimate (np.median), 1.0 when none has."""
    acov = np.atleast_2d(np.asarray(acov, dtype=np.float64))
    T = int(n_days)
    KN = max(5, math.ceil(math.sqrt(math.log10(T))))
    m_max = math.ceil(math.sqrt(T)) + KN
    b_max = math.ceil(min(3.0 * math.sqrt(T), T / 3.0))
    c = 2.0 * math.sqrt(math.log10(T) / T)
    lags = np.zeros((acov.shape[0], m_max + KN + 1))
    n = min(acov.shape[1], lags.shape[1])
    lags[:, :n] = acov[:, :n]
    out = np.full(acov.shape[0], np.nan)
    for r, R in enumerate(lags):
        if R[0] == 0.0:
            continue
        rho = R / R[0]
        m_hat = next((m for m in range(m_max + 1) if np.all(np.abs(rho[m + 1:m + KN + 1]) < c)), m_max)
        M = min(2 * max(m_hat, 1), m_max)
        k = np.arange(1, M + 1)
        s = np.abs(k / M)
        lam = np.where(s <= 0.5, 1.0, np.where(s <= 1.0, 2.0 * (1.0 - s), 0.0))
        g = R[0] + 2.0 * float(np.sum(lam * R[1:M + 1]))
        G = 2.0 * float(np.sum(lam * k * R[1:M + 1]))
        b = b_max if g == 0.0 else (2.0 * G * G / (2.0 * g * g)) ** (1.0 / 3.0) * T ** (1.0 / 3.0)
        out[r] = min(max(b, 1.0), b_max)
    ok = np.isfinite(out)
    return out, float(np.median(out[ok])) if ok.any() else 1.0


def _rows(rows: torch.Tensor, what: str, min_rows: int) -> torch.Tensor:
    if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype == torch.float64 and rows.dim() == 2):
        raise ValueError(f"{what} needs a device float64 matrix [N][T]")
    N, T = int(rows.shape[0]), int(rows.shape[1])
    if N < min_rows or not 2 <= T <= 8192:
        raise ValueError(f"{what}: N = {N} rows and T = {T} days need N >= {min_rows} and 2 <= T <= 8192")
    if not bool(torch.isfinite(rows).all()):
        raise ValueError(f"{what}: the rows hold NaN or inf (lost records? sweep again with a larger event cap)")
    return rows if rows.stride(1) == 1 else rows.contiguous()


def autocov(rows: torch.Tensor, K: int):
    """(acov [N][K+1], mean [N]) device float64 from b200bt_autocov: the rows' autocovariances at lags 0..K."""
    N, T = int(rows.shape[0]), int(rows.shape[1])
    out = torch.empty((N, K + 1), dtype=torch.float64, device=rows.device)
    mean = torch.empty(N, dtype=torch.float64, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.call("b200bt_autocov", rows.data_ptr(), _lib.ld(rows), N, T, K, out.data_ptr(), mean.data_ptr(),
                  _lib.current_stream())
    return out, mean


def optimal_block_length(rows: torch.Tensor) -> Dict:
    """Automatic mean block length for the stationary bootstrap of the rows (device float64 [N][T], finite): the
    autocovariances from b200bt_autocov, then block_length_rule on the host.  Returns {per_row [N], block_len}."""
    rows = _rows(rows, "optimal_block_length", 1)
    T = int(rows.shape[1])
    KN = max(5, math.ceil(math.sqrt(math.log10(T))))
    K = min(math.ceil(math.sqrt(T)) + 2 * KN, T - 1)
    acov, _ = autocov(rows, K)
    per_row, b = block_length_rule(acov.cpu().numpy(), T)
    return dict(per_row=per_row, block_len=b)


def _block_len(rows: torch.Tensor, block_len) -> float:
    if isinstance(block_len, str):
        if block_len != "auto":
            raise ValueError(f"block_len = {block_len!r}: a number >= 1 or 'auto'")
        return optimal_block_length(rows)["block_len"]
    return float(block_len)


def mcs_pvalues(order: np.ndarray, step_p: np.ndarray, alpha: float):
    """MCS p-values in model order: e_k gets max over l <= k of p_l, the last survivor 1; included = p >= alpha."""
    N = len(order)
    p = np.empty(N)
    run = 0.0
    for k in range(N - 1):
        run = max(run, float(step_p[k]))
        p[order[k]] = run
    p[order[N - 1]] = 1.0
    return p, p >= alpha


def distinct_rows(rows: torch.Tensor):
    """(reps, model_of): the rows of a device matrix that are byte-identical form one model.  reps (int64 [D]) is the
    first row of each model in ascending order; model_of (int64 [N]) is, for every row, the position in reps of its
    model."""
    bits = rows.contiguous().view(torch.int64)
    _, inverse = torch.unique(bits, dim=0, return_inverse=True)
    inverse = inverse.cpu().numpy()
    first = np.full(int(inverse.max()) + 1, len(inverse), dtype=np.int64)
    np.minimum.at(first, inverse, np.arange(len(inverse)))
    reps = np.sort(first)
    return reps, np.searchsorted(reps, first[inverse])


def mcs(rows: torch.Tensor, alpha: float = 0.10, statistic: str = "R", n_boot: int = 10_000, block_len=10.0,
        seed: int = 0, max_bytes: int = MCS_MAX_BYTES) -> Dict:
    """Model Confidence Set (Hansen, Lunde and Nason 2011) of the N rows of `rows` (device float64 [N][T], one per-day
    PnL per column, the same days for every row, finite): the set that contains the best model (highest mean PnL; the
    loss is the negated PnL) with probability 1 - alpha, and a p-value for every row.

    Rows that are byte-identical are one model (distinct_rows): a GA population often holds individuals whose books
    are the same, and copies must stand or fall together.  The D distinct models, in the order of their first rows, go
    through the elimination; every row then takes its model's results.

    statistic "R" (T_R, the range of the pairwise t-statistics) or "max" (T_max, each model against the set's mean), on
    the stationary bootstrap of mean block length `block_len` (a number >= 1, or "auto": optimal_block_length's median
    over the rows) with `n_boot` resamples drawn as spa() draws them for the same seed.  Definitions:
    include/b200bt.h.  Step k removes e_k from M_k with p_k = #{b : T*_b(M_k) >= T(M_k)} / B; the MCS p-value of e_k is
    max over l <= k of p_l, the last survivor's 1, and the set at level alpha is {i : p_i >= alpha}.

    Returns p_values [N], included [N], model_of [N] (the index of each row's model among the D), n_models (D),
    elimination_order [N] (the rows of each eliminated model together, ascending, the last survivor's last),
    step_stats and step_pvalues [D-1], mean [N], block_len (the length used), n_trials (N), n_days, n_boot, seed,
    statistic, alpha.  With D = 1 every row is the last survivor (p = 1) and nothing is resampled.  Nothing of size
    [B][D] leaves the device.  T_R splits the resamples over launches (boot_offset) when its [B][D] buffers do not fit
    `max_bytes` beside the [D][D] ones, recomputing the means for the maxima pass; the result does not depend on the
    split.  T_max needs every resample at once.  ValueError: non-finite rows, N < 2, bad arguments, or a budget that
    cannot hold the buffers."""
    rows = _rows(rows, "mcs", 2)
    N, T = int(rows.shape[0]), int(rows.shape[1])
    B = int(n_boot)
    if statistic not in ("R", "max") or B < 1 or not 0.0 < alpha < 1.0 or N > 16384:
        raise ValueError(f"mcs: statistic = {statistic!r}, n_boot = {B}, alpha = {alpha}, N = {N} need statistic 'R' or "
                         "'max', n_boot >= 1, 0 < alpha < 1 and N <= 16384")
    bl = _block_len(rows, block_len)
    q32 = spa_q32(bl)
    reps, model_of = distinct_rows(rows)
    D = len(reps)
    x = rows[torch.from_numpy(reps).to(rows.device)].contiguous()
    if D >= 2:
        order_d, step_stats, step_p, mean_d = _mcs_models(x, statistic, B, q32, seed, int(max_bytes))
    else:
        _, mean = autocov(x, 0)
        order_d, step_stats, step_p, mean_d = np.zeros(1, np.int64), np.empty(0), np.empty(0), mean.cpu().numpy()
    p_d, _ = mcs_pvalues(order_d, step_p, alpha)
    p = p_d[model_of]
    members = [np.flatnonzero(model_of == g) for g in range(D)]
    order = np.concatenate([members[g] for g in order_d])
    return dict(p_values=p, included=p >= alpha, model_of=model_of, n_models=D, elimination_order=order,
                step_stats=step_stats, step_pvalues=step_p, mean=mean_d[model_of], block_len=bl, n_trials=N, n_days=T,
                n_boot=B, seed=int(seed), statistic=statistic, alpha=float(alpha))


def _mcs_models(rows: torch.Tensor, statistic: str, B: int, q32: int, seed: int, budget: int):
    """(order [N], step_stats [N-1], step_pvalues [N-1], mean [N]) of the elimination over N >= 2 models."""
    N, T = int(rows.shape[0]), int(rows.shape[1])
    dev = rows.device
    f64 = lambda *s: torch.empty(s, dtype=torch.float64, device=dev)
    order = torch.empty(N, dtype=torch.int32, device=dev)
    stat = f64(N - 1)
    count = torch.zeros(N - 1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        st = _lib.current_stream()
        _, mean = autocov(rows, 0)

        def means(z, lo, n):
            _lib.call("b200bt_boot_means", rows.data_ptr(), _lib.ld(rows), N, T, q32, n, seed, lo, mean.data_ptr(),
                      z.data_ptr(), N, budget, st)

        if statistic == "R":
            per = (budget - 2 * N * N * 8) // (2 * N * 8)
            if per < 1:
                raise ValueError(f"mcs: max_bytes = {budget} cannot hold the [N][N] buffers and one resample (N = {N} "
                                 "distinct models)")
            per = min(per, B)
            z = f64(per, N)
            w = torch.zeros((N, N), dtype=torch.float64, device=dev)
            t = f64(N, N)
            for lo in range(0, B, per):
                n = min(per, B - lo)
                means(z, lo, n)
                _lib.call("b200bt_mcs_pairwise", z.data_ptr(), N, N, n, w.data_ptr(), budget, st)
            _lib.call("b200bt_mcs_range_stats", mean.data_ptr(), N, B, w.data_ptr(), t.data_ptr(), budget, st)
            _lib.call("b200bt_mcs_range_order", t.data_ptr(), w.data_ptr(), N, order.data_ptr(), stat.data_ptr(),
                      t.data_ptr(), budget, st)
            rmax = f64(per, N)
            for lo in range(0, B, per):
                n = min(per, B - lo)
                if per < B:                          # the pairwise pass's means were overwritten: draw them again
                    means(z, lo, n)
                _lib.call("b200bt_mcs_range_boot", z.data_ptr(), N, N, n, order.data_ptr(), t.data_ptr(),
                          stat.data_ptr(), rmax.data_ptr(), count.data_ptr(), budget, st)
        else:
            if B * N * 8 > budget:
                raise ValueError(f"mcs: T_max needs all {B} x {N} bootstrap means at once; max_bytes = {budget} is too "
                                 "small")
            z = f64(B, N)
            means(z, 0, B)
            ws_bytes = int(_lib.load().b200bt_mcs_max_workspace_bytes(N, B))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            _lib.call("b200bt_mcs_max", z.data_ptr(), N, N, B, mean.data_ptr(), ws.data_ptr(), ws_bytes,
                      order.data_ptr(), stat.data_ptr(), count.data_ptr(), budget, st)
        return (order.cpu().numpy().astype(np.int64), stat.cpu().numpy(),
                count.cpu().numpy().astype(np.float64) / B, mean.cpu().numpy())
