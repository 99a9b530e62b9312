"""Oracles of the backtest-overfitting path (csrc/overfitting.cu, ai_crypto_trader_b200/overfitting.py).

* cscv_exact    the arithmetic contract of b200bt_cscv (include/b200bt.h) in numpy: correctly rounded float64, explicit
                ascending loops over days and blocks (vectorised across trials and combinations only), so that every
                output is bit-identical to the kernel's.
* cscv_literal  the algorithm of Bailey, Borwein, Lopez de Prado and Zhu (2015) as written: for every split, concatenate
                the in-sample blocks, Sharpe with np.mean / np.std, first-max argmax, the out-of-sample average rank.
* lane_rows / book_rows  the per-day PnL of oracle/sim_oracle.c lane records bucketed on the host, for b200bt_daily_pnl.
"""
from __future__ import annotations

import itertools
import math

import numpy as np

BAR_MASK = 0x3FFFFFFF
SQRT252 = np.sqrt(np.float64(252.0))


def combination_masks(B: int) -> np.ndarray:
    """bool [C][B]: row c = in-sample blocks of itertools.combinations(range(B), B // 2)'s c-th split."""
    combos = list(itertools.combinations(range(B), B // 2))
    m = np.zeros((len(combos), B), dtype=bool)
    for c, J in enumerate(combos):
        m[c, list(J)] = True
    return m


def moments(x: np.ndarray, B: int) -> dict:
    """Per-trial mu, a [B][N], q [B][N], m2, m3, m4, sharpe of the kept days, in the kernel's order."""
    x = np.asarray(x, dtype=np.float64)
    N, T = x.shape
    L = T // B
    r, n = T - B * L, B * L
    k = x[:, r:r + n]
    s = np.zeros(N)
    for t in range(n):
        s = s + k[:, t]
    mu = s / np.float64(n)
    a, q = np.zeros((B, N)), np.zeros((B, N))
    m2, m3, m4 = np.zeros(N), np.zeros(N), np.zeros(N)
    for b in range(B):
        for t in range(b * L, (b + 1) * L):
            d = k[:, t] - mu
            d2 = d * d
            a[b] = a[b] + d
            q[b] = q[b] + d2
            m2 = m2 + d2
            m3 = m3 + d2 * d
            m4 = m4 + d2 * d2
    m2 = m2 / np.float64(n)
    with np.errstate(divide="ignore", invalid="ignore"):
        sr = np.where(m2 > 0, (mu / np.sqrt(m2)) * SQRT252, 0.0)
    return dict(mu=mu, a=a, q=q, m2=m2, m3=m3 / np.float64(n), m4=m4 / np.float64(n), sharpe=sr, L=L, r=r)


def _set_sharpe(mom: dict, inset: np.ndarray, n_set: float) -> np.ndarray:
    """[cc][N] Sharpe of the block sets `inset` (bool [cc][B]), A and Q summed from +0.0 in ascending block order."""
    a, q, mu = mom["a"], mom["q"], mom["mu"]
    A = np.zeros((len(inset), a.shape[1]))
    Q = np.zeros_like(A)
    for b in range(a.shape[0]):
        A = A + np.where(inset[:, b, None], a[b][None, :], 0.0)
        Q = Q + np.where(inset[:, b, None], q[b][None, :], 0.0)
    m = A / n_set
    v = Q / n_set - m * m
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(v > 0, ((mu[None, :] + m) / np.sqrt(v)) * SQRT252, 0.0)


def cscv_exact(x: np.ndarray, B: int, chunk_elems: int = 1 << 22) -> dict:
    """b200bt_cscv's outputs: sel, is_sr, oos_sr, n_below, n_tied per combination, mu, m2, m3, m4, sharpe per trial,
    plus is_gap: per combination, the relative gap between the best and the second-best in-sample Sharpe."""
    mom = moments(x, B)
    N = x.shape[0]
    masks = combination_masks(B)
    C = len(masks)
    n_set = np.float64((B // 2) * mom["L"])
    out = {k: np.zeros(C, dtype=np.int32) for k in ("sel", "n_below", "n_tied")}
    out.update({k: np.zeros(C) for k in ("is_sr", "oos_sr", "is_gap")})
    step = max(1, chunk_elems // N)
    rows = np.arange(N)
    for c0 in range(0, C, step):
        m = masks[c0:c0 + step]
        sis, soos = _set_sharpe(mom, m, n_set), _set_sharpe(mom, ~m, n_set)
        sel = np.argmax(sis, axis=1)                       # first maximum: ties go to the lowest trial
        k = np.arange(len(m))
        o = soos[k, sel]
        part = np.sort(sis, axis=1)
        out["sel"][c0:c0 + len(m)] = sel
        out["is_sr"][c0:c0 + len(m)] = sis[k, sel]
        out["oos_sr"][c0:c0 + len(m)] = o
        out["n_below"][c0:c0 + len(m)] = np.sum(soos < o[:, None], axis=1)
        out["n_tied"][c0:c0 + len(m)] = np.sum((soos == o[:, None]) & (rows[None, :] != sel[:, None]), axis=1)
        with np.errstate(divide="ignore", invalid="ignore"):
            out["is_gap"][c0:c0 + len(m)] = (part[:, -1] - part[:, -2]) / np.maximum(np.abs(part[:, -1]), 1e-300)
    out.update({k: mom[k] for k in ("mu", "m2", "m3", "m4", "sharpe")})
    out.update(block_days=mom["L"], dropped_days=mom["r"], n_blocks=B, n_trials=N, n_combinations=C)
    return out


def _sharpe(x: np.ndarray) -> np.ndarray:
    """mean / std(ddof 0) * sqrt(252) of every row, 0 where the std is 0."""
    sd = np.std(x, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(sd > 0, np.mean(x, axis=1) / sd * math.sqrt(252), 0.0)


def cscv_literal(x: np.ndarray, B: int) -> dict:
    """CSCV as the paper states it: the T x N matrix cut into B row blocks; per split J, SR of concat(J) and of
    concat(complement), n* = argmax in sample, omega = its average relative rank out of sample, logit = ln(omega/(1-omega)),
    PBO = fraction of splits with logit <= 0."""
    from scipy.stats import rankdata
    x = np.asarray(x, dtype=np.float64)
    N, T = x.shape
    L = T // B
    blocks = [x[:, T - B * L + b * L: T - B * L + (b + 1) * L] for b in range(B)]
    sel, omega = [], []
    for J in itertools.combinations(range(B), B // 2):
        Jc = [b for b in range(B) if b not in J]
        sis = _sharpe(np.concatenate([blocks[b] for b in J], axis=1))
        soos = _sharpe(np.concatenate([blocks[b] for b in Jc], axis=1))
        n = int(np.argmax(sis))
        sel.append(n)
        omega.append(rankdata(soos, method="average")[n] / (N + 1))
    omega = np.array(omega)
    logit = np.log(omega / (1 - omega))
    return dict(sel=np.array(sel), omega=omega, logit=logit, pbo=float(np.mean(logit <= 0)))


def day_of(bars: np.ndarray, cfg) -> np.ndarray:
    """Calendar day of bars (minute0 + bar * bar_minutes + the gap after gap_bar) // 1440 (cfg: sim_oracle.Config)."""
    bars = np.asarray(bars, dtype=np.int64)
    gap = np.where((cfg.gap_bar > 0) & (bars >= cfg.gap_bar), cfg.gap_minutes, 0)
    return (cfg.minute0 + bars * cfg.bar_minutes + gap) // 1440


def calendar(cfg, n_bars: int):
    """(first_day, D) of a series of n_bars under cfg."""
    first = int(day_of(np.array([0]), cfg)[0])
    return first, int(day_of(np.array([n_bars - 1]), cfg)[0]) - first + 1


def lane_rows(events, pnl, cfg, n_bars: int) -> np.ndarray:
    """float64 [D]: pnl of one lane's records summed by calendar day, in record order."""
    first, D = calendar(cfg, n_bars)
    row = np.zeros(D)
    days = day_of(np.asarray(events, dtype=np.int64) & BAR_MASK, cfg) - first
    for d, p in zip(days.tolist(), np.asarray(pnl, dtype=np.float64).tolist()):
        row[d] += p
    return row


def book_row(rows: list) -> np.ndarray:
    """Sum of the lane rows of one individual in symbol order."""
    acc = np.array(rows[0], dtype=np.float64)
    for r in rows[1:]:
        acc = acc + r
    return acc
