"""CPU restatement of the joint (portfolio) Monte-Carlo generators of csrc/montecarlo.cu (test infrastructure).

Built on oracle/mc_ref.py's Philox4x32-10, Box-Muller and bootstrap index stream, with the joint kernels' counter
(path lo, hi, step/4, (factor << 8) | mode): normal factor 0 is gbm_paths' stream, the day-index stream is
bootstrap_paths'.  Log-prices accumulate in float64, the portfolio value V_t = sum_i q_i s0_i exp(logS_i,t) and its
drawdown max_t (runmax_t - V_t) / runmax_t (monte_carlo_service.py:327-336 applied to V_t) are float64.
"""
from __future__ import annotations

import numpy as np

from oracle import mc_ref


def normals(factor, n_paths, steps, seed, path_offset=0):
    """[steps][n] float32 standard normals of one factor, as the GPU draws them."""
    gid = np.arange(n_paths, dtype=np.uint64) + np.uint64(path_offset)
    c0 = (gid & mc_ref.MASK).astype(np.uint32)
    c1 = (gid >> np.uint64(32)).astype(np.uint32)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    z = np.zeros((steps, n_paths), dtype=np.float32)
    for t0 in range(0, steps, 4):
        x = mc_ref.philox4x32_10(c0, c1, np.uint32(t0 >> 2), np.uint32(factor << 8), k0, k1)
        z0, z1 = mc_ref.box_muller(x[0], x[1])
        z2, z3 = mc_ref.box_muller(x[2], x[3])
        for j, v in enumerate((z0, z1, z2, z3)):
            if t0 + j < steps:
                z[t0 + j] = v
    return z


def joint_walk(inc64, s0, qty):
    """inc64: [S][steps][n] float64 log increments -> (finals V_T, maxdd, asset_finals [S][n]), float32 like the GPU."""
    s0 = np.asarray(s0, dtype=np.float64)
    qty = np.asarray(qty, dtype=np.float64)
    S, _, n = inc64.shape
    logS = np.concatenate([np.zeros((S, 1, n)), np.cumsum(inc64, axis=1)], axis=1)
    a = qty * s0
    V = np.zeros(logS.shape[1:])
    for i in range(S):
        V += a[i] * np.exp(logS[i])
    runmax = np.maximum.accumulate(V, axis=0)
    maxdd = ((runmax - V) / runmax).max(axis=0).astype(np.float32)
    asset_finals = np.stack([(s0[i] * np.exp(logS[i, -1])).astype(np.float32) for i in range(S)])
    return V[-1].astype(np.float32), maxdd, asset_finals


def joint_gbm_paths(s0, qty, mu, sigma, dt, chol, n_paths, steps, seed, path_offset=0):
    """Asset i moves by drift_i + vol_i (L z)_i; L is used at the fp32 precision the kernel receives it in."""
    mu = np.atleast_1d(np.asarray(mu, dtype=np.float64))
    sigma = np.atleast_1d(np.asarray(sigma, dtype=np.float64))
    S = len(mu)
    drift = (mu - 0.5 * sigma * sigma) * dt
    vol = sigma * np.sqrt(dt)
    L = np.tril(np.asarray(chol, dtype=np.float32).reshape(S, S)).astype(np.float64)
    z = np.stack([normals(k, n_paths, steps, seed, path_offset) for k in range(S)]).astype(np.float64)
    y = np.stack([sum(L[i, k] * z[k] for k in range(i + 1)) for i in range(S)]) if S else z
    return joint_walk(drift[:, None, None] + vol[:, None, None] * y, s0, qty)


def bootstrap_days(R, n_paths, steps, seed, path_offset=0, block_len=1):
    """[steps][n] row indices: bootstrap_paths' index stream (its table replaced by the row numbers)."""
    rows = np.arange(R, dtype=np.float32)
    return mc_ref._increments(1, n_paths, steps, seed, path_offset, rows, block_len, True).astype(np.int64)


def joint_bootstrap_paths(returns, log_returns, s0, qty, n_paths, steps, seed, path_offset=0, block_len=1):
    """Each step applies ONE day's row of `returns` [R][S] to every asset.  -> (finals, maxdd, asset_finals, days)."""
    table = np.asarray(returns, dtype=np.float32)
    staged = table if log_returns else np.log1p(table).astype(np.float32)
    days = bootstrap_days(len(table), n_paths, steps, seed, path_offset, block_len)
    inc = np.transpose(staged[days], (2, 0, 1)).astype(np.float64)      # [S][steps][n]
    return (*joint_walk(inc, s0, qty), days)
