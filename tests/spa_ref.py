"""CPU restatements of the data-snooping tests (csrc/overfitting.cu b200bt_spa_moments / b200bt_spa_bootstrap and
ai_crypto_trader_b200.overfitting.spa).

* exact: the kernels' index stream drawn with oracle.mc_ref.philox4x32_10, and every sum an explicit loop in ascending
  t (or lag) vectorised only across trials, lags and resamples, so the means, variance estimates and bootstrap maxima
  are bit-identical to the device's.
* literal: White's Reality Check (2000), Hansen's SPA (2005) and Romano and Wolf's StepM (2005) as the papers write
  them, with np.mean and an index stream of plain Python, independent of the exact path's vectorisation.
"""
from __future__ import annotations

import math

import numpy as np

from ai_crypto_trader_b200.overfitting import spa_shifts, spa_summary
from oracle.mc_ref import philox4x32_10


def index_stream(T: int, q32: int, seed: int, gids) -> np.ndarray:
    """theta [len(gids)][T] (int64): the stationary-bootstrap day indices of the global resamples `gids`."""
    gid = np.asarray(gids, dtype=np.uint64)
    pairs = np.arange((T + 1) // 2, dtype=np.uint64)
    c0 = (gid & np.uint64(0xFFFFFFFF))[:, None]
    c1 = (gid >> np.uint64(32))[:, None]
    x = philox4x32_10(c0, c1, pairs[None, :], np.uint64(0), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    restart = np.stack([x[0], x[2]], axis=2).reshape(len(gid), -1)[:, :T].astype(np.uint64)
    start = np.stack([x[1], x[3]], axis=2).reshape(len(gid), -1)[:, :T].astype(np.uint64)
    begins = restart < np.uint64(q32)
    begins[:, 0] = True
    s = ((start * np.uint64(T)) >> np.uint64(32)).astype(np.int64)
    theta = np.empty((len(gid), T), dtype=np.int64)
    theta[:, 0] = s[:, 0]
    for t in range(1, T):
        nxt = theta[:, t - 1] + 1
        theta[:, t] = np.where(begins[:, t], s[:, t], np.where(nxt == T, 0, nxt))
    return theta


def block_starts(T: int, q32: int, seed: int, gids) -> np.ndarray:
    """bool [len(gids)][T]: the days that start a block (day 0 always)."""
    gid = np.asarray(gids, dtype=np.uint64)
    pairs = np.arange((T + 1) // 2, dtype=np.uint64)
    x = philox4x32_10((gid & np.uint64(0xFFFFFFFF))[:, None], (gid >> np.uint64(32))[:, None], pairs[None, :],
                      np.uint64(0), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    restart = np.stack([x[0], x[2]], axis=2).reshape(len(gid), -1)[:, :T].astype(np.uint64)
    out = restart < np.uint64(q32)
    out[:, 0] = True
    return out


def moments_exact(d: np.ndarray, q: float):
    """(mean, omega2) [N] of b200bt_spa_moments, bit for bit."""
    d = np.asarray(d, dtype=np.float64)
    N, T = d.shape
    nt = float(T)
    s = np.zeros(N)
    for t in range(T):
        s = s + d[:, t]
    mean = s / nt
    c = d - mean[:, None]
    acc = np.zeros((N, T))
    for t in range(T):                       # lag i gets c_t * c_{t+i} for every t <= T-1-i, in ascending t
        acc[:, :T - t] = acc[:, :T - t] + c[:, t:t + 1] * c[:, t:]
    gam = acc / nt
    a = 1.0 - q
    p = [1.0]
    for _ in range(T):
        p.append(p[-1] * a)
    p = np.array(p)
    i = np.arange(1, T)
    kappa = (T - i) / nt * p[i] + i / nt * p[T - i]
    terms = kappa[None, :] * gam[:, 1:]
    tot = np.zeros(N)
    for j in range(T - 1):
        tot = tot + terms[:, j]
    return mean, gam[:, 0] + 2.0 * tot


def boot_means_exact(d: np.ndarray, theta: np.ndarray) -> np.ndarray:
    """m* [N][B]: (sum_t d[k][theta_b(t)]) / T, summed in ascending t."""
    d = np.asarray(d, dtype=np.float64)
    T = d.shape[1]
    acc = np.zeros((d.shape[0], theta.shape[0]))
    for t in range(T):
        acc = acc + d[:, theta[:, t]]
    return acc / float(T)


def maxima_exact(d, q32, seed, boot_offset, n_boot, shift, scale) -> np.ndarray:
    """out [n_stats][n_boot] of b200bt_spa_bootstrap, bit for bit."""
    d = np.asarray(d, dtype=np.float64)
    theta = index_stream(d.shape[1], q32, seed, np.arange(n_boot, dtype=np.uint64) + np.uint64(boot_offset))
    m = boot_means_exact(d, theta)
    return maxima_of_means(m, shift, scale)


def maxima_of_means(m, shift, scale) -> np.ndarray:
    shift, scale = np.atleast_2d(shift), np.atleast_2d(scale)
    out = np.empty((shift.shape[0], m.shape[1]))
    with np.errstate(invalid="ignore"):
        for j in range(shift.shape[0]):
            v = (m - shift[j][:, None]) * scale[j][:, None]
            v[shift[j] == np.inf] = -np.inf
            v = np.where(np.isnan(v), -np.inf, v)
            out[j] = v.max(axis=0)
    return out


def spa_exact(d, n_boot, block_len, alpha, seed, q32=None, moments=None) -> dict:
    """overfitting.spa restated on the exact paths: the moments (or the given (mean, omega2)), the maxima of every
    launch, and spa_summary's statistics."""
    from ai_crypto_trader_b200.overfitting import spa_q32
    d = np.asarray(d, dtype=np.float64)
    T = d.shape[1]
    q32 = spa_q32(block_len) if q32 is None else q32
    mean, omega2 = moments if moments is not None else moments_exact(d, q32 / 2.0 ** 32)
    omega = np.where(omega2 > 0, np.sqrt(np.where(omega2 > 0, omega2, 1.0)), np.nan)
    theta = index_stream(T, q32, seed, np.arange(n_boot, dtype=np.uint64))
    m = boot_means_exact(d, theta)
    shift, scale = spa_shifts(mean, omega, T)
    out = maxima_of_means(m, shift, scale)
    res = spa_summary(mean, omega, T, out, lambda active: maxima_of_means(m, np.where(active, mean, np.inf),
                                                                           scale[1])[0], alpha)
    res.update(mean=mean, omega=omega, out=out)
    return res


# ---- literal ---------------------------------------------------------------------------------------------------------

def stationary_indices(T: int, q32: int, seed: int, gid: int) -> list:
    """One resample's indices, walked day by day in plain Python integers (Philox words from the same generator)."""
    P = (T + 1) // 2
    words = philox4x32_10(np.full(P, gid & 0xFFFFFFFF), np.full(P, gid >> 32), np.arange(P), 0, seed & 0xFFFFFFFF,
                          (seed >> 32) & 0xFFFFFFFF)
    x = [[int(v) for v in w] for w in words]
    th = []
    for t in range(T):
        restart, start = x[2 * (t & 1)][t >> 1], x[2 * (t & 1) + 1][t >> 1]
        if t == 0 or restart < q32:
            th.append(start * T >> 32)
        else:
            th.append((th[-1] + 1) % T)
    return th


def hansen_omega2(x: np.ndarray, q: float) -> float:
    """Hansen (2005) eq. for the stationary-bootstrap variance of sqrt(T) * mean, kappa by pow."""
    T = len(x)
    c = x - np.mean(x)
    g = [np.dot(c[:T - i], c[i:]) / T for i in range(T)]
    k = [((T - i) / T) * (1 - q) ** i + (i / T) * (1 - q) ** (T - i) for i in range(T)]
    return g[0] + 2 * sum(k[i] * g[i] for i in range(1, T))


def spa_literal(d, n_boot, block_len, alpha, seed) -> dict:
    """The three tests as written, with np.mean on each resample (indices from stationary_indices)."""
    from ai_crypto_trader_b200.overfitting import spa_q32
    d = np.asarray(d, dtype=np.float64)
    N, T = d.shape
    q32 = spa_q32(block_len)
    q = q32 / 2.0 ** 32
    dbar = d.mean(axis=1)
    w2 = np.array([hansen_omega2(row, q) for row in d])
    ok = w2 > 0
    w = np.sqrt(np.where(ok, w2, 1.0))
    mstar = np.array([d[:, stationary_indices(T, q32, seed, b)].mean(axis=1) for b in range(n_boot)])   # [B][N]
    # Reality Check
    V = np.max(np.sqrt(T) * dbar)
    Vb = np.max(np.sqrt(T) * (mstar - dbar), axis=1)
    p_rc = np.mean(Vb > V)
    # SPA
    t = np.where(ok, np.sqrt(T) * dbar / w, -np.inf)
    T_spa = max(0.0, np.max(t)) if ok.any() else math.nan
    thr = math.sqrt(max(0.0, 2 * math.log(math.log(T)) / T)) if T > 2 else 0.0
    mu = {"lower": np.maximum(dbar, 0), "consistent": dbar * (dbar > -w * thr), "upper": dbar}
    p = {}
    for name, g in mu.items():
        Z = np.sqrt(T) * (mstar - g) / w
        Tb = np.maximum(0.0, np.max(np.where(ok, Z, -np.inf), axis=1))
        p[name] = np.mean(Tb > T_spa) if ok.any() else math.nan
    # StepM (studentized)
    rejected = np.zeros(N, dtype=bool)
    active = ok.copy()
    crit = []
    while active.any():
        Z = np.sqrt(T) * (mstar - dbar) / w
        mx = np.max(np.where(active, Z, -np.inf), axis=1)
        c = np.sort(mx)[math.ceil((1 - alpha) * n_boot) - 1]
        crit.append(c)
        new = active & (t > c)
        if not new.any():
            break
        rejected |= new
        active &= ~new
    return dict(mean=dbar, omega2=w2, reality_check=dict(stat=V, pvalue=p_rc),
                spa=dict(stat=T_spa, pvalue_lower=p["lower"], pvalue_consistent=p["consistent"],
                         pvalue_upper=p["upper"]),
                stepm=dict(rejected=rejected, critical_values=crit))
