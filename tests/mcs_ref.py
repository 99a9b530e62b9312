"""CPU restatements of the Model Confidence Set (csrc/overfitting.cu b200bt_boot_means / b200bt_autocov / b200bt_mcs_*,
ai_crypto_trader_b200.overfitting.mcs and optimal_block_length).

* exact: spa_ref.index_stream and explicit loops in the ascending orders of include/b200bt.h, vectorised only across
  models, pairs and resamples, so that every mean, variance, t-statistic, count and p-value is bit-identical to the
  device's.  The T_R bootstrap maxima are taken directly over the pairs of each M_k, not by the device's rank relabelling.
* literal: Hansen, Lunde and Nason (2011) as the paper writes the algorithm, with np.mean, the plain-Python
  spa_ref.stationary_indices and divisions by the standard deviations; and Politis and White's block-length rule step
  by step in plain Python.
"""
from __future__ import annotations

import math

import numpy as np

import spa_ref
from ai_crypto_trader_b200.overfitting import spa_q32


def pvalues(order, step_p, alpha):
    """MCS p-values by model: a running max of the step p-values along the order, 1 for the last survivor."""
    p = np.ones(len(order))
    for k in range(len(order) - 1):
        p[order[k]] = max(step_p[:k + 1])
    return p, p >= alpha


def expand(x, run, alpha):
    """Byte-identical rows are one model: run(models) on the distinct rows (first occurrences, ascending), then every
    row takes its model's p-value; elimination_order lists the rows of each model together."""
    x = np.asarray(x, dtype=np.float64)
    _, first, inverse = np.unique(x.view(np.uint64), axis=0, return_index=True, return_inverse=True)
    reps = np.sort(first)
    model_of = np.searchsorted(reps, first[inverse.ravel()])
    if len(reps) >= 2:
        res = run(x[reps])
    else:
        res = dict(elimination_order=np.zeros(1, dtype=np.int64), step_pvalues=np.empty(0), mean=mean_exact(x[reps]))
    p_m, _ = pvalues(res["elimination_order"], res["step_pvalues"], alpha)
    order = np.concatenate([np.flatnonzero(model_of == g) for g in res["elimination_order"]])
    out = dict(res, p_values=p_m[model_of], included=p_m[model_of] >= alpha, elimination_order=order,
               model_of=model_of, n_models=len(reps), mean=res["mean"][model_of])
    return out


def _zero_rule_t(dm, s):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(s > 0, dm / np.where(s > 0, s, 1.0), np.where(dm == 0, 0.0, np.where(dm > 0, np.inf, -np.inf)))


# ---- exact -----------------------------------------------------------------------------------------------------------

def mean_exact(x):
    x = np.asarray(x, dtype=np.float64)
    s = np.zeros(x.shape[0])
    for t in range(x.shape[1]):
        s = s + x[:, t]
    return s / float(x.shape[1])


def autocov_exact(x, K):
    """[N][K+1]: spa_moments' gamma_i for i = 0..K."""
    x = np.asarray(x, dtype=np.float64)
    N, T = x.shape
    c = x - mean_exact(x)[:, None]
    out = np.empty((N, K + 1))
    for i in range(K + 1):
        s = np.zeros(N)
        for t in range(T - i):
            s = s + c[:, t] * c[:, t + i]
        out[:, i] = s / float(T)
    return out


def boot_means_exact(x, q32, seed, n_boot, boot_offset=0):
    """m* [n_boot][N] of b200bt_boot_means (resample-major)."""
    x = np.asarray(x, dtype=np.float64)
    theta = spa_ref.index_stream(x.shape[1], q32, seed, np.arange(n_boot, dtype=np.uint64) + np.uint64(boot_offset))
    return spa_ref.boot_means_exact(x, theta).T


def zeta_exact(x, q32, seed, n_boot):
    mean = mean_exact(x)
    return mean, boot_means_exact(x, q32, seed, n_boot) - mean[None, :]


def range_stats_exact(zeta, mean):
    """(s2, rho, t) [N][N]: s2_ij = sum_b (zeta_bj - zeta_bi)^2 in ascending b, rho = 1 / sigma (0 at sigma = 0)."""
    B, N = zeta.shape
    s2 = np.zeros((N, N))
    for b in range(B):
        d = zeta[b][None, :] - zeta[b][:, None]
        s2 = s2 + d * d
    sigma = np.sqrt(s2 / float(B))
    with np.errstate(divide="ignore"):
        rho = np.where(sigma > 0, 1.0 / np.where(sigma > 0, sigma, 1.0), 0.0)
    t = _zero_rule_t(mean[None, :] - mean[:, None], sigma)
    np.fill_diagonal(rho, 0.0)
    np.fill_diagonal(t, 0.0)
    return s2, rho, t


def mcs_range_exact(zeta, mean):
    """(order, stats, counts) of T_R."""
    B, N = zeta.shape
    _, rho, t = range_stats_exact(zeta, mean)
    alive = list(range(N))
    order, stats, counts = [], [], []
    for _ in range(N - 1):
        M = np.array(alive)
        rm = t[np.ix_(M, M)].max(axis=1)
        k = int(np.argmax(rm))
        T_R = rm[k]
        zm = zeta[:, M]
        tstar = np.zeros(B)
        for a in range(len(M)):
            tstar = np.maximum(tstar, (np.abs(zm - zm[:, a:a + 1]) * rho[M[a], M][None, :]).max(axis=1))
        order.append(int(M[k]))
        stats.append(T_R)
        counts.append(int(np.count_nonzero(tstar >= T_R)))
        alive.remove(int(M[k]))
    order.append(alive[0])
    return np.array(order), np.array(stats), np.array(counts)


def mcs_max_exact(zeta, mean):
    """(order, stats, counts) of T_max."""
    B, N = zeta.shape
    alive = list(range(N))
    order, stats, counts = [], [], []
    for _ in range(N - 1):
        M = np.array(alive)
        m = len(M)
        acc = np.zeros(B)
        for j in M:
            acc = acc + zeta[:, j]
        zbar = acc / float(m)
        v = np.zeros(m)
        for b in range(B):
            d = zbar[b] - zeta[b, M]
            v = v + d * d
        s = np.sqrt(v / float(B))
        xs = 0.0
        for j in M:
            xs = xs + mean[j]
        xm = xs / float(m)
        t = _zero_rule_t(xm - mean[M], s)
        k = int(np.argmax(t))
        with np.errstate(divide="ignore", invalid="ignore"):
            terms = np.where(s[None, :] > 0, (zbar[:, None] - zeta[:, M]) / np.where(s > 0, s, 1.0)[None, :], 0.0)
        tstar = terms.max(axis=1)
        order.append(int(M[k]))
        stats.append(t[k])
        counts.append(int(np.count_nonzero(tstar >= t[k])))
        alive.remove(int(M[k]))
    order.append(alive[0])
    return np.array(order), np.array(stats), np.array(counts)


def mcs_exact(x, alpha=0.10, statistic="R", n_boot=1000, block_len=10.0, seed=0):
    """overfitting.mcs restated on the exact paths (a numeric block_len), copies collapsed into one model."""
    def run(models):
        mean, zeta = zeta_exact(models, spa_q32(block_len), seed, n_boot)
        order, stats, counts = (mcs_range_exact if statistic == "R" else mcs_max_exact)(zeta, mean)
        return dict(elimination_order=order, step_stats=stats, step_pvalues=counts / float(n_boot), mean=mean)

    return expand(x, run, alpha)


# ---- literal ---------------------------------------------------------------------------------------------------------

def mcs_literal(x, alpha=0.10, statistic="R", n_boot=1000, block_len=10.0, seed=0):
    """HLN's MCS algorithm: test H0,M with T_R or T_max, eliminate e_M if rejected ... with p-values as max over the
    earlier steps, on np.mean bootstrap means.  Identical rows are one model (grouped by their bytes in plain Python)."""
    x = np.asarray(x, dtype=np.float64)
    groups = {}
    for i, r in enumerate(x):
        groups.setdefault(r.tobytes(), []).append(i)
    members = sorted(groups.values())
    if len(members) == 1:
        p = np.ones(len(x))
        return dict(p_values=p, included=p >= alpha, elimination_order=np.arange(len(x)), step_pvalues=np.empty(0),
                    mean=np.mean(x, axis=1))
    res = _literal_models(x[[g[0] for g in members]], alpha, statistic, n_boot, block_len, seed)
    p = np.empty(len(x))
    for g, rows in enumerate(members):
        p[rows] = res["p_values"][g]
    order = np.array([i for g in res["elimination_order"] for i in members[g]])
    return dict(p_values=p, included=p >= alpha, elimination_order=order, step_pvalues=res["step_pvalues"],
                mean=np.mean(x, axis=1))


def _literal_models(x, alpha, statistic, n_boot, block_len, seed):
    N, T = x.shape
    q32 = spa_q32(block_len)
    dbar = np.mean(x, axis=1)
    mstar = np.array([x[:, spa_ref.stationary_indices(T, q32, seed, b)].mean(axis=1) for b in range(n_boot)])
    zeta = mstar - dbar[None, :]
    M = list(range(N))
    elim, pvals = [], []
    while len(M) > 1:
        Z, d = zeta[:, M], dbar[M]
        if statistic == "R":
            var = np.array([[np.mean((Z[:, j] - Z[:, i]) ** 2) for j in range(len(M))] for i in range(len(M))])
            sd = np.sqrt(var)
            t = _zero_rule_t(d[None, :] - d[:, None], sd)
            stat = t.max()
            e = int(np.argmax(t.max(axis=1)))
            with np.errstate(divide="ignore", invalid="ignore"):
                tb = np.where(sd[None] > 0, np.abs(Z[:, None, :] - Z[:, :, None]) / np.where(sd > 0, sd, 1.0)[None], 0.0)
            tstar = tb.reshape(n_boot, -1).max(axis=1)
        else:
            zbar = Z.mean(axis=1)
            var = np.mean((zbar[:, None] - Z) ** 2, axis=0)
            sd = np.sqrt(var)
            t = _zero_rule_t(np.mean(d) - d, sd)
            stat = t.max()
            e = int(np.argmax(t))
            with np.errstate(divide="ignore", invalid="ignore"):
                tstar = np.where(sd[None] > 0, (zbar[:, None] - Z) / np.where(sd > 0, sd, 1.0)[None], 0.0).max(axis=1)
        pvals.append(np.mean(tstar >= stat))
        elim.append(M.pop(e))
    order = np.array(elim + M)
    p = np.ones(N)
    running = 0.0
    for k, e in enumerate(elim):
        running = max(running, pvals[k])
        p[e] = running
    return dict(p_values=p, included=p >= alpha, elimination_order=order, step_pvalues=np.array(pvals), mean=dbar)


def block_length_literal(row):
    """Politis and White (2004) / Patton, Politis and White (2009) for one row, step by step."""
    x = np.asarray(row, dtype=np.float64)
    T = len(x)
    c = x - np.mean(x)

    def R(k):
        return float(np.dot(c[:T - k], c[k:])) / T if k < T else 0.0

    if R(0) == 0.0:
        return math.nan
    KN = max(5, math.ceil(math.sqrt(math.log10(T))))
    m_max = math.ceil(math.sqrt(T)) + KN
    b_max = math.ceil(min(3 * math.sqrt(T), T / 3))
    crit = 2 * math.sqrt(math.log10(T) / T)
    m_hat = m_max
    for m in range(m_max + 1):
        if all(abs(R(m + j) / R(0)) < crit for j in range(1, KN + 1)):
            m_hat = m
            break
    M = min(2 * max(m_hat, 1), m_max)

    def lam(s):
        s = abs(s)
        return 1.0 if s <= 0.5 else (2 * (1 - s) if s <= 1 else 0.0)

    g = R(0) + 2 * sum(lam(k / M) * R(k) for k in range(1, M + 1))
    G = 2 * sum(lam(k / M) * k * R(k) for k in range(1, M + 1))
    b = b_max if g == 0 else (2 * G ** 2 / (2 * g ** 2)) ** (1 / 3) * T ** (1 / 3)
    return min(max(b, 1.0), b_max)
