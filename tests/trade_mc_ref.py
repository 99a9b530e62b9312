"""Float64 NumPy restatement of the trade-sequence Monte-Carlo (csrc/trade_mc.cu), for the tests and smoke().

  * `trips_from_records`: (fee, trip PnL) of a lane from its trade records (oracle/simulate_ref.simulate_trades or
    StrategyEvaluationSystem._simulate_trades): entry records carry pnl -fee, exit records the trip's pnl.
  * `bootstrap_indices`, `shuffle_indices`: the index streams, on oracle/mc_ref's Philox4x32-10 and its block rule,
    and the keyed Feistel bijection.
  * `walk`: the LITERAL per-record equity and drawdown rule of calculate_metrics (strategy_evaluation.py:119-139), one
    record at a time -- not the kernel's closed form, so that the tests check the closed form.
  * `simulate`: all of it, rounded once to fp32 as the kernel stores it.
  * `statistics`: the result blocks of StrategyEvaluationSystem.monte_carlo_trades with the reference's NumPy calls
    (monte_carlo_service.py:305-336 via oracle/mc_ref.risk_statistics, equity for price, plus the 95th percentile of
    the maximum drawdown).
"""
from __future__ import annotations

import numpy as np

from oracle import mc_ref

MASK = np.uint64(0xFFFFFFFF)
SHUFFLE_BLOCK = 0xFFFFFFFE        # round keys: the first words of the Philox blocks SHUFFLE_BLOCK, SHUFFLE_BLOCK + 1


def trips_from_records(records):
    """-> (fee, float64 trip PnL array) of a record list in entry / exit pairs."""
    assert len(records) % 2 == 0
    entries = [r["pnl"] for r in records[0::2]]
    fee = -entries[0] if entries else 0.0
    assert all(-e == fee for e in entries)
    return fee, np.array([r["pnl"] for r in records[1::2]], dtype=np.float64)


def net_profit(fee, trips):
    """calculate_metrics' net profit (:93-98): sum of the winning records plus sum of the losing ones, in record order."""
    pnl = []
    for t in np.asarray(trips, dtype=np.float64).tolist():
        pnl += [-fee, t]
    return sum(p for p in pnl if p > 0) + sum(p for p in pnl if p < 0)


def _counters(n_paths, path_offset):
    gid = np.arange(n_paths, dtype=np.uint64) + np.uint64(path_offset)
    return (gid & MASK).astype(np.uint32), (gid >> np.uint64(32)).astype(np.uint32)


def bootstrap_indices(T, n_paths, seed, lane_id=0, path_offset=0, block_len=1):
    """[n_paths][T] trip indices: b200bt_mc_bootstrap's draw and circular block rule, counter (gid, trip / 4, lane id)."""
    c0, c1 = _counters(n_paths, path_offset)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    out = np.zeros((n_paths, T), dtype=np.int64)
    idx = np.zeros(n_paths, dtype=np.int64)
    left = np.zeros(n_paths, dtype=np.int64)
    for t0 in range(0, T, 4):
        x = mc_ref.philox4x32_10(c0, c1, np.uint32(t0 >> 2), np.uint32(lane_id), k0, k1)
        for j in range(4):
            if t0 + j >= T:
                break
            fresh = left == 0
            start = ((x[j].astype(np.uint64) * np.uint64(T)) >> np.uint64(32)).astype(np.int64)
            nxt = np.where(idx + 1 == T, 0, idx + 1)
            idx = np.where(fresh, start, nxt)
            left = np.where(fresh, block_len, left) - 1
            out[:, t0 + j] = idx
    return out


FEISTEL_ROUNDS, FEISTEL_MIN_HALF = 6, 4


def feistel_half_bits(T):
    b = int(T - 1).bit_length() if T > 1 else 0
    return (b + 1) // 2 if b > 2 * FEISTEL_MIN_HALF else FEISTEL_MIN_HALF


def feistel(v, keys, h):
    """Balanced Feistel on 2h bits, one round per key; v uint64 array, keys uint64 arrays (one round key per path)."""
    mask = np.uint64((1 << h) - 1)
    L, R = v >> np.uint64(h), v & mask
    for k in keys:
        y = ((R ^ k) * np.uint64(0x9E3779B1)) & MASK
        y ^= y >> np.uint64(15)
        y = (y * np.uint64(0x85EBCA77)) & MASK
        L, R = R, L ^ (y >> np.uint64(32 - h))
    return (L << np.uint64(h)) | R


def shuffle_indices(T, n_paths, seed, lane_id=0, path_offset=0):
    """[n_paths][T]: position j holds pi(j), the path's Feistel bijection cycle-walked into [0, T)."""
    c0, c1 = _counters(n_paths, path_offset)
    keys = [k.astype(np.uint64) for b in (SHUFFLE_BLOCK, SHUFFLE_BLOCK + 1) for k in
            mc_ref.philox4x32_10(c0, c1, np.uint32(b), np.uint32(lane_id), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)]
    keys = keys[:FEISTEL_ROUNDS]
    h = feistel_half_bits(max(T, 1))
    out = np.zeros((n_paths, T), dtype=np.int64)
    step = max(1, (1 << 22) // max(T, 1))                 # paths per block of at most ~4M indices
    for a in range(0, n_paths, step):
        k = [key[a:a + step, None] for key in keys]
        v = feistel(np.tile(np.arange(T, dtype=np.uint64), (len(k[0]), 1)), k, h)
        while True:
            out_of_range = v >= np.uint64(T)
            if not out_of_range.any():
                break
            v = np.where(out_of_range, feistel(v, k, h), v)
        out[a:a + step] = v.astype(np.int64)
    return out


def walk(fee, trips, idx, initial_capital=10000.0):
    """Per-record equity walk of every path (rows of idx): -> (final equity, max drawdown), float64."""
    trips = np.asarray(trips, dtype=np.float64)
    n = idx.shape[0]
    E = np.full(n, float(initial_capital))
    peak = E.copy()
    dd = np.zeros(n)
    for j in range(idx.shape[1]):
        for x in (np.full(n, -fee), trips[idx[:, j]]):
            E = E + x
            new = E > peak                       # :139-144
            dd = np.where(new, dd, np.maximum(dd, (peak - E) / peak))
            peak = np.where(new, E, peak)
    return E, dd


def indices(method, T, n_paths, seed, lane_id=0, path_offset=0, block_len=1):
    if method == "bootstrap":
        return bootstrap_indices(T, n_paths, seed, lane_id, path_offset, block_len)
    if method == "shuffle":
        return shuffle_indices(T, n_paths, seed, lane_id, path_offset)
    raise ValueError(method)


def simulate(fee, trips, n_paths, seed, method="bootstrap", lane_id=0, path_offset=0, block_len=1,
             initial_capital=10000.0):
    """-> (finals fp32 [n_paths], maxdd fp32 [n_paths]) as b200bt_trade_mc stores them for one lane."""
    idx = indices(method, len(trips), n_paths, seed, lane_id, path_offset, block_len)
    E, dd = walk(fee, trips, idx, initial_capital)
    return E.astype(np.float32), dd.astype(np.float32)


def statistics(finals, maxdd, initial_capital, confidence):
    """percentiles / expected / risk_metrics blocks of monte_carlo_trades, with np.percentile."""
    st = mc_ref.risk_statistics(finals, maxdd, initial_capital, confidence)
    md = np.asarray(maxdd, dtype=np.float64)
    rm = dict(st["risk_metrics"])
    rm["max_drawdown"] = dict(rm["max_drawdown"], p95=float(np.percentile(md, 95)))
    return {
        "percentiles": {k: {"equity": v["price"], "pct_change": v["pct_change"]} for k, v in st["percentiles"].items()},
        "expected": {"equity": st["expected"]["price"], "pct_change": st["expected"]["pct_change"]},
        "risk_metrics": rm,
    }
