"""The contract of b200bt_pareto_rank (include/b200bt.h) restated on the host, in three forms.

pareto_exact    the contract with plain Python floats and ascending loops: every float64 operation is one IEEE
                operation in a fixed order, so its results are the kernel's bit for bit.
pareto_numpy    the same contract vectorised, for sizes the pure-Python form cannot reach: the dominance relation built in
                row blocks and kept bit-packed (n^2 / 8 bytes), Deb's counting peel (a chain of n fronts is n vector steps),
                crowding as a loop over objectives of elementwise float64 operations, which round like the scalar form.
fast_nondominated_sort_literal
                Deb, Pratap, Agarwal, Meyarivan 2002 (NSGA-II, section III-A and III-B) as the paper gives it, on
                minimised objectives; a cross-check of the fronts that shares no code with the other two.

Each returns (front int32 [n], crowding float64 [n], order int32 [n], key float64 [n]) -- the literal form returns
(front, crowding) only.
"""
from __future__ import annotations

import math
import operator
from typing import List, Sequence, Tuple

import numpy as np


def _matrix(obj, maximize) -> Tuple[np.ndarray, List[bool]]:
    obj = np.asarray(obj, dtype=np.float64)
    if obj.ndim == 1:
        obj = obj[:, None]
    mx = [bool(m) for m in maximize]
    if len(mx) != obj.shape[1]:
        raise ValueError("one direction per objective")
    return obj, mx


def values(obj, maximize) -> np.ndarray:
    """v[p][j] = maximize_j ? obj[p][j] : -obj[p][j], NaN -> -inf (larger is better)."""
    obj, mx = _matrix(obj, maximize)
    v = np.where(np.array(mx)[None, :], obj, -obj)
    return np.where(np.isnan(v), -np.inf, v)


def _order_and_key(front: Sequence[int], crowd: Sequence[float]):
    n = len(front)
    order = sorted(range(n), key=lambda p: (front[p], -crowd[p], p))
    key = [0.0] * n
    for pos, p in enumerate(order):
        key[p] = float(-pos)
    return np.array(order, dtype=np.int32), np.array(key, dtype=np.float64)


# -- the scalar form ----------------------------------------------------------------------------------------------------
def pareto_exact(obj, maximize):
    obj, mx = _matrix(obj, maximize)
    n, M = obj.shape
    v = []
    for p in range(n):
        row = []
        for j in range(M):
            x = float(obj[p, j])
            y = x if mx[j] else -x
            row.append(-math.inf if math.isnan(y) else y)
        v.append(tuple(row))
    # dominance: p dominates q iff v[p] >= v[q] everywhere and not v[q] >= v[p] everywhere
    dominates: List[List[int]] = [[] for _ in range(n)]
    count = [0] * n
    for p in range(n):
        vp = v[p]
        for q in range(p + 1, n):
            vq = v[q]
            pq = all(map(operator.ge, vp, vq))
            qp = all(map(operator.ge, vq, vp))
            if pq and not qp:
                dominates[p].append(q)
                count[q] += 1
            elif qp and not pq:
                dominates[q].append(p)
                count[p] += 1
    front = [-1] * n
    current = [p for p in range(n) if count[p] == 0]
    fronts = []
    k = 0
    while current:
        for p in current:
            front[p] = k
        fronts.append(current)
        nxt = []
        for p in current:
            for q in dominates[p]:
                count[q] -= 1
                if count[q] == 0:
                    nxt.append(q)
        current = sorted(nxt)
        k += 1
    crowd = [0.0] * n
    for F in fronts:
        for j in range(M):
            s = sorted(F, key=lambda p: (v[p][j], p))
            r = v[s[-1]][j] - v[s[0]][j]
            use = r != 0.0 and math.isfinite(r)
            for i, p in enumerate(s):
                if i == 0 or i == len(s) - 1:
                    crowd[p] = crowd[p] + math.inf
                elif use:
                    crowd[p] = crowd[p] + (v[s[i + 1]][j] - v[s[i - 1]][j]) / r
    order, key = _order_and_key(front, crowd)
    return np.array(front, dtype=np.int32), np.array(crowd, dtype=np.float64), order, key


# -- the vectorised form ------------------------------------------------------------------------------------------------
def dominance_bits(v: np.ndarray, block: int = 64) -> Tuple[np.ndarray, np.ndarray]:
    """(bits uint8 [n][ceil(n / 8)], bit q of row p (little-endian bit order) set iff p dominates q; count int64 [n], the
    number of points dominating each point)."""
    n, M = v.shape
    bits = np.zeros((n, (n + 7) // 8), dtype=np.uint8)
    count = np.zeros(n, dtype=np.int64)
    for lo in range(0, n, block):
        hi = min(n, lo + block)
        a = v[lo:hi]
        pq = np.ones((hi - lo, n), dtype=bool)            # v[p] >= v[q] for every objective
        qp = np.ones((hi - lo, n), dtype=bool)            # v[q] >= v[p] for every objective
        for j in range(M):
            pq &= a[:, j, None] >= v[None, :, j]
            qp &= v[None, :, j] >= a[:, j, None]
        dom = pq & ~qp
        bits[lo:hi] = np.packbits(dom, axis=1, bitorder="little")
        count += dom.sum(axis=0)
    return bits, count


def fronts_numpy(v: np.ndarray, rows: int = 1024) -> np.ndarray:
    """Deb's counting peel over the packed relation: one vector step per front."""
    n = v.shape[0]
    bits, count = dominance_bits(v)
    front = np.full(n, -1, dtype=np.int32)
    current = np.flatnonzero(count == 0)
    k = 0
    while current.size:
        front[current] = k
        dec = np.zeros(n, dtype=np.int64)
        for lo in range(0, current.size, rows):
            dec += np.unpackbits(bits[current[lo:lo + rows]], axis=1, count=n, bitorder="little").sum(axis=0,
                                                                                                     dtype=np.int64)
        count -= dec
        current = np.flatnonzero((count == 0) & (dec > 0))
        k += 1
    return front


def crowding_numpy(v: np.ndarray, front: np.ndarray) -> np.ndarray:
    n, M = v.shape
    idx = np.arange(n)
    d = np.zeros(n, dtype=np.float64)
    for j in range(M):
        s = np.lexsort((idx, v[:, j], front))           # (front, v_j, index) ascending
        f, x = front[s], v[s, j]
        first = np.ones(n, dtype=bool)
        first[1:] = f[1:] != f[:-1]
        last = np.ones(n, dtype=bool)
        last[:-1] = f[:-1] != f[1:]
        seg = np.cumsum(first) - 1                       # segment of each sorted slot
        starts = np.flatnonzero(first)
        ends = np.flatnonzero(last)
        with np.errstate(invalid="ignore", over="ignore"):
            r = (x[ends] - x[starts])[seg]
        prev = np.concatenate(([0.0], x[:-1]))
        nxt = np.concatenate((x[1:], [0.0]))
        boundary = first | last
        use = ~boundary & (r != 0.0) & np.isfinite(r)
        add = np.zeros(n, dtype=np.float64)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            add[use] = (nxt[use] - prev[use]) / r[use]
        add[boundary] = np.inf
        contrib = np.empty(n, dtype=np.float64)
        contrib[s] = add
        d = d + contrib
    return d


def pareto_numpy(obj, maximize):
    v = values(obj, maximize)
    front = fronts_numpy(v)
    crowd = crowding_numpy(v, front)
    n = v.shape[0]
    order = np.lexsort((np.arange(n), -crowd, front)).astype(np.int32)
    key = np.empty(n, dtype=np.float64)
    key[order] = -np.arange(n, dtype=np.float64)
    key[order[0]] = 0.0
    return front, crowd, order, key


# -- Deb 2002 as the paper gives it -------------------------------------------------------------------------------------
def fast_nondominated_sort_literal(obj, maximize):
    """fast-non-dominated-sort and crowding-distance-assignment (NSGA-II, section III) on minimised objectives f = -v."""
    f = -values(obj, maximize)
    n, M = f.shape
    pop = range(n)

    def dominates(p, q):           # p is no worse in every objective and better in one (minimisation)
        return all(f[p, m] <= f[q, m] for m in range(M)) and any(f[p, m] < f[q, m] for m in range(M))

    S = [[] for _ in pop]
    cnt = [0] * n
    F = [[]]
    rank = [0] * n
    for p in pop:
        for q in pop:
            if dominates(p, q):
                S[p].append(q)
            elif dominates(q, p):
                cnt[p] += 1
        if cnt[p] == 0:
            rank[p] = 0
            F[0].append(p)
    i = 0
    while F[i]:
        Q = []
        for p in F[i]:
            for q in S[p]:
                cnt[q] -= 1
                if cnt[q] == 0:
                    rank[q] = i + 1
                    Q.append(q)
        i += 1
        F.append(Q)
    dist = [0.0] * n
    for I in F[:-1]:
        l = len(I)
        for m in range(M):
            I = sorted(I, key=lambda p: f[p, m])
            dist[I[0]] = dist[I[l - 1]] = math.inf
            with np.errstate(invalid="ignore"):
                span = f[I[l - 1], m] - f[I[0], m]
            for k in range(1, l - 1):
                if span > 0 and math.isfinite(span):
                    dist[I[k]] += (f[I[k + 1], m] - f[I[k - 1], m]) / span
    return np.array(rank, dtype=np.int32), np.array(dist, dtype=np.float64)


# -- inputs the tests draw ----------------------------------------------------------------------------------------------
KINDS = ("uniform", "ties", "anti", "chain", "equal", "nonfinite", "mixed")


def make_input(kind: str, n: int, M: int, seed: int = 0):
    """(obj [n][M] float64, maximize [M]) of one input kind."""
    rng = np.random.default_rng([seed, n, M, KINDS.index(kind)])
    maximize = [True] * M
    if kind == "uniform":
        obj = rng.random((n, M))
    elif kind == "ties":                              # small-range integers: ties and duplicate rows
        obj = rng.integers(0, 4, (n, M)).astype(np.float64)
    elif kind == "anti":                              # objectives that trade off: most points in one front
        t = rng.random(n)
        obj = np.stack([t if j % 2 == 0 else 1.0 - t for j in range(M)], axis=1) + 1e-3 * rng.random((n, M))
        if M == 1:
            obj = t[:, None]
    elif kind == "chain":                             # perfectly correlated: n fronts
        t = rng.permutation(n).astype(np.float64)
        obj = np.stack([t * (j + 1) for j in range(M)], axis=1)
    elif kind == "equal":
        obj = np.full((n, M), 0.25)
    elif kind == "nonfinite":
        obj = rng.integers(-3, 4, (n, M)).astype(np.float64)
        pick = rng.random((n, M))
        obj[pick < 0.1] = np.nan
        obj[(pick >= 0.1) & (pick < 0.15)] = np.inf
        obj[(pick >= 0.15) & (pick < 0.2)] = -np.inf
        obj[(pick >= 0.2) & (pick < 0.25)] = -0.0
    elif kind == "mixed":
        obj = np.round(rng.normal(size=(n, M)), 2)
        maximize = [j % 2 == 0 for j in range(M)]
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(obj), maximize
