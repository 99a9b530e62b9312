"""The grid and DCA backtests at their limits on the H100, against the plain restatements: b200bt_grid_sweep and
b200bt_grid_service_sweep at the 2 048-tick price tile and the 32-tick pass seams, 16-warp CTAs, level tables of 1 .. 127
levels, fp32 index estimates far off or infinite, repeated levels, NaN closes, strided rows, label rows, other bar clocks
and the S limit; b200bt_dca_sweep at the 32 / 1 024 / 32 768-bar seams of its dip-search pyramid, over 2^20 bars, with
NaN dip runs, cooldown edges, other clocks and a rebalance on every tick.

Oracles: grid_ref.simulate (tick by tick) and grid_service_ref.simulate_service on short series, grid_ref.simulate_fast
on a long one, dca_ref.simulate (event-driven) for DCA.  Grid rules: the EXACT fields equal; profits within the
existing tolerance, and on arithmetic lanes (levels bit-equal to Python's) total profit within a relative tolerance with
no absolute floor, as it is a sum of non-negative steps; geometric lanes with near ties only bound the trade count.  DCA:
every field, service total and day row equal."""
import math

import numpy as np
import pytest

import dca_ref
import grid_ref
import grid_service_ref
from gpu_fixtures import torch_cuda  # noqa: F401
from test_gpu_dca import check as check_dca
from test_gpu_dca import market_of as dca_market
from test_gpu_grid import EXACT
from test_gpu_grid_service import SERVICE_EXACT

pytestmark = pytest.mark.gpu
M0 = 28_401_120                       # a UTC midnight
NEVER = 2 ** 31 - 1                   # a check period no series here reaches
PROFITS = ("total_profit", "cash", "profit_per_day", "mark_to_market", "win_rate")
FIELDS = grid_ref.FIELDS


def ind(n=10, kind=0, reb=NEVER, adj=NEVER, adapt=0, lo=3.0, up=3.0):
    """b200bt_grid_individual's fields (num_grids, grid_type, rebalance_ticks, adjust_ticks, flags, lower_pct, upper_pct)."""
    return (n, kind, reb, adj, adapt, lo, up)


def valid(iv):
    n, kind, reb, adj = iv[:4]
    return 1 <= n <= 127 and kind in (0, 1) and reb >= 1 and adj >= 1


def lattice(rng, N, p0=100.0, step=0.25, jump=6):
    """A walk on a 1/4 lattice (exact level hits on 0.25-step arithmetic grids) with flat ticks."""
    w = np.where(rng.random(N) < 0.3, 0, rng.integers(-jump, jump + 1, N))
    return np.clip(p0 + step * np.cumsum(w), 0.6 * p0, 1.4 * p0).astype(np.float32)


def trend(rng, N, p0, drift):
    return (p0 * np.exp(np.cumsum(drift + 0.002 * rng.standard_normal(N)))).astype(np.float32)


class GridCase:
    """One market and population for both grid entry points, launched with hand-packed individuals.

    close [S][N] float32, stored in rows of ld >= N floats; inds: ind() tuples; bounds [pop][S][2] (default: the pcts
    around the start bar's close); labels [R][N] uint8 (R = 1: one shared row) stored in rows of ld_labels; rules
    {label: (num_grids, lower_pct, upper_pct)} or None (no regime source)."""

    def __init__(self, close, start, inds, bounds=None, qty=None, bm=1, m0=M0, labels=None, rules=None, ld=None,
                 ld_labels=None):
        self.close = np.atleast_2d(np.asarray(close, dtype=np.float32))
        self.S, self.N = self.close.shape
        self.start, self.inds, self.bm, self.m0, self.rules = start, list(inds), bm, m0, rules
        self.qty = np.asarray(qty if qty is not None else [0.01 * (s + 1) for s in range(self.S)], dtype=np.float64)
        if bounds is None:                    # around the first finite close from the start bar on
            p0 = [float(r[np.isfinite(r)][0]) for r in self.close[:, start:].astype(np.float64)]
            bounds = [[(p * (1 - iv[5] / 100), p * (1 + iv[6] / 100)) for p in p0] for iv in self.inds]
        self.bounds = np.asarray(bounds, dtype=np.float64).reshape(len(self.inds), self.S, 2)
        self.labels = None if labels is None else np.atleast_2d(np.asarray(labels, dtype=np.uint8))
        self.ld = ld or self.N
        self.ld_labels = (0 if self.labels is None or len(self.labels) == 1 else self.N) if ld_labels is None \
            else ld_labels
        self.first_day = m0 // 1440
        self.D = (m0 + (self.N - 1) * bm) // 1440 - self.first_day + 1

    def subset(self, keep):
        return GridCase(self.close, self.start, [self.inds[i] for i in keep], self.bounds[keep], self.qty, self.bm,
                        self.m0, self.labels, self.rules, self.ld, self.ld_labels)

    def run(self, torch, service=False, days=False):
        """(stats [pop][S][20], service [pop][12] or None, day rows [pop][D] or None) as NumPy arrays."""
        from ai_crypto_trader_b200 import _lib
        S, N, pop = self.S, self.N, len(self.inds)
        px = torch.full((S, self.ld), math.nan, dtype=torch.float32, device="cuda")
        px[:, :N] = torch.from_numpy(self.close)
        rows = (_lib.GridIndividual * pop)(*[_lib.GridIndividual(n, k, r, a, f, 0, lo, up)
                                             for n, k, r, a, f, lo, up in self.inds])
        indiv = torch.from_numpy(np.frombuffer(bytes(rows), dtype=np.uint8).copy()).cuda()
        bnd = torch.from_numpy(self.bounds.copy()).cuda()
        qty = torch.from_numpy(self.qty.copy()).cuda()
        lab = table = None
        if self.labels is not None:
            R = len(self.labels)
            lab = torch.full((R, max(self.ld_labels, N)), 4, dtype=torch.uint8, device="cuda")
            lab[:, :N] = torch.from_numpy(self.labels)
        if self.rules is not None:
            table = (_lib.GridRegimeRule * 5)()
            for r, (n, lo, up) in self.rules.items():
                table[r] = _lib.GridRegimeRule(1, n, lo, up)
        stats = torch.full((pop, S, 20), -7.0, dtype=torch.float64, device="cuda")
        sv = torch.full((pop, 12), -7.0, dtype=torch.float64, device="cuda") if service else None
        day = torch.full((pop, self.D), -7.0, dtype=torch.float64, device="cuda") if days else None
        args = [px.data_ptr(), self.ld, S, N, self.start, self.bm, self.m0, indiv.data_ptr(), pop, qty.data_ptr(),
                bnd.data_ptr(), _lib.ptr(lab), self.ld_labels, table, stats.data_ptr()]
        if service:
            args.append(sv.data_ptr())
        _lib.call("b200bt_grid_service_sweep" if service else "b200bt_grid_sweep", *args, _lib.ptr(day),
                  self.D if days else 0, _lib.current_stream())
        torch.cuda.synchronize()
        return stats.cpu().numpy(), None if sv is None else sv.cpu().numpy(), None if day is None else day.cpu().numpy()

    def _common(self, i):
        n, kind, reb, adj, flags, lo, up = self.inds[i]
        T = self.N - self.start
        return dict(n=n, kind=kind, lower_pct=lo, upper_pct=up, rebalance_ticks=reb, adjust_ticks=adj,
                    adapt=bool(flags & 1), table={} if self.rules is None else dict(self.rules), bar_seconds=60 * self.bm,
                    days=[(self.m0 + (self.start + k) * self.bm) // 1440 for k in range(T)])

    def prices(self, s):
        return self.close[s, self.start:].astype(np.float64)

    def label_row(self, s):
        if self.labels is None:
            return None
        return self.labels[0 if self.ld_labels == 0 else s][self.start:]

    def ref_lane(self, i, s):
        kw = self._common(i)
        return grid_ref.simulate(self.prices(s), float(self.bounds[i, s, 0]), float(self.bounds[i, s, 1]),
                                 qty=float(self.qty[s]), labels=self.label_row(s), **kw)

    def ref_service(self, i):
        kw = self._common(i)
        n, kind = kw.pop("n"), kw.pop("kind")
        return grid_service_ref.simulate_service([self.prices(s) for s in range(self.S)],
                                                 [tuple(self.bounds[i, s]) for s in range(self.S)], n, kind,
                                                 list(self.qty), labels=self.label_row(0), **kw)


def same(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


def check_lane(got, want, kind, where):
    """One lane's stats row against the restatement; returns 1 for a geometric lane with near ties (count bound only)."""
    g = dict(zip(FIELDS, (float(x) for x in got)))
    if g["near_ties"] > 0:
        assert kind == 1, where
        assert abs(g["total_trades"] - want["total_trades"]) <= 2 * g["near_ties"] * 128, where
        return 1
    for f in EXACT:
        assert same(g[f], float(want[f])), (where, f, g[f], want[f])
    for f in PROFITS:
        w = float(want[f])
        assert same(g[f], w) or math.isclose(g[f], w, rel_tol=1e-9, abs_tol=1e-9 * max(1.0, abs(want["cash"]))), \
            (where, f, g[f], w)
    if kind == 0:
        assert g["near_ties"] == 0, where
        for f in ("total_profit", "profit_per_day"):
            assert math.isclose(g[f], want[f], rel_tol=1e-9, abs_tol=0.0), (where, f, g[f], want[f])
    return 0


def check_row(got, want_days, first_day, strict, where):
    want = np.zeros(len(got))
    for d, v in want_days.items():
        want[d - first_day] += v
    assert np.allclose(got, want, rtol=1e-9, atol=0.0 if strict else 1e-9), where


def check_grid(torch, case, service=True, days=True):
    """Both entry points (the service when asked and possible), with and without day rows: stats equal either way,
    every valid individual against the restatement, invalid ones all-NaN.  Returns (lanes, near-tie lanes) checked."""
    lanes = tied = 0
    modes = [False] + ([True] if service and case.ld_labels == 0 else [])
    for svc in modes:
        st, sv, _ = case.run(torch, svc)
        if days:
            st_d, sv_d, rows = case.run(torch, svc, days=True)
            assert np.array_equal(st, st_d, equal_nan=True), svc              # the day path changes no stat
            if svc:
                assert np.array_equal(sv, sv_d, equal_nan=True)
        for i, iv in enumerate(case.inds):
            where = ("service" if svc else "lanes", i, iv)
            if not valid(iv):
                assert np.all(np.isnan(st[i])), where
                if svc:
                    assert np.all(np.isnan(sv[i])), where
                if days:
                    assert np.all(rows[i] == 0.0), where
                continue
            if svc:
                want = case.ref_service(i)
                wl, wdays = want["lanes"], want["day_profit"]
            else:
                wl = [case.ref_lane(i, s) for s in range(case.S)]
                wdays = {}
                for w in wl:
                    for d, v in w["day_profit"].items():
                        wdays[d] = wdays.get(d, 0.0) + v
            t = sum(check_lane(st[i, s], wl[s], iv[1], where + (s,)) for s in range(case.S))
            lanes += case.S
            tied += t
            if t:
                continue
            if svc:
                g = dict(zip(grid_service_ref.SERVICE_FIELDS, sv[i]))
                for f in SERVICE_EXACT:
                    assert g[f] == want["service"][f], (where, f, g[f], want["service"][f])
                for f in ("total_profit", "profit_per_day"):
                    assert math.isclose(g[f], want["service"][f], rel_tol=1e-9, abs_tol=0.0), (where, f)
            if days:
                check_row(rows[i], wdays, case.first_day, iv[1] == 0, where)
    assert tied <= max(2, lanes // 2), (tied, lanes)
    return lanes, tied


# ---- grid: tile, pass and CTA seams ------------------------------------------------------------------------------


@pytest.mark.parametrize("T", [1, 2, 32, 33, 2048, 2049, 2050, 4097])
def test_grid_tile_and_pass_seams(torch_cuda, T):
    """Check periods on both sides of 32 and 2 048, on a tile's last tick (2 048) and on T - 1 and T; a start bar that
    is not a multiple of 32; 1 .. 127 levels, regime rules on a shared label row (one sets 127)."""
    rng = np.random.default_rng(T)
    start = 37
    N = start + T
    close = np.stack([lattice(rng, N), trend(rng, N, 2000.0, 0.0003)])
    labels = rng.integers(0, 7, N).astype(np.uint8)[None]
    periods = sorted({1, 2, 31, 32, 33, 2047, 2048, 2049, max(1, T - 1), T, NEVER})
    ns = (1, 2, 31, 32, 33, 127)
    inds = [ind(ns[j % 6], j % 2, p, periods[(j + 3) % len(periods)], adapt=j % 3 == 0, lo=2.0 + j % 3, up=3.0)
            for j, p in enumerate(periods)]
    case = GridCase(close, start, inds, labels=labels, rules={2: (127, 2.0, 2.0), 3: (33, 4.0, 1.5)})
    check_grid(torch_cuda, case)


@pytest.mark.parametrize("pop", [1, 15, 16, 17, 33])
def test_grid_population_seams(torch_cuda, pop):
    """Partly filled 16-warp CTAs; every lane against the restatement."""
    rng = np.random.default_rng(pop)
    N = 1500
    close = np.stack([lattice(rng, N), trend(rng, N, 50.0, -0.0002)])
    inds = [ind(int(rng.integers(1, 128)), int(rng.integers(0, 2)), int(rng.integers(1, 400)), int(rng.integers(1, 700)),
                lo=float(rng.uniform(0.5, 6)), up=float(rng.uniform(0.5, 6))) for _ in range(pop)]
    check_grid(torch_cuda, GridCase(close, 100, inds))


def test_grid_invalid_individuals_leave_their_neighbours_alone(torch_cuda):
    """num_grids 0 / 128, grid_type 2, periods of 0 (all refused by decode_individual) get NaN stats, NaN service records
    and zero day rows; the valid individuals around them are bit-equal to a run without them."""
    rng = np.random.default_rng(3)
    N = 2600
    close = np.stack([lattice(rng, N), trend(rng, N, 300.0, 0.0001)])
    bad = [ind(0), ind(128), ind(10, kind=2), ind(10, reb=0), ind(10, adj=0)]
    inds = []
    for j in range(28):
        inds.append(ind(int(rng.integers(1, 128)), j % 2, int(rng.integers(1, 300)), int(rng.integers(1, 900))))
        if j % 6 == 2:
            inds.append(bad[j // 6])
    case = GridCase(close, 64, inds)
    keep = [i for i, iv in enumerate(inds) if valid(iv)]
    assert len(keep) == len(inds) - len(bad)
    check_grid(torch_cuda, case)
    alone = case.subset(keep)
    for svc in (False, True):
        for days in (False, True):
            a, sa, ra = case.run(torch_cuda, svc, days)
            b, sb, rb = alone.run(torch_cuda, svc, days)
            assert np.array_equal(a[keep].view(np.int64), b.view(np.int64)), (svc, days)
            if svc:
                assert np.array_equal(sa[keep].view(np.int64), sb.view(np.int64))
            if days:
                assert np.array_equal(ra[keep].view(np.int64), rb.view(np.int64))


# ---- grid: level tables and the index estimate -------------------------------------------------------------------


def test_grid_level_tables(torch_cuda):
    """1, 2, 31, 32, 33 and 127 levels, arithmetic and geometric; a regime rule that sets 127; the win-rate rule stepping
    down from 127 (a falling market) and up from 3 (a rising one)."""
    rng = np.random.default_rng(7)
    N = 3101
    k = np.arange(N)
    close = np.stack([lattice(rng, N), 100.0 * 1.002 ** k, 100.0 * 0.998 ** k]).astype(np.float32)
    inds = [ind(n, kind, reb=17, adj=NEVER) for n in (1, 2, 31, 32, 33, 127) for kind in (0, 1)]
    # regenerated every tick around a price that moves 0.2 % a tick: every crossing on the rise is profitable, none on
    # the fall
    inds += [ind(n, kind, reb=1, adj=40, lo=0.05, up=0.05) for n in (127, 3) for kind in (0, 1)]
    inds += [ind(5, kind, reb=23, adj=50, adapt=1) for kind in (0, 1)]
    case = GridCase(close, 101, inds, labels=np.full((1, N), 2, dtype=np.uint8), rules={2: (127, 1.5, 2.5)})
    check_grid(torch_cuda, case)
    st, _, _ = case.run(torch_cuda)
    n = st[12:16, :, FIELDS.index("num_grids")]
    assert np.all(n[:, 1] == 20) and np.all(n[:, 2] == 5)                # up from 3 and 127, down from both


def test_grid_index_estimate_extremes(torch_cuda):
    """Ticks that jump from below lower to above upper and back (every level crossed), prices far outside the grid,
    prices on an arithmetic lattice's levels, and grids of pct 1e-6 and 1e-14 whose fp32 scale is huge or infinite."""
    rng = np.random.default_rng(9)
    N = 2600
    k = np.arange(N)
    jump = np.where(k % 2 == 0, 50.0, 200.0)
    jump[::7] = 100.0
    far = np.where(k % 3 == 0, 1e-3, np.where(k % 3 == 1, 1e6, 100.0))
    on_levels = 100.0 + 0.25 * rng.integers(-40, 41, N)
    narrow = 100.0 + np.where(rng.random(N) < 0.5, 0.0, rng.integers(-3, 4, N) * 2.0 ** -16)
    close = np.stack([jump, far, on_levels, narrow]).astype(np.float32)
    inds = [ind(n, kind, reb) for n in (127, 33, 8) for kind in (0, 1) for reb in (1, 7, NEVER)]
    inds += [ind(n, kind, reb, lo=pct, up=pct) for n in (127, 9) for kind in (0, 1) for reb in (1, 5)
             for pct in (1e-6, 1e-14)]
    bounds = []
    for iv in inds:
        b = [(95.0, 105.0), (95.0, 105.0), (90.0, 110.0), (100.0 * (1 - iv[5] / 100), 100.0 * (1 + iv[6] / 100))]
        bounds.append(b)
    check_grid(torch_cuda, GridCase(close, 0, inds, bounds=bounds, qty=[1.0, 0.5, 0.25, 2.0]))


def test_grid_repeated_levels(torch_cuda):
    """Every copy of a repeated level earns the step under its first copy (levels.index): an arithmetic step under an
    ulp, grids regenerated at a pct of 1e-14 (all levels equal) and a geometric ratio of 1.0, in lanes and the service."""
    tiny = GridCase([[99, 101, 99, 101]], 0, [ind(8, 0)], bounds=[[(100.0, 100 * (1 + 6e-16))]], qty=[1.0])
    check_grid(torch_cuda, tiny)
    st, _, _ = tiny.run(torch_cuda)
    assert st[0, 0, FIELDS.index("profitable_trades")] == 16 and st[0, 0, FIELDS.index("up_crossings")] == 18
    rng = np.random.default_rng(4)
    N = 2300
    close = np.stack([100.0 + np.where(np.arange(N) % 2 == 0, -1.0, 1.0) * rng.integers(1, 3, N),
                      lattice(rng, N, 100.0, 0.5)]).astype(np.float32)
    inds = [ind(n, 0, reb, adj, lo=1e-14, up=1e-14) for n in (8, 127) for reb in (3, 64) for adj in (NEVER, 100)]
    inds += [ind(n, 0, NEVER) for n in (8, 40)]                           # an initial step under an ulp
    inds += [ind(n, 1, NEVER, adj) for n in (8, 127) for adj in (NEVER, 100)]    # ratio 1.0, off the price lattices
    bounds = [[(100.25, 100.25)] * 2 if iv[1] == 1 else [(100.0, 100.0)] * 2 if iv[5] == 1e-14
              else [(100.0, 100.0 * (1 + 6e-16))] * 2 for iv in inds]
    _, tied = check_grid(torch_cuda, GridCase(close, 0, inds, bounds=bounds, qty=[1.0, 3.0]))
    assert tied == 0


# ---- grid: missing closes ----------------------------------------------------------------------------------------


def test_grid_missing_closes(torch_cuda):
    """NaN closes are no move, so the tick with one and the tick after it do nothing: at tick 0, mid-series, on a
    rebalance tick (nothing regenerates), on an adjust tick, in runs across a tile seam and on the last tick
    (mark_to_market NaN), with day rows."""
    rng = np.random.default_rng(12)
    start, N = 5, 5 + 4400
    close = np.stack([lattice(rng, N), lattice(rng, N, 100.0, 0.5, 3), trend(rng, N, 80.0, 0.0)])
    for t in (0, 777, 100, 140, 2040, 2041, 2050, 2051, 2052, 2060, 3000, 3001):
        close[:, start + t] = np.nan
    close[0, start + 1500: start + 1520] = np.nan
    close[1, -1] = np.nan
    close[2, start + 2047: start + 2050] = np.nan                                     # across the first tile's end
    inds = [ind(n, kind, reb, adj, adapt) for n in (10, 40, 127) for kind in (0, 1)
            for reb, adj, adapt in ((50, 70, 1), (1, 3, 0), (NEVER, 1, 1))]
    labels = rng.integers(0, 5, N).astype(np.uint8)[None]
    case = GridCase(close, start, inds, labels=labels, rules={2: (31, 2.0, 2.0), 3: (12, 6.0, 6.0)})
    check_grid(torch_cuda, case)
    st, _, _ = case.run(torch_cuda)
    mtm = st[:, :, FIELDS.index("mark_to_market")]
    assert np.all(np.isnan(mtm[:, 1])) and np.all(np.isfinite(mtm[:, [0, 2]]))


# ---- grid: layouts, clocks and the service ------------------------------------------------------------------------


def test_grid_strided_rows_and_label_rows(torch_cuda):
    """Close rows of ld > N; per-symbol label rows of ld_labels > N (labels >= 5 among them) against the restatement,
    and the same row in every symbol bit-equal to one shared row."""
    rng = np.random.default_rng(21)
    S, N = 3, 2200
    close = np.stack([lattice(rng, N, 100.0 + 10 * s) for s in range(S)])
    labels = rng.choice(np.array([0, 1, 2, 3, 4, 5, 7, 255], dtype=np.uint8), (S, N))
    inds = [ind(n, kind, 29, 61, adapt=1) for n in (12, 70) for kind in (0, 1)]
    rules = {2: (40, 1.0, 1.5), 3: (127, 2.0, 2.0), 4: (5, 4.0, 4.0)}
    check_grid(torch_cuda, GridCase(close, 40, inds, labels=labels, rules=rules, ld=N + 45, ld_labels=N + 3))
    shared = GridCase(close, 40, inds, labels=labels[:1], rules=rules, ld=N + 45)
    check_grid(torch_cuda, shared)
    per_symbol = GridCase(close, 40, inds, labels=np.repeat(labels[:1], S, 0), rules=rules, ld=N + 45, ld_labels=N + 3)
    for days in (False, True):
        a, _, ra = shared.run(torch_cuda, days=days)
        b, _, rb = per_symbol.run(torch_cuda, days=days)
        assert np.array_equal(a.view(np.int64), b.view(np.int64))
        if days:
            assert np.array_equal(ra.view(np.int64), rb.view(np.int64))


@pytest.mark.parametrize("bm,m0", [(1440, M0), (7, M0 + 613), (1, M0 + 1000)])
def test_grid_day_rows_on_other_clocks(torch_cuda, bm, m0):
    """Daily bars (a 32-tick pass spans 32 days), a bar that does not divide a day, minute0 in the middle of a day."""
    rng = np.random.default_rng(bm)
    N = {1440: 400, 7: 2100, 1: 3000}[bm]
    close = np.stack([lattice(rng, N), trend(rng, N, 40.0, 0.0005)])
    inds = [ind(n, kind, reb, adj) for n in (6, 64) for kind in (0, 1) for reb, adj in ((NEVER, NEVER), (45, 90))]
    check_grid(torch_cuda, GridCase(close, 3, inds, bm=bm, m0=m0))


@pytest.mark.parametrize("S", [1, 16, 17, 32, 33])
def test_grid_service_symbol_counts(torch_cuda, S):
    """The service with adjust_ticks = 1 and a regime rule, one to three warps' worth of symbols, and day rows (one warp
    runs every symbol)."""
    rng = np.random.default_rng(40 + S)
    N = 700
    close = np.stack([lattice(rng, N, 50.0 + 5 * s) if s % 2 else trend(rng, N, 50.0 + 5 * s, 0.0002 * (s % 3 - 1))
                      for s in range(S)])
    labels = np.repeat(rng.integers(0, 5, N // 20 + 1), 20)[:N].astype(np.uint8)[None]
    inds = [ind(10, 0, 5, 1, adapt=1), ind(30, 1, 2, 1, adapt=1), ind(127, 0, 40, 1, adapt=0)]
    case = GridCase(close, 11, inds, labels=labels, rules={2: (127, 1.0, 1.0), 3: (9, 3.0, 3.0)})
    check_grid(torch_cuda, case)


def test_grid_sweep_refuses_65536_symbols(torch_cuda):
    """The lane sweep's launch has S CTAs along y: S = 65 536 is refused before the device; the service (one CTA per
    individual) takes it."""
    from ai_crypto_trader_b200 import _lib
    S = 65536
    close = np.full((S, 2), 100.0, dtype=np.float32)
    close[:, 1] = 101.0
    case = GridCase(close, 0, [ind(4)], bounds=np.tile([99.0, 103.0], (1, S, 1)), qty=np.ones(S))
    with pytest.raises(_lib.B200btError, match="65535"):
        case.run(torch_cuda)
    st, sv, _ = case.run(torch_cuda, service=True)
    assert np.all(st[0, :, FIELDS.index("up_crossings")] == 2) and sv[0, 1] == 2 * S


def test_grid_long_series_against_the_fast_restatement(torch_cuda):
    """300 000 ticks over many tiles: NaN closes and repeated levels against grid_ref.simulate_fast."""
    rng = np.random.default_rng(31)
    N = 300_000
    close = np.stack([lattice(rng, N, 1000.0, 0.25, 12), trend(rng, N, 100.0, 0.0)])
    close[:, rng.integers(0, N, 400)] = np.nan
    close[0, 2047 * 40: 2047 * 40 + 70] = np.nan
    inds = [ind(n, kind, reb, adj, lo=pct, up=pct) for n, kind, reb, adj, pct in
            ((20, 0, 1441, 2881, 2.0), (127, 0, 307, 1000, 1e-14), (45, 0, 2048, 999, 0.7), (16, 1, 600, 1441, 1.5))]
    case = GridCase(close, 1000, inds, qty=[0.5, 2.0])
    st, _, _ = case.run(torch_cuda)
    for i, iv in enumerate(inds):
        for s in range(2):
            kw = case._common(i)
            kw.pop("days")
            want = grid_ref.simulate_fast(case.prices(s), float(case.bounds[i, s, 0]), float(case.bounds[i, s, 1]),
                                          qty=float(case.qty[s]), labels=None, **kw)
            check_lane(st[i, s], want, iv[1], (i, s))


# ---- DCA: the dip search's pyramid ----------------------------------------------------------------------------------


def flat_dips(N, dips, depth_pct, m0):
    """A flat market (close = high = 100) whose dips drop one bar's close; the dip series the rule gives it: NaN on the
    series' first day (one kline), else ((100 - close) / 100) * 100."""
    close = np.full(N, 100.0, dtype=np.float32)
    for j, b in enumerate(dips):
        close[b] = np.float32(100.0 * (1 - depth_pct[j % len(depth_pct)] / 100))
    day = (m0 + np.arange(N, dtype=np.int64)) // 1440
    c = close.astype(np.float64)
    dip = ((100.0 - c) / 100.0) * 100
    dip[day == day[0]] = np.nan
    return close, dip


def dca_genes(thr, cooldown_days=0, **kw):
    return dict({"interval_hours": 500.0, "base_order_size_usdc": 100.0, "price_dip_detection": 1,
                 "dip_threshold_pct": thr, "additional_dip_allocation": 0.5, "max_dip_frequency_days": cooldown_days,
                 "adaptive_scheduling": 0, "periodic_rebalancing": 0}, **kw)


def run_dca(torch, market, pop, start_bar, days=True, **kw):
    from ai_crypto_trader_b200.dca import DCASweep
    sweep = DCASweep(market, start_bar=start_bar, **kw)
    sweep.dca_stats(pop)
    rows = sweep.day_pnl(pop)[0].cpu().numpy() if days else None
    return sweep, check_dca(sweep, pop, rows=rows)


@pytest.mark.parametrize("N", [3 * 32768 + 5, 32 * 32768 + 40_003])
def test_dca_dip_search_block_seams(torch_cuda, N):
    """Isolated dips on the 32 / 1 024 / 32 768-bar block seams and the last bar, N just above a multiple of 32 768
    and above 2^20 (the top level steps through 32-entry groups), start bars inside blocks, thresholds below, equal to
    and above the dips, and a one-day cooldown that ends exactly on a hit or one tick after one."""
    from ai_crypto_trader_b200 import dca
    m0 = M0 + 1430                                                        # the first day holds 10 bars
    dips = [31, 32, 1023, 1024, 5000, 5000 + 1440, 10000, 10000 + 1439, 32767, 32768, 32769, 65535, 65536, N - 5, N - 1]
    if N > 2 ** 20:
        dips += [2 ** 20 - 1, 2 ** 20, 2 ** 20 + 1, 2 ** 20 + 32768]
    dips = sorted(set(dips))
    close, want_dip = flat_dips(N, dips, (1.0, 2.0, 3.0), m0)
    m = dca_market(torch_cuda, close, np.full(N, 100.0, dtype=np.float32), 1, m0)
    two = float(want_dip[dips[1]])                                        # a 2 % dip, exactly
    assert two == want_dip[dips[4]] and 1.9 < two < 2.1
    pop = [dca_genes(0.5), dca_genes(two), dca_genes(np.nextafter(two, 3.0)), dca_genes(50.0), dca_genes(0.5, 1)]
    for start in (0, 1000, 32768 + 5):
        sweep, st = run_dca(torch_cuda, m, pop, start, days=start == 1000)
        assert np.array_equal(sweep.dip.cpu().numpy()[0], want_dip, equal_nan=True)
        after = [b for b in dips if b >= start]
        n_dip = st["n_dip"][:, 0]
        assert n_dip[0] == len(after) and n_dip[3] == 0
        assert n_dip[1] == sum(want_dip[b] >= two for b in after) > n_dip[2]
        if start == 0:                                                    # the cooldown: 6440 bought, 11439 not
            dec = dca.decode_individual(pop[4], sweep.block, m.symbols, 1)
            ref = dca_ref.simulate(close[None].astype(np.float64), want_dip[None], m0, 1, 0, dec)
            bought = [k for k, kind, *_ in ref["purchases"][0] if kind == "dip"]
            assert 5000 + 1440 in bought and 10000 + 1439 not in bought and 10000 in bought


def test_dca_nan_dip_runs(torch_cuda):
    """Highs of 0 for nine days: the drop is NaN (no dip) over whole 32- and 1 024-bar blocks; dips on both sides."""
    N = 16 * 1440
    m0 = M0 + 300
    close = np.full(N, 100.0, dtype=np.float32)
    high = np.full(N, 100.0, dtype=np.float32)
    high[3 * 1440: 12 * 1440] = 0.0
    for b in (2 * 1440 + 5, 9 * 1440 + 1, 10 * 1440, 12 * 1440 - 1, 12 * 1440, 12 * 1440 + 31, N - 1):
        close[b] = 97.0
    m = dca_market(torch_cuda, close, high, 1, m0)
    want = dca_ref.dip_series(high.astype(np.float64), close.astype(np.float64), m0, 1)
    assert np.isnan(want[14 * 1024: 16 * 1024]).all()                     # two whole 1 024-bar blocks, and more
    pop = [dca_genes(0.5), dca_genes(3.0), dca_genes(2.0, 1)]
    for start in (0, 9 * 1440 + 7):
        sweep, st = run_dca(torch_cuda, m, pop, start)
        assert np.array_equal(sweep.dip.cpu().numpy()[0], want, equal_nan=True)
        assert st["n_dip"][0, 0] == np.sum(want[start:] >= 0.5) > 0


# ---- DCA: clocks and coupling ------------------------------------------------------------------------------------------


def test_dca_clock_edges(torch_cuda):
    """A 7-minute bar (no divisor of a day), minute0 in the middle of a day, weighted scheduling with purchases on both
    sides of the Friday / Saturday and Sunday / Monday boundaries, and T = 1."""
    from ai_crypto_trader_b200 import dca
    rng = np.random.default_rng(5)
    S, N, bm, m0 = 2, 4 * 7 * 1440 // 7, 7, M0 + 613
    close = (100 * np.exp(np.cumsum(0.004 * rng.standard_normal((S, N)), axis=1))).astype(np.float32)
    high = np.maximum(close * (1 + np.abs(rng.normal(0, 0.004, (S, N)))), close).astype(np.float32)
    m = dca_market(torch_cuda, close, high, bm, m0)
    cfg = {"scheduling_strategies": {"weighted_scheduling": {"enabled": True}}}
    pop = [dca_genes(1.0, 1, interval_hours=h, adaptive_scheduling=1, day_of_week_weight=w, periodic_rebalancing=1,
                     rebalance_interval_days=2) for h, w in ((5.0, 1.0), (7.5, 0.5), (23.0, 1.0))]
    sweep, _ = run_dca(torch_cuda, m, pop, 200, config=cfg)
    dec = dca.decode_individual(pop[0], sweep.block, m.symbols, bm)
    ref = dca_ref.simulate(m.close.cpu().numpy().astype(np.float64), sweep.dip.cpu().numpy(), m0, bm, 200, dec)
    weekdays = {((m0 + (200 + k) * bm) // 1440 + 3) % 7 for k, kind, *_ in ref["purchases"][0] if kind == "scheduled"}
    assert {4, 5, 6, 0} <= weekdays                                       # Friday, Saturday, Sunday, Monday
    run_dca(torch_cuda, m, pop, N - 1, config=cfg)                        # T = 1


def test_dca_rebalance_on_every_tick_with_32_symbols(torch_cuda):
    """S = 32 coupled at every tick (rebalance_interval_days = 0), with day rows."""
    rng = np.random.default_rng(32)
    S, N = 32, 3 * 288
    close = (np.round(100 * 10.0 ** (np.arange(S) % 3)[:, None] *
                      np.exp(np.cumsum(0.003 * rng.standard_normal((S, N)), axis=1)) * 16) / 16).astype(np.float32)
    high = np.maximum(close * 1.002, close).astype(np.float32)
    m = dca_market(torch_cuda, close, high, 5, M0 + 100)
    pop = [dca_genes(1.0, 0, interval_hours=h, periodic_rebalancing=1, rebalance_interval_days=0, max_deviation_pct=d)
           for h, d in ((2.0, 5.0), (9.0, 1.0), (30.0, 20.0))]
    _, st = run_dca(torch_cuda, m, pop, 20, usdc_balance=700.0)
    assert np.all(st["n_rebalance_checks"] == N - 20) and st["n_rebalance"].sum() > 0
