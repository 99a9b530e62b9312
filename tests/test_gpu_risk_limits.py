"""Risk kernels at their limits, called through the C ABI, against float64 references (oracle/portfolio_ref.py,
oracle/mc_ref.py, tests/mc_joint_ref.py and NumPy).

Correlation at every tile and pair-block seam up to S = 512, rows that are not a dense [S][N] tensor, the missing-data
shapes of real return banks (newly listed and delisted assets, stale feeds, ±inf returns after a zero close);
pct_change, tail sums, order statistics and moments at their grid-stride seams and on ties, infinities and subnormals;
the path kernels at their counter, size and bootstrap-table limits.
"""
import math

import numpy as np
import pandas as pd
import pytest

import mc_joint_ref
from gpu_fixtures import torch_cuda
from oracle import mc_ref, portfolio_ref

pytestmark = pytest.mark.gpu

# kernel constants and host formulas (csrc/portfolio.cu, csrc/montecarlo.cu)
CORR_THREADS = 256
PCT_GRID, TAIL_GRID = 1184, 592          # grid caps of pct_change_kernel and tail_partial_kernel (256 threads per CTA)
DEFAULT_SMEM = 48 * 1024
MC_MAX_TABLE = 12288                     # bootstrap table entries (48 KB of fp32)
CORR_ATOL = 1e-9


def corr_tile(S):
    T = min(98304 // (4 * S) - 1, 256)
    return T & ~31


def corr_pair_blocks(S):
    return (S * (S + 1) // 2 + CORR_THREADS - 1) // CORR_THREADS


def corr_splits(S, N):
    T = corr_tile(S)
    splits = min((296 + corr_pair_blocks(S) - 1) // corr_pair_blocks(S), (N + T - 1) // T)
    return max(splits, 1)


def corr_smem(S):
    return S * (corr_tile(S) + 1) * 4


def tail_blocks(n):
    return min(TAIL_GRID, (n + 255) // 256)


@pytest.fixture(scope="module")
def engine(torch_cuda):
    from ai_crypto_trader_b200.monte_carlo import PathEngine
    return PathEngine()


# ---------------------------------------------------------------------------------------------------------------------
# direct calls of the entry points
# ---------------------------------------------------------------------------------------------------------------------
def _rows_on_device(torch, x, ld=None, off=0, fill=7.0):
    """x [S][N] float32 -> (device buffer, pointer to row 0): rows ld apart, starting `off` floats into the buffer; the
    padding holds a finite value, so a kernel that read it would change its result."""
    S, N = x.shape
    ld = N if ld is None else ld
    host = np.full(off + S * ld, fill, dtype=np.float32)
    host[off:].reshape(S, ld)[:, :N] = x
    buf = torch.from_numpy(host).cuda()
    return buf, buf.data_ptr() + 4 * off, ld


def _correlation(torch, x, ld=None, off=0):
    from ai_crypto_trader_b200 import _lib
    S, N = x.shape
    buf, ptr, ld = _rows_on_device(torch, x, ld, off)
    need = int(_lib.load().b200bt_correlation_workspace_bytes(S, N))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.full((S, S), 3.0, dtype=torch.float64, device="cuda")
    _lib.call("b200bt_correlation", ptr, ld, S, N, out.data_ptr(), ws.data_ptr(), need, _lib.current_stream())
    res = out.cpu().numpy()
    del buf
    return res


def _check_corr(got, x, what=""):
    want = portfolio_ref.correlation(x)
    bad = np.argwhere(np.isnan(got) != np.isnan(want))
    assert bad.size == 0, (what, "NaN pattern differs at pairs", bad[:8].tolist(),
                           [(got[i, j], want[i, j]) for i, j in bad[:8]])
    m = ~np.isnan(want)
    np.testing.assert_allclose(got[m], want[m], rtol=0, atol=CORR_ATOL, err_msg=str(what))
    return want


def _returns(S, N, seed, holes=0.01, mean=5e-4):
    """float32 [S][N] returns: a common factor with per-row loadings plus noise, row means of a few 1e-3, NaN holes."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal(N)
    load = np.linspace(-1, 1, S)[:, None]
    x = mean * (1 + np.arange(S) % 7)[:, None] + 0.01 * (rng.standard_normal((S, N)) + load * base)
    x = x.astype(np.float32)
    x[rng.random((S, N)) < holes] = np.nan
    return x


# ---------------------------------------------------------------------------------------------------------------------
# correlation
# ---------------------------------------------------------------------------------------------------------------------
def test_corr_seams_are_where_the_cases_say():
    assert corr_pair_blocks(22) == 1 and corr_pair_blocks(23) == 2                 # 253 vs 276 pairs
    assert corr_smem(47) <= DEFAULT_SMEM < corr_smem(48)                          # staged tile past the default 48 KB
    assert corr_tile(95) == 256 and corr_tile(96) == 224
    assert corr_tile(253) == 96 and corr_tile(254) == 64
    assert corr_tile(378) == 64 and corr_tile(379) == 32
    assert corr_tile(512) == 32 and corr_smem(512) == 66 * 1024


@pytest.mark.parametrize("S", [1, 2, 22, 23, 47, 48, 95, 96, 253, 254, 378, 379, 512])
def test_correlation_at_s_seams(torch_cuda, S):
    T = corr_tile(S)
    N = 3 * T + 7
    x = _returns(S, N, seed=S)
    got = _correlation(torch_cuda, x)
    _check_corr(got, x, ("S", S))
    assert np.array_equal(got, _correlation(torch_cuda, x), equal_nan=True)     # deterministic: no atomics


@pytest.mark.parametrize("S", [5, 300])
def test_correlation_at_n_seams(torch_cuda, S):
    T = corr_tile(S)
    splits = corr_splits(S, 1 << 40)
    n_loop = 3 * splits * T + 5               # every time split walks three or more tiles
    assert (n_loop + T - 1) // T >= 3 * corr_splits(S, n_loop)
    for N in (1, 2, T - 1, T, T + 1, n_loop):
        x = _returns(S, N, seed=S + N)
        _check_corr(_correlation(torch_cuda, x), x, ("S", S, "N", N))


def test_correlation_rows_not_dense(torch_cuda):
    S, N = 30, 776
    x = _returns(S, N, seed=3)
    dense = _correlation(torch_cuda, x)
    _check_corr(dense, x)
    for ld, off in ((N + 64, 0), (N + 5, 0), (N, 1), (N + 5, 3)):   # padded, odd stride, off 16 B, both
        got = _correlation(torch_cuda, x, ld=ld, off=off)
        assert np.array_equal(got, dense, equal_nan=True), (ld, off)


def test_correlation_missing_data_shapes(torch_cuda):
    S, N = 13, 2000
    rng = np.random.default_rng(13)
    x = _returns(S, N, seed=13, holes=0.0)
    nan = np.float32(np.nan)
    x[2] = nan; x[2, 5] = x[0, 5]                                     # one observation
    x[3] = nan; x[3, [5, 900]] = [0.01, -0.02]                        # two observations
    x[4, :1400] = nan                                                 # newly listed
    x[5, 700:] = nan                                                  # delisted: disjoint from row 4
    x[6] = nan                                                        # no data
    x[7] = np.float32(0.1)                                            # constant rows, not powers of two
    x[8] = np.float32(1e-3)
    x[9] = np.float32(0.0)
    x[10, 1400:] = 0.0                                                # stale feed while row 4 trades
    x[11, :1400] = rng.normal(2e-2, 0.01, 1400)                       # one tick inside a stale window
    x[11, 1400:] = 0.0
    x[11, 1700] = 0.015
    x[12, 100], x[12, 1500], x[12, 1501] = np.inf, -np.inf, np.inf    # infinite returns
    got = _correlation(torch_cuda, x)
    want = _check_corr(got, x)
    assert np.isnan(want[2]).all() and np.isnan(want[6]).all() and np.isnan(want[4, 5])
    assert np.isnan(want[10, 4]) and np.isfinite(want[11, 4]) and np.isfinite(want[12, [0, 1, 3, 4, 5, 12]]).all()
    for r in (7, 8, 9):
        assert np.isnan(got[r]).all(), r


def test_correlation_stale_assets_against_newly_listed(torch_cuda):
    """Rows 0..23 go stale at bar 1000 (zero returns, or a pegged value that is not a power of two) after histories of
    different means; rows 24.. list at bars >= 1000.  Over every stale-vs-new pair's joint observations the stale row is
    constant: NaN for all 576 pairs.  Any rounding residue left in a variance would carry the sign its row's history
    gives it, so many stale rows, not many partners of one, keep the outcome from resting on that sign."""
    S, N, K = 48, 3000, 24
    rng = np.random.default_rng(48)
    x = _returns(S, N, seed=48, holes=0.0)
    for i in range(K):
        x[i, :1000] = rng.normal(rng.uniform(-5e-3, 5e-3), 0.02, 1000)
        x[i, 1000:] = 0.0 if i % 2 == 0 else np.float32(rng.uniform(-1e-3, 1e-3))
    for k in range(K, S):
        x[k, :1000 + int(rng.integers(0, 1900))] = np.nan
    got = _correlation(torch_cuda, x)
    want = _check_corr(got, x)
    assert np.isnan(want[:K, K:]).all() and np.isfinite(want[:K, :K]).all()
    assert np.isnan(got[:K, K:]).all() and np.isnan(got[K:, :K]).all()


def test_correlation_one_tick_in_stale_window(torch_cuda):
    """An asset that rallied (mean 2e-2 over 2000 bars) then went stale with one tick: its correlation with the assets
    listed since is set by that tick alone, and must not drown in its row mean."""
    S, N = 21, 3000
    rng = np.random.default_rng(21)
    x = _returns(S, N, seed=21, holes=0.0)
    x[0, :2000] = rng.normal(2e-2, 0.01, 2000)
    x[0, 2000:] = 0.0
    x[0, 2600] = 0.01
    for k in range(1, S):
        x[k, :2000 + int(rng.integers(0, 500))] = np.nan
    want = _check_corr(_correlation(torch_cuda, x), x)
    assert np.isfinite(want[0]).all()


def test_correlation_skips_infinite_returns(torch_cuda):
    S, N = 6, 1500
    x = _returns(S, N, seed=6)
    x[0, 10], x[0, 700] = np.inf, -np.inf
    x[1, 1499] = np.inf
    x[2, 300:] = np.inf                                           # finite only where it trades before bar 300
    x[3] = -np.inf                                                # never finite
    got = _correlation(torch_cuda, x)
    want = _check_corr(got, x)
    assert np.isfinite(want[:3, :3]).all() and np.isnan(want[3]).all()


def test_asset_correlation_from_closes_with_a_zero(torch_cuda):
    from ai_crypto_trader_b200.portfolio_risk import PortfolioRiskService, ReturnBank
    rng = np.random.default_rng(8)
    S, N = 4, 600
    close = (100 * np.exp(np.cumsum(rng.normal(0, 0.01, (S, N)), axis=1))).astype(np.float32)
    close[1, 200] = 0.0                                  # -1 then +inf
    close[2, 300:302] = 0.0                              # -1, 0/0, +inf
    syms = [f"A{i}USDC" for i in range(S)]
    bank = ReturnBank.from_close(syms, close)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = portfolio_ref.pct_change(close).astype(np.float32)
    assert np.isposinf(r[1, 201]) and np.isnan(r[2, 301]) and np.isposinf(r[2, 302])
    assert np.array_equal(bank.returns.cpu().numpy(), r, equal_nan=True)
    corr = PortfolioRiskService(bank).calculate_asset_correlation(syms)
    got = np.array([[corr[a][b] for b in syms] for a in syms])
    want = portfolio_ref.correlation(r)
    assert np.isfinite(want).all()
    np.testing.assert_allclose(got, want, rtol=0, atol=CORR_ATOL)


def test_joint_monte_carlo_falls_back_on_a_stale_asset(torch_cuda):
    """AAA's feed is stale (zero returns) over the whole life of the newly listed BBB: their correlation is NaN, so the
    joint simulation uses the identity, as the reference's policy does."""
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService
    rng = np.random.default_rng(17)
    a = pd.Series(np.concatenate([rng.normal(3e-3, 0.02, 150), np.zeros(90)]))
    b = pd.Series(rng.normal(1e-3, 0.03, 90), index=np.arange(150, 240))
    want = pd.DataFrame({"AAA": a, "BBB": b}).corr().to_numpy()
    assert np.isnan(want[0, 1])
    svc = MonteCarloService(seed=5)
    svc.mc_params.update(num_simulations=4096, time_horizon_days=10)
    svc.historical_data = {"AAAUSDC": pd.DataFrame({"returns": a}), "BBBUSDC": pd.DataFrame({"returns": b})}
    holdings = {"total_value": 3000.0, "assets": {"AAA": {"value_usdc": 2000.0, "current_price": 10.0},
                                                  "BBB": {"value_usdc": 1000.0, "current_price": 2.0}}}
    res = svc.run_joint_portfolio_monte_carlo(holdings, scenarios=["base"])
    assert res and res["correlation_fallback"] is True
    assert res["correlation"]["AAA"]["BBB"] == 0.0 and res["correlation"]["AAA"]["AAA"] == 1.0


# ---------------------------------------------------------------------------------------------------------------------
# pct_change
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,N,ld,ld_out", [(3, 1000, 1000, 1000), (3, 999, 1031, 1013), (2, PCT_GRID * 256 - 1, None, None),
                                           (2, PCT_GRID * 256 + 1, PCT_GRID * 256 + 9, PCT_GRID * 256 + 4)])
def test_pct_change_bitwise(torch_cuda, S, N, ld, ld_out):
    from ai_crypto_trader_b200 import _lib
    torch = torch_cuda
    rng = np.random.default_rng(N)
    close = (100 * np.exp(np.cumsum(rng.normal(0, 0.01, (S, N)), axis=1))).astype(np.float32)
    close[0, N // 2] = 0.0                                   # -1, +inf
    close[-1, N - 3:N - 1] = 0.0                             # -1, 0/0, +inf
    close[-1, 0] = 0.0                                       # a zero first close
    buf, ptr, ld = _rows_on_device(torch, close, ld)
    ld_out = N if ld_out is None else ld_out
    out = torch.full((S * ld_out,), 12345.0, dtype=torch.float32, device="cuda")
    _lib.call("b200bt_pct_change", ptr, ld, S, N, out.data_ptr(), ld_out, _lib.current_stream())
    got = out.cpu().numpy().reshape(S, ld_out)
    assert (got[:, N:] == 12345.0).all()                    # the padding of the output rows is not written
    got = got[:, :N]
    with np.errstate(divide="ignore", invalid="ignore"):
        want = portfolio_ref.pct_change(close).astype(np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    m = ~np.isnan(want)
    assert np.array_equal(got[m].view(np.uint32), want[m].view(np.uint32))
    assert np.isposinf(got[0, N // 2 + 1]) and np.isnan(got[-1, N - 2]) and np.isnan(got[:, 0]).all()


# ---------------------------------------------------------------------------------------------------------------------
# tail sums
# ---------------------------------------------------------------------------------------------------------------------
def _tail_stats(torch, x, threshold):
    from ai_crypto_trader_b200 import _lib
    xd = torch.from_numpy(x).cuda()
    n = int(x.size)
    need = int(_lib.load().b200bt_tail_stats_workspace_bytes(n))
    assert need == tail_blocks(n) * 32
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(4, dtype=torch.float64, device="cuda")
    _lib.call("b200bt_tail_stats", xd.data_ptr(), n, float(threshold), out.data_ptr(), ws.data_ptr(), need,
              _lib.current_stream())
    return out.cpu().numpy()


def _tail_ref(x, threshold):
    v = x.astype(np.float64)
    ok = ~np.isnan(v)
    tail = ok & (v <= threshold)
    with np.errstate(invalid="ignore"):
        return np.array([v[tail].sum(), tail.sum(), ok.sum(), v[ok].sum()]), np.array([np.abs(v[tail]).sum(), 0, 0,
                                                                                        np.abs(v[ok]).sum()])


def _check_sums(got, want, scale, rel=1e-12):
    for k, (g, w, s) in enumerate(zip(got, want, scale)):
        if not np.isfinite(w):
            assert g == w or (np.isnan(g) and np.isnan(w)), (k, g, w)
        else:
            assert abs(g - w) <= rel * s, (k, g, w, s)


@pytest.mark.parametrize("n", [1, 255, 256, 257, TAIL_GRID * 256 - 1, TAIL_GRID * 256 + 1, 3_000_001])
def test_tail_stats(torch_cuda, n):
    rng = np.random.default_rng(n)
    x = (np.round(rng.normal(0, 0.02, n) * 512) / 512).astype(np.float32)    # quantised: heavy ties
    if n > 10:
        x[::97] = np.nan
    finite = x[~np.isnan(x)]
    tied = np.float32(np.median(finite)) if finite.size else np.float32(0)
    for thr in (float(finite.min()) - 1.0, float(tied), float(finite.max()) + 1.0, float(finite.max())):
        got = _tail_stats(torch_cuda, x, thr)
        want, scale = _tail_ref(x, thr)
        _check_sums(got, want, scale)
        assert np.array_equal(got, _tail_stats(torch_cuda, x, thr))
    assert _tail_stats(torch_cuda, x, float(finite.min()) - 1.0)[1] == 0


def test_tail_stats_infinite_and_all_nan(torch_cuda):
    rng = np.random.default_rng(1)
    x = rng.normal(0, 0.02, 100_003).astype(np.float32)
    x[[5, 70_000]] = -np.inf
    x[[9, 99_999]] = np.inf
    x[::50] = np.nan
    for thr in (-np.inf, -0.01, 0.0, np.inf):
        got = _tail_stats(torch_cuda, x, thr)
        want, scale = _tail_ref(x, thr)
        _check_sums(got, want, scale)
    y = np.full(70_000, np.nan, dtype=np.float32)
    assert np.array_equal(_tail_stats(torch_cuda, y, 0.0), [0.0, 0.0, 0.0, 0.0])


# ---------------------------------------------------------------------------------------------------------------------
# order statistics
# ---------------------------------------------------------------------------------------------------------------------
def _select(torch, x, ranks):
    from ai_crypto_trader_b200 import _lib
    xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    rk = torch.tensor(list(ranks), dtype=torch.int64, device="cuda")
    need = int(_lib.load().b200bt_select_workspace_bytes(len(ranks)))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(len(ranks), dtype=torch.float32, device="cuda")
    _lib.call("b200bt_select", xd.data_ptr(), int(x.size), rk.data_ptr(), len(ranks), out.data_ptr(), ws.data_ptr(),
              need, _lib.current_stream())
    return out.cpu().numpy()


def _bits(u):
    return np.asarray(u, dtype=np.uint32).view(np.float32)


def _select_keys(kind, n, rng):
    if kind == "equal":
        return np.full(n, np.float32(3.7))
    if kind == "two":
        return np.where(rng.random(n) < 0.3, np.float32(-1.25), np.float32(0.1)).astype(np.float32)
    if kind == "zeros":
        zeros = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0))
        return np.where(rng.random(n) < 0.02, rng.normal(0, 1, n).astype(np.float32), zeros).astype(np.float32)
    if kind == "inf":
        x = rng.normal(0, 1, n).astype(np.float32)
        x[rng.random(n) < 0.05] = np.inf
        x[rng.random(n) < 0.05] = -np.inf
        return x
    if kind == "subnormal":
        x = _bits(rng.integers(1, 1 << 23, n, dtype=np.uint32))
        return np.where(rng.random(n) < 0.5, -x, x).astype(np.float32)
    if kind == "negative":
        return -rng.lognormal(0, 2, n).astype(np.float32)
    if kind == "ulp":                                                     # 1.0 + k ulp: one high-16 bin
        return _bits(0x3F800000 + rng.integers(0, 1 << 16, n, dtype=np.uint32))
    if kind == "edges":                                                   # both sides of high-16 bin edges
        hi = rng.integers(0x3F00, 0x4100, n, dtype=np.uint32) << np.uint32(16)
        lo = np.array([0xFFFE, 0xFFFF, 0x0000, 0x0001], dtype=np.uint32)[rng.integers(0, 4, n)]
        u = np.where(lo >= 0xFFFE, hi - np.uint32(0x10000) + lo, hi + lo).astype(np.uint32)
        x = _bits(u)
        return np.where(rng.random(n) < 0.3, -x, x).astype(np.float32)
    raise KeyError(kind)


@pytest.mark.parametrize("n", [1, 1000, 300_001])
@pytest.mark.parametrize("kind", ["equal", "two", "zeros", "inf", "subnormal", "negative", "ulp", "edges"])
def test_select_exact(torch_cuda, kind, n):
    rng = np.random.default_rng(n)
    x = _select_keys(kind, n, rng)
    xs = np.sort(x)
    spread = sorted(set(np.linspace(0, n - 1, 64).astype(np.int64).tolist()) | {0, n - 1})
    cases = [
        [0, n - 1, n // 2],
        np.linspace(0, n - 1, 64).astype(np.int64).tolist(),               # 64 ranks, repeated when n < 64
        [n - 1, 0, n // 3, n // 3, n - 1],                                  # repeated and unsorted
    ]
    if len(spread) > 3:
        cases.append([spread[1], spread[-2], spread[2], spread[0], spread[-1]])   # a bin's ranks with others between
    for ranks in cases:
        got = _select(torch_cuda, x, ranks)
        assert np.array_equal(got, xs[ranks]), (kind, n, ranks, got, xs[ranks])


def test_select_bins_interleaved(torch_cuda):
    """Ranks in the order bin A, bin B, bin A, B, A: each run of one bin builds its own low-16 histogram."""
    rng = np.random.default_rng(4)
    a = _bits(0x3F800000 + rng.integers(0, 1 << 16, 5000, dtype=np.uint32))          # [1, 1 + 2^-7)
    b = _bits(0x40000000 + rng.integers(0, 1 << 16, 7000, dtype=np.uint32))          # [2, 2 + 2^-6)
    x = rng.permutation(np.concatenate([a, b])).astype(np.float32)
    xs = np.sort(x)
    ranks = [17, 9000, 4999, 5000, 0, 11999, 2500, 2500]
    assert np.array_equal(_select(torch_cuda, x, ranks), xs[ranks])


@pytest.mark.parametrize("conf", [0.0, 0.5, 0.999, 1.0])
def test_var_cvar_at_confidence_limits(torch_cuda, conf):
    from ai_crypto_trader_b200.portfolio_risk import PortfolioRiskService
    rng = np.random.default_rng(7)
    x = rng.normal(1e-3, 0.02, 100_001).astype(np.float32)
    x[::13] = np.nan
    svc = PortfolioRiskService(device="cuda")
    assert svc.calculate_var(x, conf, 3.0) == pytest.approx(portfolio_ref.value_at_risk(x, conf, 3.0), rel=1e-12)
    assert svc.calculate_conditional_var(x, conf, 3.0) == pytest.approx(
        portfolio_ref.conditional_value_at_risk(x, conf, 3.0), rel=1e-9)


# ---------------------------------------------------------------------------------------------------------------------
# moments
# ---------------------------------------------------------------------------------------------------------------------
def _moments_ref(f32, dd32, s0, thr):
    f = f32.astype(np.float64)
    pct = (f / s0 - 1.0) * 100.0
    tail = pct <= thr
    dd = dd32.astype(np.float64) if dd32 is not None else np.zeros(0)
    want = np.array([f.sum(), pct.sum(), (f > s0).sum(), dd.sum(), dd.max() if dd.size else 0.0, pct[tail].sum(),
                     tail.sum()])
    scale = np.array([np.abs(f).sum(), np.abs(pct).sum(), 0, dd.sum(), 0, np.abs(pct[tail]).sum(), 0])
    return want, scale


@pytest.mark.parametrize("which_n", ["1", "255", "257", "grid+1"])
def test_mc_moments(engine, torch_cuda, which_n):
    torch = torch_cuda
    n = {"1": 1, "255": 255, "257": 257,
         "grid+1": torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256 + 1}[which_n]
    rng = np.random.default_rng(n)
    s0 = 100.0
    f = (np.round(rng.lognormal(np.log(s0), 0.2, n) * 4) / 4).astype(np.float32)     # quarter ticks: ties, some == s0
    f[:: 11] = np.float32(s0)
    dd = rng.uniform(0, 0.6, n).astype(np.float32)
    fd, ddd = torch.from_numpy(f).cuda(), torch.from_numpy(dd).cuda()
    tied = float((np.float64(f[n // 2]) / s0 - 1.0) * 100.0)
    for thr in (np.inf, tied, -np.inf):
        for with_dd in (True, False):
            got = engine.moments(fd, ddd if with_dd else None, s0, thr)
            want, scale = _moments_ref(f, dd if with_dd else None, s0, thr)
            for k in (2, 4, 6):
                assert got[k] == want[k], (thr, with_dd, k, got[k], want[k])
            for k in (0, 1, 3, 5):
                assert abs(got[k] - want[k]) <= 1e-12 * scale[k], (thr, with_dd, k, got[k], want[k])
    assert engine.moments(fd, ddd, s0, tied)[6] >= 1


# ---------------------------------------------------------------------------------------------------------------------
# path kernels
# ---------------------------------------------------------------------------------------------------------------------
OFFSET_2_32 = (1 << 32) - 100


@pytest.mark.parametrize("seed", [2024, (0xDEADBEEF << 32) | 7, (1 << 64) - 1])
def test_gbm_counter_limits(engine, seed):
    mu, sigma, dt, s0, n, steps = 0.126, 0.3175, 1 / 252, 100.0, 257, 13
    f, d, _ = engine.gbm(s0, mu, sigma, dt, n, steps, seed, path_offset=OFFSET_2_32)
    fo, do, _ = mc_ref.gbm_paths(s0, mu, sigma, dt, n, steps, seed, path_offset=OFFSET_2_32)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-5)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)
    # sharded at 2^32: the two runs are the one run
    fa, da, _ = engine.gbm(s0, mu, sigma, dt, 100, steps, seed, path_offset=OFFSET_2_32)
    fb, db, _ = engine.gbm(s0, mu, sigma, dt, n - 100, steps, seed, path_offset=1 << 32)
    assert np.array_equal(np.concatenate([fa.cpu().numpy(), fb.cpu().numpy()]), f.cpu().numpy())
    assert np.array_equal(np.concatenate([da.cpu().numpy(), db.cpu().numpy()]), d.cpu().numpy())


@pytest.mark.parametrize("seed", [77, (1 << 64) - 1])
def test_bootstrap_counter_limits(engine, seed):
    ret = np.random.default_rng(3).normal(5e-4, 0.02, 60).astype(np.float32)
    f, d, _ = engine.bootstrap(ret, True, 100.0, 257, 45, seed, path_offset=OFFSET_2_32, block_len=3)
    fo, do, _ = mc_ref.bootstrap_paths(ret, True, 100.0, 257, 45, seed, path_offset=OFFSET_2_32, block_len=3)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=1e-6)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=1e-5, atol=1e-7)
    fa, _, _ = engine.bootstrap(ret, True, 100.0, 100, 45, seed, path_offset=OFFSET_2_32, block_len=3)
    fb, _, _ = engine.bootstrap(ret, True, 100.0, 157, 45, seed, path_offset=1 << 32, block_len=3)
    assert np.array_equal(np.concatenate([fa.cpu().numpy(), fb.cpu().numpy()]), f.cpu().numpy())


def _block_lens(R, steps):
    return sorted({b for b in (R - 1, R, R + 1, steps + 1) if b >= 1})


@pytest.mark.parametrize("R", [1, 7, MC_MAX_TABLE])
@pytest.mark.parametrize("log_returns", [True, False])
def test_bootstrap_table_limits(engine, R, log_returns):
    rng = np.random.default_rng(R)
    ret = rng.normal(5e-4, 0.02, R).astype(np.float32)
    steps = 45
    for block_len in _block_lens(R, steps):
        f, d, _ = engine.bootstrap(ret, log_returns, 100.0, 2000, steps, 11, block_len=block_len)
        fo, do, _ = mc_ref.bootstrap_paths(ret, log_returns, 100.0, 2000, steps, 11, block_len=block_len)
        np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=(1e-6 if log_returns else 3e-6), err_msg=str(block_len))
        np.testing.assert_allclose(d.cpu().numpy(), do, rtol=1e-5, atol=1e-7, err_msg=str(block_len))


def test_bootstrap_total_loss(engine):
    """A simple return of -1 (a close of 0) in the table: paths that draw it end at 0 with a drawdown of 1, no NaN."""
    ret = np.random.default_rng(5).normal(5e-4, 0.02, 20).astype(np.float32)
    ret[7] = -1.0
    f, d, p = engine.bootstrap(ret, False, 100.0, 1000, 30, 3, block_len=2, store_paths=True)
    f, d, p = f.cpu().numpy(), d.cpu().numpy(), p.cpu().numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        fo, do, _ = mc_ref.bootstrap_paths(ret, False, 100.0, 1000, 30, 3, block_len=2)
    assert not np.isnan(f).any() and not np.isnan(d).any() and not np.isnan(p).any()
    lost = fo == 0
    assert 0 < lost.sum() < lost.size
    assert (f[lost] == 0).all() and (d[lost] == 1).all() and (do[lost] == 1).all()
    np.testing.assert_allclose(f[~lost], fo[~lost], rtol=3e-6)
    np.testing.assert_allclose(d, do, rtol=1e-5, atol=1e-7)


def test_joint_bootstrap_full_table(engine):
    S, R = 32, MC_MAX_TABLE // 32
    rng = np.random.default_rng(32)
    table = rng.normal(5e-4, 0.02, (R, S)).astype(np.float32)
    s0, qty = rng.uniform(1, 100, S), rng.uniform(0.1, 5, S)
    for log_returns, block_len in ((True, 1), (False, R + 1)):
        f, d, af = engine.portfolio_bootstrap(table, log_returns, s0, qty, 777, 60, 11, block_len=block_len,
                                              asset_finals=True)
        fo, do, afo, _ = mc_joint_ref.joint_bootstrap_paths(table, log_returns, s0, qty, 777, 60, 11, block_len=block_len)
        np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-6)
        np.testing.assert_allclose(af.cpu().numpy(), afo, rtol=3e-6)
        np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)


def test_joint_gbm_counter_limits(engine):
    S = 5
    rng = np.random.default_rng(5)
    A = rng.normal(size=(S, S + 2))
    c = A @ A.T
    c = c / np.sqrt(np.outer(np.diag(c), np.diag(c)))
    L = np.linalg.cholesky(c).astype(np.float32)
    s0, qty = rng.uniform(1, 100, S), rng.uniform(0.1, 5, S)
    mu, sigma = rng.uniform(-0.3, 0.4, S), rng.uniform(0.1, 0.9, S)
    seed = (1 << 64) - 1
    f, d, af = engine.portfolio_gbm(s0, qty, mu, sigma, 1 / 252, L, 257, 9, seed, path_offset=OFFSET_2_32,
                                    asset_finals=True)
    fo, do, afo = mc_joint_ref.joint_gbm_paths(s0, qty, mu, sigma, 1 / 252, L, 257, 9, seed, path_offset=OFFSET_2_32)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-5)
    np.testing.assert_allclose(af.cpu().numpy(), afo, rtol=3e-5)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)
