"""Data-snooping tests on the GPU (csrc/overfitting.cu b200bt_spa_moments / b200bt_spa_bootstrap, overfitting.spa,
StrategyEvaluationSystem.data_snooping) bit for bit against the exact restatement of tests/spa_ref.py."""
import math

import numpy as np
import pytest

import spa_ref
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu


def _bits_equal(a, b, what):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    assert a.shape == b.shape, what
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (what, np.nanmax(np.abs(a - b)))


def _same(a, b):
    """Dicts of floats equal, NaN equal to NaN."""
    return a.keys() == b.keys() and all(a[k] == b[k] or (math.isnan(a[k]) and math.isnan(b[k])) for k in a)


def _dev(torch, x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


def _boot(torch, d, q32, n_boot, seed, boot_offset, shift, scale, ld=None):
    """b200bt_spa_bootstrap on host arrays; d may be a padded [N][ld] view."""
    from ai_crypto_trader_b200 import _lib
    N, T = d.shape
    buf = np.zeros((N, ld or T))
    buf[:, :T] = d
    dd, sh, sc = _dev(torch, buf), _dev(torch, np.atleast_2d(shift)), _dev(torch, np.atleast_2d(scale))
    out = torch.empty((sh.shape[0], n_boot), dtype=torch.float64, device="cuda")
    _lib.call("b200bt_spa_bootstrap", dd.data_ptr(), buf.shape[1], N, T, q32, n_boot, seed, boot_offset, sh.shape[0],
              sh.data_ptr(), sc.data_ptr(), out.data_ptr(), _lib.current_stream())
    return out.cpu().numpy()


def _moments(torch, d, q):
    from ai_crypto_trader_b200 import _lib
    N, T = d.shape
    dd = _dev(torch, d)
    mean = torch.empty(N, dtype=torch.float64, device="cuda")
    omega2 = torch.empty(N, dtype=torch.float64, device="cuda")
    _lib.call("b200bt_spa_moments", dd.data_ptr(), T, N, T, q, mean.data_ptr(), omega2.data_ptr(), _lib.current_stream())
    return mean.cpu().numpy(), omega2.cpu().numpy()


def _stats(rng, N, n_stats, exclude=0.3):
    shift = rng.normal(0.0, 0.05, (n_stats, N))
    shift[rng.random((n_stats, N)) < exclude] = np.inf
    scale = rng.uniform(0.5, 20.0, (n_stats, N))
    return shift, scale


# (N, T, block_len, n_stats, B): trial tiles of 32 (N = 1, 31, 33, 65), odd T (half a Philox block), the smallest and
# largest T, the largest staged T (768) and the first one read through L2 (769), q = 1 and a q so small that most
# resamples are one block, 1 and 8 statistics
CASES = [(1, 2, 10.0, 1, 300), (33, 7, 3.0, 8, 500), (31, 64, 1.0, 4, 257), (65, 695, 10.0, 4, 200),
         (40, 768, 2.0, 2, 100), (40, 769, 10.0, 8, 100), (3, 8192, 10.0, 3, 48), (2, 8192, 1.0, 1, 17),
         (100, 129, 2.0 ** 40, 8, 64)]


@pytest.mark.parametrize("N, T, block_len, n_stats, B", CASES)
def test_bootstrap_maxima_match_the_exact_restatement(torch_cuda, N, T, block_len, n_stats, B):
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(N * 7 + T)
    d = rng.normal(0.0, 1.0, (N, T)) * rng.uniform(0.1, 3.0, (N, 1))
    shift, scale = _stats(rng, N, n_stats)
    shift[0] = np.inf                                        # every trial excluded: -inf
    if n_stats > 1:
        shift[1] = 0.0                                       # none excluded
    q32 = spa_q32(block_len)
    got = _boot(torch_cuda, d, q32, B, 77, 5, shift, scale, ld=T + 3)
    want = spa_ref.maxima_exact(d, q32, 77, 5, B, shift, scale)
    _bits_equal(got, want, f"N={N} T={T}")
    assert np.all(got[0] == -np.inf)
    if block_len == 2.0 ** 40:                               # q32 = 1: one block per resample, nearly always
        starts = spa_ref.block_starts(T, q32, 77, np.arange(B, dtype=np.uint64) + np.uint64(5))
        assert starts[:, 1:].sum() <= 1


def test_one_hot_shifts_recover_every_bootstrap_mean(torch_cuda):
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(3)
    N, T, B = 21, 333, 150
    d = rng.normal(0.001, 0.02, (N, T))
    q32 = spa_q32(7.0)
    theta = spa_ref.index_stream(T, q32, 11, np.arange(B, dtype=np.uint64))
    want = spa_ref.boot_means_exact(d, theta)
    for lo in range(0, N, 8):
        ks = list(range(lo, min(N, lo + 8)))
        shift = np.full((len(ks), N), np.inf)
        shift[np.arange(len(ks)), ks] = 0.0
        got = _boot(torch_cuda, d, q32, B, 11, 0, shift, np.ones((len(ks), N)))
        _bits_equal(got, want[ks], f"trials {ks}")


def test_resample_split_and_trial_order_do_not_matter(torch_cuda):
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(4)
    N, T, B = 70, 200, 301
    d = rng.normal(0.0, 1.0, (N, T))
    shift, scale = _stats(rng, N, 4)
    q32 = spa_q32(10.0)
    whole = _boot(torch_cuda, d, q32, B, 2 ** 40 + 9, 1000, shift, scale)
    half = 137
    parts = np.hstack([_boot(torch_cuda, d, q32, half, 2 ** 40 + 9, 1000, shift, scale),
                       _boot(torch_cuda, d, q32, B - half, 2 ** 40 + 9, 1000 + half, shift, scale)])
    _bits_equal(parts, whole, "two boot_offset halves")
    perm = rng.permutation(N)
    _bits_equal(_boot(torch_cuda, d[perm], q32, B, 2 ** 40 + 9, 1000, shift[:, perm], scale[:, perm]), whole, "permuted")
    _bits_equal(whole, _boot(torch_cuda, d, q32, B, 2 ** 40 + 9, 1000, shift, scale), "repeated")


@pytest.mark.parametrize("N, T, block_len", [(1, 2, 10.0), (37, 695, 10.0), (5, 8192, 25.0), (300, 61, 1.0)])
def test_moments_match_the_restatement(torch_cuda, N, T, block_len):
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(N + T)
    d = rng.normal(0.0, 1.0, (N, T))
    d[:, 1:] += 0.5 * d[:, :-1]
    if N > 2:
        d[1] = 0.0                                           # omega2 exactly 0
    q = spa_q32(block_len) / 2.0 ** 32
    mean, omega2 = _moments(torch_cuda, d, q)
    want_mean, want_omega2 = spa_ref.moments_exact(d, q)
    _bits_equal(mean, want_mean, "mean")
    _bits_equal(omega2, want_omega2, "omega2")
    if block_len == 1.0:
        _, g0 = spa_ref.moments_exact(d, 1.0)
        _bits_equal(omega2, g0, "q = 1: gamma_0")
    # the header's tolerance against kappa by pow
    if T <= 695:
        hansen = np.array([spa_ref.hansen_omega2(r, q) for r in d])
        c = d - mean[:, None]
        bound = T * 2.0 ** -52 * (np.abs(hansen) + 2 * (c * c).sum(axis=1)) + 1e-13 * np.abs(hansen)
        assert np.all(np.abs(omega2 - hansen) <= bound)


def _spa_vs_exact(torch, x, bench, **kw):
    from ai_crypto_trader_b200.overfitting import spa, spa_q32
    got = spa(_dev(torch, x), None if bench is None else _dev(torch, bench), **kw)
    d = x if bench is None else x - bench[None, :]
    mean, omega2 = _moments(torch, d, spa_q32(kw["block_len"]) / 2.0 ** 32)
    want = spa_ref.spa_exact(d, kw["n_boot"], kw["block_len"], kw["alpha"], kw["seed"], moments=(mean, omega2))
    assert got["reality_check"] == want["reality_check"] and _same(got["spa"], want["spa"])
    assert np.array_equal(got["stepm"]["rejected"], want["stepm"]["rejected"])
    assert got["stepm"]["critical_values"] == want["stepm"]["critical_values"]
    _bits_equal(got["mean"], mean, "mean")
    _bits_equal(got["t_stat"], want["t_stat"], "t_stat")
    assert got["best"] == want["best"]
    return got


def test_spa_matches_the_restatement_and_chunks(torch_cuda):
    rng = np.random.default_rng(8)
    N, T = 90, 300
    x = rng.normal(0.0, 1.0, (N, T))
    bench = rng.normal(0.05, 0.5, T)
    x[[4, 50, 88]] += 0.45                                   # edged
    x[10] = bench                                            # equals the benchmark: no variance, excluded
    kw = dict(n_boot=1000, block_len=10.0, alpha=0.05, seed=12)
    whole = _spa_vs_exact(torch_cuda, x, bench, **kw)
    assert {4, 50, 88} <= set(np.flatnonzero(whole["stepm"]["rejected"])) and math.isnan(whole["t_stat"][10])
    assert whole["spa"]["pvalue_lower"] <= whole["spa"]["pvalue_consistent"] <= whole["spa"]["pvalue_upper"]
    chunked = _spa_vs_exact(torch_cuda, x, bench, max_out_bytes=4 * 8 * 333, **kw)     # four launches per statistic row
    for k in ("reality_check", "spa"):
        assert chunked[k] == whole[k]
    assert chunked["stepm"]["critical_values"] == whole["stepm"]["critical_values"]
    noise = _spa_vs_exact(torch_cuda, rng.normal(0.0, 1.0, (33, 61)), None, n_boot=500, block_len=3.0, alpha=0.1, seed=1)
    assert noise["n_trials"] == 33 and noise["n_days"] == 61 and noise["n_boot"] == 500


def test_spa_without_eligible_trials_gives_nan(torch_cuda):
    from ai_crypto_trader_b200.overfitting import spa
    res = spa(_dev(torch_cuda, np.zeros((4, 30))), n_boot=50)
    assert all(math.isnan(res["spa"][k]) for k in ("stat", "pvalue_lower", "pvalue_consistent", "pvalue_upper"))
    assert res["best"] is None and not res["stepm"]["rejected"].any() and res["stepm"]["critical_values"] == []
    assert res["reality_check"]["stat"] == 0.0 and np.all(np.isnan(res["t_stat"]))
    with pytest.raises(ValueError):
        spa(_dev(torch_cuda, np.full((2, 30), np.nan)))


def test_data_snooping_end_to_end(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(2, 40_000))
    base = synth.random_population(30, seed=4)
    pop = base + [dict(base[3]), dict(base[0])]              # duplicates: one trial each
    ses = StrategyEvaluationSystem(config={})
    sweep = PopulationSweep(market)
    kw = dict(n_boot=400, block_len=5.0, alpha=0.05, seed=3)
    res = ses.data_snooping(pop, market, sweep=sweep, **kw)
    book, _, first = sweep.daily_pnl(pop)
    _, unique, expand = sweep._unique(pop)
    assert res["n_trials"] == len(unique) <= len(base) and res["first_day"] == first
    rows = book.cpu().numpy()
    want = _spa_vs_exact(torch_cuda, rows[[pop.index(u) for u in unique]], None, **kw)
    assert res["reality_check"] == want["reality_check"] and res["stepm"]["critical_values"] == want["stepm"]["critical_values"]
    _bits_equal(res["mean"], want["mean"][expand], "mean in population order")
    assert res["mean"][30] == res["mean"][3] and res["mean"][31] == res["mean"][0]
    np.testing.assert_array_equal(res["stepm"]["rejected"], want["stepm"]["rejected"][expand])
    if res["best"] is not None:
        assert res["t_stat"][res["best"]["index"]] == res["best"]["t_stat"] == np.nanmax(res["t_stat"])
    # the incumbent: a member of the population as the benchmark
    vs = ses.data_snooping(pop, market, benchmark=dict(base[7]), sweep=sweep, **kw)
    bench = rows[7]
    want_b = _spa_vs_exact(torch_cuda, rows[[pop.index(u) for u in unique]], bench, **kw)
    assert vs["mean"][7] == 0.0 and math.isnan(vs["t_stat"][7]) and not vs["stepm"]["rejected"][7]
    assert _same(vs["spa"], want_b["spa"]) and vs["reality_check"] == want_b["reality_check"]
    assert ses.data_snooping(pop, market, block_len=0.5, sweep=sweep) == {}
