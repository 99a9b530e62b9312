"""Model Confidence Set on the GPU (csrc/overfitting.cu b200bt_boot_means / b200bt_autocov / b200bt_mcs_*,
overfitting.mcs / optimal_block_length, StrategyEvaluationSystem.model_confidence_set) bit for bit against the exact
restatement of tests/mcs_ref.py."""
import numpy as np
import pytest

import mcs_ref
import spa_ref
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu
BIG = 1 << 40


def _bits_equal(a, b, what):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    assert a.shape == b.shape, what
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (what, np.nanmax(np.abs(a - b)))


def _dev(torch, x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


def _boot_means(torch, x, q32, n_boot, seed, boot_offset, ld=None, ld_out=None, center=None):
    from ai_crypto_trader_b200 import _lib
    N, T = x.shape
    buf = np.zeros((N, ld or T))
    buf[:, :T] = x
    d = _dev(torch, buf)
    ldo = ld_out or N
    out = torch.full((n_boot, ldo), 7.0, dtype=torch.float64, device="cuda")
    c = None if center is None else _dev(torch, center)
    _lib.call("b200bt_boot_means", d.data_ptr(), buf.shape[1], N, T, q32, n_boot, seed, boot_offset,
              None if c is None else c.data_ptr(), out.data_ptr(), ldo, BIG, _lib.current_stream())
    o = out.cpu().numpy()
    assert np.all(o[:, N:] == 7.0)                           # the padding of ld_out is not written
    return o[:, :N]


@pytest.mark.parametrize("N, T, block_len, B", [(1, 2, 10.0, 70), (31, 768, 4.0, 40), (33, 769, 10.0, 40),
                                                (65, 129, 1.0, 65), (3, 8192, 25.0, 9)])
def test_boot_means_match_the_restatement_across_seams_and_splits(torch_cuda, N, T, block_len, B):
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(N + T)
    x = rng.normal(0.0, 1.0, (N, T)) * rng.uniform(0.1, 3.0, (N, 1))
    q32 = spa_q32(block_len)
    want = mcs_ref.boot_means_exact(x, q32, 5, B, 3)
    _bits_equal(_boot_means(torch_cuda, x, q32, B, 5, 3, ld=T + 5, ld_out=N + 3), want, "one call, padded ld")
    h = B // 3
    parts = np.vstack([_boot_means(torch_cuda, x, q32, h, 5, 3), _boot_means(torch_cuda, x, q32, B - h, 5, 3 + h)])
    _bits_equal(parts, want, "two boot_offset parts")
    mean = mcs_ref.mean_exact(x)
    _bits_equal(_boot_means(torch_cuda, x, q32, B, 5, 3, center=mean), want - mean[None, :], "centred")


def test_boot_means_equal_the_spa_bootstrap_one_hot_maxima(torch_cuda):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.overfitting import spa_q32
    rng = np.random.default_rng(2)
    N, T, B = 37, 300, 90
    x = rng.normal(0.0, 0.02, (N, T))
    q32 = spa_q32(6.0)
    got = _boot_means(torch_cuda, x, q32, B, 9, 11)
    d = _dev(torch_cuda, x)
    for lo in range(0, N, 8):
        ks = list(range(lo, min(N, lo + 8)))
        shift = np.full((len(ks), N), np.inf)
        shift[np.arange(len(ks)), ks] = 0.0
        sh, sc = _dev(torch_cuda, shift), _dev(torch_cuda, np.ones((len(ks), N)))
        out = torch_cuda.empty((len(ks), B), dtype=torch_cuda.float64, device="cuda")
        _lib.call("b200bt_spa_bootstrap", d.data_ptr(), T, N, T, q32, B, 9, 11, len(ks), sh.data_ptr(), sc.data_ptr(),
                  out.data_ptr(), _lib.current_stream())
        _bits_equal(out.cpu().numpy(), got[:, ks].T, f"trials {ks}")


@pytest.mark.parametrize("N, T, K", [(1, 2, 1), (40, 695, 40), (3, 8192, 100)])
def test_autocov_equals_the_spa_moments_gamma(torch_cuda, N, T, K):
    from ai_crypto_trader_b200.overfitting import autocov
    rng = np.random.default_rng(T)
    x = rng.normal(0.0, 1.0, (N, T))
    x[:, 1:] += 0.6 * x[:, :-1]
    if N > 2:
        x[1] = 0.0
    acov, mean = autocov(_dev(torch_cuda, x), K)
    _bits_equal(acov.cpu().numpy(), mcs_ref.autocov_exact(x, K), "gamma")
    _bits_equal(mean.cpu().numpy(), spa_ref.moments_exact(x, 0.5)[0], "mean")


def _rows_with_copies(rng, N, T):
    x = rng.normal(0.0, 1.0, (N, T)) + np.linspace(-0.3, 0.3, N)[:, None]
    if N < 8:                                                # one all-zero row
        x[0] = 0.0
        return x
    x[N // 2] = 0.0                                          # never trading
    x[N // 2 + 1] = 0.0
    x[3] = x[7]                                              # duplicate
    return x


@pytest.mark.parametrize("N", [2, 33, 70])
def test_pairwise_pass_and_range_stats_match(torch_cuda, N):
    from ai_crypto_trader_b200 import _lib
    rng = np.random.default_rng(N)
    B = 150
    zeta = rng.normal(0.0, 0.1, (B, N))
    zeta[:, 1] = zeta[:, 0]                                  # sigma = 0
    mean = rng.normal(0.0, 0.01, N)
    mean[1] = mean[0]
    if N > 5:
        zeta[:, 5] = zeta[:, 4]
        mean[5] = mean[4] + 1e-3                             # sigma = 0, means differ: +-inf
    s2, rho, t = mcs_ref.range_stats_exact(zeta, mean)
    z = _dev(torch_cuda, zeta)
    w = torch_cuda.zeros((N, N), dtype=torch_cuda.float64, device="cuda")
    st = _lib.current_stream()
    for lo, hi in ((0, 17), (17, 100), (100, B)):            # three launches continue one ascending sum
        _lib.call("b200bt_mcs_pairwise", z[lo:].data_ptr(), N, N, hi - lo, w.data_ptr(), BIG, st)
    iu = np.triu_indices(N, 1)
    _bits_equal(w.cpu().numpy()[iu], s2[iu], "s2")
    tt = torch_cuda.empty((N, N), dtype=torch_cuda.float64, device="cuda")
    _lib.call("b200bt_mcs_range_stats", _dev(torch_cuda, mean).data_ptr(), N, B, w.data_ptr(), tt.data_ptr(), BIG, st)
    _bits_equal(w.cpu().numpy(), rho, "rho")
    _bits_equal(tt.cpu().numpy(), t, "t")
    if N > 5:
        assert tt[4, 5].item() == np.inf and tt[5, 4].item() == -np.inf and tt[0, 1].item() == 0.0


@pytest.mark.parametrize("statistic", ["R", "max"])
@pytest.mark.parametrize("N, T, B", [(2, 40, 200), (40, 120, 300), (70, 61, 150)])
def test_mcs_matches_the_exact_restatement(torch_cuda, statistic, N, T, B):
    from ai_crypto_trader_b200.overfitting import mcs
    x = _rows_with_copies(np.random.default_rng(N * T), N, T)
    got = mcs(_dev(torch_cuda, x), alpha=0.1, statistic=statistic, n_boot=B, block_len=5.0, seed=4)
    want = mcs_ref.mcs_exact(x, 0.1, statistic, B, 5.0, 4)
    np.testing.assert_array_equal(got["elimination_order"], want["elimination_order"])
    _bits_equal(got["step_stats"], want["step_stats"], "step stats")
    _bits_equal(got["step_pvalues"], want["step_pvalues"], "step p-values")
    _bits_equal(got["p_values"], want["p_values"], "MCS p-values")
    np.testing.assert_array_equal(got["included"], want["included"])
    _bits_equal(got["mean"], want["mean"], "mean")
    np.testing.assert_array_equal(got["model_of"], want["model_of"])
    assert got["n_models"] == want["n_models"] == (N - 2 if N >= 8 else N)
    assert np.all(np.diff(got["p_values"][got["elimination_order"]]) >= 0)
    if N >= 8:                                               # copies share one p-value
        assert got["p_values"][N // 2] == got["p_values"][N // 2 + 1] and got["p_values"][3] == got["p_values"][7]


def test_identical_rows_stay_at_p_one_on_both_statistics(torch_cuda):
    from ai_crypto_trader_b200.overfitting import mcs
    for x in (np.zeros((5, 30)), np.tile(np.random.default_rng(1).normal(0, 1, 30), (4, 1))):
        for stat in ("R", "max"):
            r = mcs(_dev(torch_cuda, x), statistic=stat, n_boot=100)
            assert r["included"].all() and np.all(r["p_values"] == 1.0) and r["n_models"] == 1, stat


@pytest.mark.parametrize("statistic", ["R", "max"])
@pytest.mark.parametrize("seed", [0, 2, 5])
def test_copies_of_the_best_row_stand_together(torch_cuda, statistic, seed):
    from ai_crypto_trader_b200.overfitting import mcs
    rng = np.random.default_rng(seed)
    best = rng.normal(1.0, 0.01, 120)
    x = np.vstack([rng.normal(0.0, 0.01, (2, 120)), np.tile(best, (4, 1)), rng.normal(0.0, 0.01, (2, 120)),
                   np.tile(best, (3, 1))])
    got = mcs(_dev(torch_cuda, x), statistic=statistic, n_boot=200, block_len=5.0, seed=seed)
    want = mcs_ref.mcs_exact(x, 0.1, statistic, 200, 5.0, seed)
    for k in ("p_values", "step_pvalues", "step_stats", "elimination_order", "model_of"):
        np.testing.assert_array_equal(got[k], want[k])
    copies = [2, 3, 4, 5, 8, 9, 10]
    assert np.all(got["p_values"][copies] == 1.0) and got["n_models"] == 5


def test_split_resamples_give_the_same_result(torch_cuda):
    from ai_crypto_trader_b200.overfitting import mcs
    N, B = 30, 500
    x = _rows_with_copies(np.random.default_rng(5), N, 90)
    whole = mcs(_dev(torch_cuda, x), n_boot=B, block_len=3.0, seed=7)
    D = whole["n_models"]
    per = 64                                                 # resamples per launch over the D distinct models
    split = mcs(_dev(torch_cuda, x), n_boot=B, block_len=3.0, seed=7, max_bytes=2 * D * D * 8 + 2 * D * 8 * per)
    for k in ("p_values", "step_pvalues", "step_stats", "elimination_order"):
        np.testing.assert_array_equal(split[k], whole[k])
    with pytest.raises(ValueError):
        mcs(_dev(torch_cuda, x), n_boot=B, max_bytes=2 * D * D * 8)
    with pytest.raises(ValueError):
        mcs(_dev(torch_cuda, x), statistic="max", n_boot=B, max_bytes=B * D * 8 - 1)
    with pytest.raises(ValueError):
        mcs(_dev(torch_cuda, np.full((3, 20), np.nan)))
    with pytest.raises(ValueError):
        mcs(_dev(torch_cuda, np.zeros((1, 20))))


def test_auto_block_length_uses_the_device_lags(torch_cuda):
    from ai_crypto_trader_b200.overfitting import block_length_rule, mcs, optimal_block_length, spa
    rng = np.random.default_rng(9)
    T = 400
    e = rng.normal(0.0, 1.0, (12, T))
    x = e.copy()
    for t in range(1, T):
        x[:, t] += 0.7 * x[:, t - 1]
    x[0] = 0.0                                               # no estimate
    res = optimal_block_length(_dev(torch_cuda, x))
    K = min(int(np.ceil(np.sqrt(T))) + 2 * 5, T - 1)
    per_row, b = block_length_rule(mcs_ref.autocov_exact(x, K), T)
    np.testing.assert_array_equal(res["per_row"], per_row)
    assert res["block_len"] == b and np.isnan(res["per_row"][0]) and b > 3.0
    r = mcs(_dev(torch_cuda, x), n_boot=100, block_len="auto")
    assert r["block_len"] == b
    s = spa(_dev(torch_cuda, x), n_boot=100, block_len="auto")
    assert s["block_len"] == optimal_block_length(_dev(torch_cuda, x))["block_len"]


def test_model_confidence_set_end_to_end(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.overfitting import mcs
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    market = MarketData(synth.synth_ohlcv(2, 40_000))
    base = synth.random_population(30, seed=4)
    pop = base + [dict(base[3]), dict(base[0])]
    incumbent = dict(synth.random_population(1, seed=99)[0])
    ses = StrategyEvaluationSystem(config={})
    sweep = PopulationSweep(market)
    kw = dict(n_boot=300, block_len=5.0, seed=3)
    res = ses.model_confidence_set(pop, market, incumbent=incumbent, sweep=sweep, **kw)
    _, unique, expand = sweep._unique(pop)
    book, _, first = sweep.daily_pnl(unique)
    inc_row = sweep.daily_pnl([incumbent])[0]
    rows = np.vstack([book.cpu().numpy(), inc_row.cpu().numpy()])
    want = mcs(_dev(torch_cuda, rows), **kw)
    assert res["n_trials"] == len(unique) + 1 and res["first_day"] == first
    np.testing.assert_array_equal(res["p_values"], want["p_values"][:-1][expand])
    assert res["p_values"][30] == res["p_values"][3] and res["p_values"][31] == res["p_values"][0]
    assert res["incumbent"]["p_value"] == want["p_values"][-1]
    assert res["incumbent"]["included"] == (want["p_values"][-1] >= 0.10)
    exact = mcs_ref.mcs_exact(rows, 0.10, "R", 300, 5.0, 3)
    np.testing.assert_array_equal(want["p_values"], exact["p_values"])
    assert ses.model_confidence_set(pop, market, block_len=0.5, sweep=sweep) == {}
    assert ses.data_snooping(pop, market, block_len="auto", n_boot=100, sweep=sweep)["block_len"] >= 1.0
