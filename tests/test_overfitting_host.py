"""The CSCV oracles (tests/cscv_ref.py) against each other and against known answers, and the host statistics of
ai_crypto_trader_b200/overfitting.py (PBO summary, Deflated Sharpe Ratio) against independent restatements.  CPU only."""
import math

import numpy as np
import pytest

import cscv_ref


def _noise(N, T, seed):
    return np.random.default_rng(seed).normal(0.0, 1.0, (N, T))


@pytest.mark.parametrize("N, T, B, seed", [(7, 101, 4, 1), (40, 333, 8, 2), (25, 250, 10, 3), (12, 96, 6, 4)])
def test_exact_and_literal_agree(N, T, B, seed):
    """The contract's arithmetic (ascending sums of per-block deviations) and the paper's literal algorithm (concatenated
    blocks, np.mean / np.std) select the same trials, give the same ranks and the same PBO, on cases whose in-sample
    winners are separated by more than the rounding difference of the two formulations."""
    x = _noise(N, T, seed) + np.linspace(-0.05, 0.05, N)[:, None]
    ex, lit = cscv_ref.cscv_exact(x, B), cscv_ref.cscv_literal(x, B)
    assert ex["is_gap"].min() > 1e-12
    np.testing.assert_array_equal(ex["sel"], lit["sel"])
    from ai_crypto_trader_b200.overfitting import summarize
    s = summarize(ex["is_sr"], ex["oos_sr"], ex["n_below"], ex["n_tied"], N)
    np.testing.assert_allclose(s["omega"], lit["omega"], rtol=0, atol=1e-15)
    assert s["pbo"] == lit["pbo"]
    assert ex["dropped_days"] == T % B and ex["block_days"] == T // B


def test_iid_noise_is_a_coin_flip():
    x = _noise(100, 1000, 7)
    ex = cscv_ref.cscv_exact(x, 16)
    from ai_crypto_trader_b200.overfitting import summarize
    s = summarize(ex["is_sr"], ex["oos_sr"], ex["n_below"], ex["n_tied"], 100)
    assert 0.3 <= s["pbo"] <= 0.7, s["pbo"]


def test_a_persistent_edge_is_not_overfit():
    x = _noise(50, 800, 8)
    x[17] += 0.6
    ex = cscv_ref.cscv_exact(x, 16)
    from ai_crypto_trader_b200.overfitting import summarize
    s = summarize(ex["is_sr"], ex["oos_sr"], ex["n_below"], ex["n_tied"], 50)
    assert np.all(ex["sel"] == 17)
    assert s["pbo"] == 0.0 and np.all(s["logit"] > 0)


def test_a_ranking_that_reverses_out_of_sample_is_overfit():
    """Every trial has the same full-sample mean, spread unevenly over the blocks: a set of blocks with a high mean leaves
    its complement with a low one, so the in-sample winner is near the bottom out of sample."""
    rng = np.random.default_rng(9)
    N, B, L = 40, 12, 50
    z = rng.normal(0, 1, (N, B))
    z -= z.mean(axis=1, keepdims=True)
    x = 1.0 + 0.3 * np.repeat(z, L, axis=1) + 0.5 * rng.normal(0, 1, (N, B * L))
    ex = cscv_ref.cscv_exact(x, B)
    from ai_crypto_trader_b200.overfitting import summarize
    s = summarize(ex["is_sr"], ex["oos_sr"], ex["n_below"], ex["n_tied"], N)
    assert s["pbo"] > 0.9, s["pbo"]
    assert s["degradation"]["slope"] < 0


def test_combination_order_is_itertools():
    m = cscv_ref.combination_masks(6)
    assert m.shape == (20, 6) and m[0].tolist() == [True] * 3 + [False] * 3 and m[-1].tolist() == [False] * 3 + [True] * 3


def _dsr_scipy(mu, m2, m3, m4, N, T):
    from scipy.stats import norm
    sr = mu / np.sqrt(m2)
    skew, kurt = m3 / m2 ** 1.5, m4 / m2 ** 2
    g = np.euler_gamma
    sr0 = np.std(sr) * ((1 - g) * norm.ppf(1 - 1 / N) + g * norm.ppf(1 - 1 / (N * np.e)))
    return norm.cdf((sr - sr0) * np.sqrt(T - 1) / np.sqrt(1 - skew * sr + (kurt - 1) / 4 * sr ** 2))


def test_deflated_sharpe_matches_a_scipy_restatement():
    from ai_crypto_trader_b200.overfitting import deflated_sharpe
    x = _noise(64, 520, 10) * 0.02 + np.linspace(0, 0.004, 64)[:, None]
    x[5] += np.random.default_rng(1).exponential(0.01, 520)       # a skewed, fat-tailed trial
    mom = cscv_ref.moments(x, 16)
    res = dict(mom, n_blocks=16, block_days=mom["L"])
    got = deflated_sharpe(res, 64)
    want = _dsr_scipy(mom["mu"], mom["m2"], mom["m3"], mom["m4"], 64, 16 * mom["L"])
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    assert got.min() < 0.5 < got.max()
    # zero variance: NaN; fewer than two trials: refused
    res["m2"] = res["m2"].copy()
    res["m2"][0] = 0.0
    assert math.isnan(deflated_sharpe(res, 64)[0])
    with pytest.raises(ValueError):
        deflated_sharpe(res, 1)


def test_lane_rows_bucket_by_calendar_day():
    from oracle import sim_oracle
    cfg = sim_oracle.config_of(1440 * 100 + 1400, 7, gap_bar=30, gap_minutes=3 * 1440)
    first, D = cscv_ref.calendar(cfg, 40)
    assert first == 100 and D == (1440 * 100 + 1400 + 39 * 7 + 3 * 1440) // 1440 - 100 + 1
    ev = np.array([0, 5 | 0x40000000, 29, 30 | 0x40000000], dtype=np.uint32)
    row = cscv_ref.lane_rows(ev, [1.0, 2.0, 4.0, 8.0], cfg, 40)
    # bars 0 and 5 end before midnight (minute 1435 of day 100), bar 29 is on day 101, bar 30 after the 3-day gap on 104
    assert row.tolist() == [3.0, 4.0, 0.0, 0.0, 8.0]
