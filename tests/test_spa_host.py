"""Properties of the data-snooping restatements (tests/spa_ref.py), which the GPU tests hold the kernels to: the
stationary-bootstrap index stream, Hansen's variance estimate, the exact path against the literal one, and the
behaviour of the Reality Check, SPA and StepM on data whose answer is known.  No GPU."""
import math

import numpy as np
import pytest

import spa_ref
from ai_crypto_trader_b200.overfitting import spa_q32

N, T, B = 40, 250, 1000


def test_q32_is_the_rounded_restart_threshold():
    assert spa_q32(1.0) == 1 << 32 and spa_q32(10.0) == round(2 ** 32 / 10) and spa_q32(2.0 ** 40) == 1
    for bad in (0.5, 0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError):
            spa_q32(bad)


@pytest.mark.parametrize("T_, block_len", [(2, 10.0), (7, 3.0), (250, 10.0), (695, 10.0), (1000, 1e6)])
def test_blocks_are_runs_of_consecutive_days(T_, block_len):
    q32 = spa_q32(block_len)
    gids = np.arange(300, dtype=np.uint64) + np.uint64(1 << 33)
    theta = spa_ref.index_stream(T_, q32, 12345, gids)
    starts = spa_ref.block_starts(T_, q32, 12345, gids)
    assert theta.min() >= 0 and theta.max() < T_
    cont = ~starts[:, 1:]
    assert np.all(theta[:, 1:][cont] == (theta[:, :-1][cont] + 1) % T_)      # inside a block: the next day, wrapping
    assert np.all(starts[:, 0])
    # restart frequency of days 1.. within a 5-sigma binomial bound of q
    n = starts[:, 1:].size
    q = q32 / 2.0 ** 32
    assert abs(starts[:, 1:].sum() - n * q) <= 5 * math.sqrt(n * q * (1 - q)) + 1
    # a literal day-by-day walk of the same words gives the same stream
    for i in (0, 7, 299):
        assert list(theta[i]) == spa_ref.stationary_indices(T_, q32, 12345, int(gids[i]))


def test_iid_at_q_one():
    theta = spa_ref.index_stream(97, 1 << 32, 5, np.arange(4000, dtype=np.uint64))
    assert np.all(spa_ref.block_starts(97, 1 << 32, 5, np.arange(4000, dtype=np.uint64)))
    counts = np.bincount(theta.ravel(), minlength=97)                       # uniform over days
    e = theta.size / 97
    assert ((counts - e) ** 2 / e).sum() < 97 + 6 * math.sqrt(2 * 97)
    r = np.corrcoef(theta[:, :-1].ravel(), theta[:, 1:].ravel())[0, 1]      # consecutive draws independent
    assert abs(r) < 5 / math.sqrt(theta.size)


def test_omega2_at_q_one_is_gamma0_and_the_bootstrap_variance():
    rng = np.random.default_rng(1)
    x = rng.standard_t(5, (6, 120))
    mean, omega2 = spa_ref.moments_exact(x, 1.0)
    c = x - mean[:, None]
    g0 = np.zeros(6)
    for t in range(120):
        g0 = g0 + c[:, t] * c[:, t]
    assert np.array_equal(omega2, g0 / 120.0)
    theta = spa_ref.index_stream(120, 1 << 32, 9, np.arange(20000, dtype=np.uint64))
    m = spa_ref.boot_means_exact(x, theta)
    var = 120 * m.var(axis=1)
    # sampling error of a variance over 20 000 resamples: about sqrt(2 / 20000) = 1%
    np.testing.assert_allclose(var, omega2, rtol=0.05)


def test_omega2_matches_hansen_with_pow():
    rng = np.random.default_rng(2)
    x = rng.normal(0.1, 1.0, (5, 300))
    x[:, 1:] += 0.6 * x[:, :-1]                                             # serially dependent
    for block_len in (1.5, 10.0, 200.0):
        q = spa_q32(block_len) / 2.0 ** 32
        mean, omega2 = spa_ref.moments_exact(x, q)
        want = np.array([spa_ref.hansen_omega2(r, q) for r in x])
        np.testing.assert_allclose(omega2, want, rtol=1e-12)
        np.testing.assert_allclose(mean, x.mean(axis=1), rtol=1e-14)


def _noise(seed, n=N):
    return np.random.default_rng(seed).normal(0.0, 1.0, (n, T))


def test_exact_agrees_with_literal():
    x = _noise(5, 12)
    x[3] += 0.4
    x[7] = 0.0                                                              # never trades: excluded from SPA and StepM
    x[9] -= 0.3
    for block_len, alpha in ((5.0, 0.05), (1.0, 0.1), (40.0, 0.05)):
        ex = spa_ref.spa_exact(x, 400, block_len, alpha, 3)
        li = spa_ref.spa_literal(x, 400, block_len, alpha, 3)
        assert math.isclose(ex["reality_check"]["stat"], li["reality_check"]["stat"], rel_tol=1e-12)
        assert ex["reality_check"]["pvalue"] == li["reality_check"]["pvalue"]
        assert math.isclose(ex["spa"]["stat"], li["spa"]["stat"], rel_tol=1e-12)
        for k in ("pvalue_lower", "pvalue_consistent", "pvalue_upper"):
            assert ex["spa"][k] == li["spa"][k], (block_len, k)
        assert np.array_equal(ex["stepm"]["rejected"], li["stepm"]["rejected"])
        np.testing.assert_allclose(ex["stepm"]["critical_values"], li["stepm"]["critical_values"], rtol=1e-12)
        assert math.isnan(ex["t_stat"][7]) and not ex["stepm"]["rejected"][7]
        p = ex["spa"]
        assert p["pvalue_lower"] <= p["pvalue_consistent"] <= p["pvalue_upper"]


def test_strong_edge_is_found_and_named():
    x = _noise(0)
    edged = [5, 17, 31]
    x[edged] += 0.6
    r = spa_ref.spa_exact(x, B, 10.0, 0.05, 3)
    assert r["reality_check"]["pvalue"] < 0.01
    assert r["spa"]["pvalue_consistent"] < 0.01 and r["spa"]["pvalue_upper"] < 0.01
    assert list(np.flatnonzero(r["stepm"]["rejected"])) == edged
    assert r["best"]["index"] in edged


def test_pure_noise_is_not_significant():
    ps = []
    for seed in range(20):
        r = spa_ref.spa_exact(_noise(seed), B, 10.0, 0.05, seed)
        p = r["spa"]
        assert p["pvalue_lower"] <= p["pvalue_consistent"] <= p["pvalue_upper"]
        ps.append((r["reality_check"]["pvalue"], p["pvalue_consistent"], int(r["stepm"]["rejected"].sum())))
    rc, cons, rej = np.array(ps).T
    # under the null the p-values spread over (0, 1): at most two of 20 data sets below 0.05, none below 0.01
    assert (cons < 0.05).sum() <= 2 and cons.min() >= 0.01 and np.median(cons) > 0.2
    assert (rc < 0.05).sum() <= 2 and np.median(rc) > 0.2
    assert (rej > 0).sum() <= 2


def test_poor_trials_move_rc_not_spa_consistent():
    """Hansen's point: the Reality Check centres every trial at zero, so adding trials that are plainly worse than the
    benchmark raises its p-value; SPA-consistent recentres those trials at their own negative means and barely moves.
    On this data the exact restatement gives RC 0.312 -> 0.761, SPA-consistent 0.561 -> 0.561 and SPA-upper
    0.561 -> 0.959; the thresholds below leave room for a change of seed."""
    x = _noise(0)
    bad = np.vstack([x, np.random.default_rng(99).normal(-1.0, 1.0, (200, T))])
    a = spa_ref.spa_exact(x, B, 10.0, 0.05, 0)
    b = spa_ref.spa_exact(bad, B, 10.0, 0.05, 0)
    assert a["reality_check"]["stat"] == b["reality_check"]["stat"] and a["spa"]["stat"] == b["spa"]["stat"]
    assert b["reality_check"]["pvalue"] >= a["reality_check"]["pvalue"] + 0.3
    assert abs(b["spa"]["pvalue_consistent"] - a["spa"]["pvalue_consistent"]) <= 0.02
    assert b["spa"]["pvalue_upper"] > b["spa"]["pvalue_consistent"]
