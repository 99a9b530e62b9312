"""Host side of the joint (portfolio) Monte-Carlo: the float64 restatement agrees with the single-asset one, the factor
policy, which holdings are simulated, and the {} error convention.  No GPU needed."""
import numpy as np
import pandas as pd
import pytest

import mc_joint_ref
from oracle import mc_ref


@pytest.mark.parametrize("steps", [0, 1, 7, 29])
def test_one_asset_joint_gbm_equals_gbm_paths(steps):
    mu, sigma, dt, s0, seed = 0.126, 0.3175, 1 / 252, 100.0, 2024
    f, d, af = mc_joint_ref.joint_gbm_paths([s0], [1.0], [mu], [sigma], dt, [[1.0]], 257, steps, seed, path_offset=9)
    fo, do, _ = mc_ref.gbm_paths(s0, mu, sigma, dt, 257, steps, seed, path_offset=9)
    assert np.array_equal(f, fo) and np.array_equal(af[0], fo)
    np.testing.assert_allclose(d, do, rtol=1e-12, atol=1e-15)


def test_joint_gbm_factor_zero_is_the_single_asset_stream():
    rng = np.random.default_rng(1)
    A = rng.normal(size=(3, 3))
    c = A @ A.T
    c = c / np.sqrt(np.outer(np.diag(c), np.diag(c)))
    L = np.linalg.cholesky(c)
    L[0, 0] = 1.0
    _, _, af = mc_joint_ref.joint_gbm_paths([50.0, 2.0, 7.0], [1, 1, 1], [0.1, -0.2, 0.3], [0.4, 0.5, 0.6], 1 / 252, L,
                                            100, 13, 77)
    fo, _, _ = mc_ref.gbm_paths(50.0, 0.1, 0.4, 1 / 252, 100, 13, 77)
    assert np.array_equal(af[0], fo)


@pytest.mark.parametrize("log_returns,block_len", [(True, 1), (False, 1), (True, 5), (False, 5)])
def test_joint_bootstrap_columns_equal_bootstrap_paths(log_returns, block_len):
    rng = np.random.default_rng(3)
    table = rng.normal(5e-4, 0.02, (60, 3)).astype(np.float32)
    s0 = [100.0, 3.0, 0.5]
    _, _, af, _ = mc_joint_ref.joint_bootstrap_paths(table, log_returns, s0, [1, 2, 3], 500, 45, 77, block_len=block_len)
    for i in range(3):
        fo, _, _ = mc_ref.bootstrap_paths(table[:, i], log_returns, s0[i], 500, 45, 77, block_len=block_len)
        assert np.array_equal(af[i], fo), i


def test_joint_bootstrap_draws_whole_rows():
    rng = np.random.default_rng(4)
    table = rng.normal(0, 0.03, (37, 4)).astype(np.float32)
    s0 = np.array([10.0, 20.0, 30.0, 40.0])
    _, _, af, days = mc_joint_ref.joint_bootstrap_paths(table, True, s0, [1, 1, 1, 1], 2000, 1, 5)
    # one step: every asset's log return is the same day's entry of its column
    r = np.log(af.astype(np.float64) / s0[:, None]).T                      # [n][S]
    row = np.abs(r[:, None, :] - table[None, :, :]).max(axis=2).argmin(axis=1)
    np.testing.assert_allclose(r, table[row], atol=1e-6)
    assert np.array_equal(row, days[0])
    assert len(np.unique(row)) > 30                                          # the stream covers the table


def test_joint_walk_drawdown_is_the_portfolio_rule():
    inc = np.array([[[0.1], [-0.3], [0.2]], [[-0.1], [0.2], [0.0]]])         # two assets, three steps, one path
    f, d, af = mc_joint_ref.joint_walk(inc, [1.0, 2.0], [3.0, 0.5])
    V = 3.0 * np.exp(np.concatenate([[0], np.cumsum(inc[0, :, 0])])) + 1.0 * np.exp(np.concatenate([[0], np.cumsum(inc[1, :, 0])]))
    runmax = np.maximum.accumulate(V)
    assert f[0] == np.float32(V[-1]) and d[0] == np.float32(((runmax - V) / runmax).max())


def test_joint_factor_policy():
    from ai_crypto_trader_b200.monte_carlo import joint_factor
    good = np.array([[1.0, 0.3, -0.2], [0.3, 1.0, 0.1], [-0.2, 0.1, 1.0]])
    c, L, fb = joint_factor(good * (1 + 1e-12))                     # diagonal is reset to exactly 1
    assert not fb and L[0, 0] == 1.0 and np.allclose(L @ L.T, good, atol=1e-11) and np.all(np.diag(c) == 1.0)
    nan = good.copy()
    nan[0, 2] = nan[2, 0] = np.nan
    for bad in (nan, np.array([[1.0, 0.9, -0.9], [0.9, 1.0, 0.9], [-0.9, 0.9, 1.0]]), np.ones((3, 3))):
        c, L, fb = joint_factor(bad)
        assert fb and np.array_equal(c, np.eye(3)) and np.array_equal(L, np.eye(3))


def _holdings():
    return {"total_value": 20000.0, "assets": {
        "AAA": {"value_usdc": 6000.0, "current_price": 10.0},
        "USDC": {"value_usdc": 5000.0, "current_price": 1.0},
        "BBB": {"value_usdc": 4000.0, "current_price": 2.5},
        "CCC": {"value_usdc": 3000.0, "current_price": 0},          # no price: skipped
        "DDD": {"value_usdc": 2000.0, "current_price": 4.0},        # no return sample: skipped
    }}


def test_joint_assets_come_from_holdings():
    from ai_crypto_trader_b200.monte_carlo import joint_assets
    rng = np.random.default_rng(5)
    data = {s: pd.DataFrame({"returns": rng.normal(0, 0.02, 30)}) for s in ("AAAUSDC", "BBBUSDC", "CCCUSDC")}
    used = joint_assets(_holdings(), data)
    assert [u[0] for u in used] == ["AAA", "BBB"]
    assert [u[1] for u in used] == [10.0, 2.5] and [u[2] for u in used] == [600.0, 1600.0]
    assert [u[3] for u in used] == [6000.0, 4000.0]


def test_joint_service_error_paths_return_empty():
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService
    svc = MonteCarloService()
    assert svc.run_joint_portfolio_monte_carlo(None) == {}
    assert svc.run_joint_portfolio_monte_carlo({"assets": {}}) == {}
    assert svc.run_joint_portfolio_monte_carlo({"total_value": 1.0, "assets": {"USDC": {"value_usdc": 1.0}}}) == {}
    assert svc.run_joint_portfolio_monte_carlo(_holdings()) == {}                     # no return samples at all
    svc.set_returns("AAAUSDC", np.random.default_rng(6).normal(0, 0.02, 30))
    svc.mc_params["simulation_method"] = "nope"
    # without a device the engine raises, with one the method is unknown: logged either way, not raised
    assert svc.run_joint_portfolio_monte_carlo(_holdings()) == {}
