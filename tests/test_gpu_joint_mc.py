"""GPU joint (portfolio) Monte-Carlo kernels: bit parity with the single-asset kernels, the float64 restatement,
comonotone and correlation properties, sharding, and the service's joint portfolio result."""
import json

import numpy as np
import pytest

import mc_joint_ref
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

DT = 1 / 252


@pytest.fixture(scope="module")
def engine(native_lib):
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    from ai_crypto_trader_b200.monte_carlo import PathEngine
    return PathEngine()


def _params(S, seed):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(S, S + 2))
    c = A @ A.T
    c = c / np.sqrt(np.outer(np.diag(c), np.diag(c)))
    L = np.linalg.cholesky(c)
    L[0, 0] = 1.0
    s0 = rng.uniform(0.5, 200.0, S)
    qty = rng.uniform(0.1, 10.0, S)
    mu = rng.uniform(-0.3, 0.4, S)
    sigma = rng.uniform(0.1, 0.9, S)
    return s0, qty, mu, sigma, L.astype(np.float32)


@pytest.mark.parametrize("S", [1, 3, 8, 16, 32])
def test_asset0_bit_equals_single_asset_gbm(engine, S):
    s0, qty, mu, sigma, L = _params(S, S)
    f, _, af = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, 3000, 61, 2024, path_offset=5, asset_finals=True)
    fo, _, _ = engine.gbm(s0[0], mu[0], sigma[0], DT, 3000, 61, 2024, path_offset=5)
    assert np.array_equal(af[0].cpu().numpy(), fo.cpu().numpy())


@pytest.mark.parametrize("log_returns,block_len", [(True, 1), (False, 1), (True, 5), (False, 5)])
def test_bootstrap_assets_bit_equal_single_asset_bootstrap(engine, log_returns, block_len):
    rng = np.random.default_rng(3)
    S = 5
    table = rng.normal(5e-4, 0.02, (60, S)).astype(np.float32)
    s0 = rng.uniform(1, 100, S)
    _, _, af = engine.portfolio_bootstrap(table, log_returns, s0, np.ones(S), 3000, 45, 77, block_len=block_len,
                                          asset_finals=True)
    for i in range(S):
        fo, _, _ = engine.bootstrap(table[:, i], log_returns, s0[i], 3000, 45, 77, block_len=block_len)
        assert np.array_equal(af[i].cpu().numpy(), fo.cpu().numpy()), i


@pytest.mark.parametrize("n_paths", [1, 129])
@pytest.mark.parametrize("steps", [0, 1, 3, 29, 1001])
@pytest.mark.parametrize("S", [1, 3, 4, 5, 8, 9, 17, 32])
def test_joint_gbm_matches_oracle(engine, S, steps, n_paths):
    s0, qty, mu, sigma, L = _params(S, 100 + S)
    f, d, af = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, n_paths, steps, 99, path_offset=3, asset_finals=True)
    fo, do, afo = mc_joint_ref.joint_gbm_paths(s0, qty, mu, sigma, DT, L, n_paths, steps, 99, path_offset=3)
    # same Philox bits; normals through the MUFU log / sin / cos on the GPU and libm on the CPU (as test_gpu_mc.py)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-5)
    np.testing.assert_allclose(af.cpu().numpy(), afo, rtol=3e-5)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize("log_returns,block_len", [(True, 1), (False, 5)])
@pytest.mark.parametrize("S", [1, 3, 32])
def test_joint_bootstrap_matches_oracle(engine, S, log_returns, block_len):
    rng = np.random.default_rng(S)
    table = rng.normal(5e-4, 0.02, (300, S)).astype(np.float32)
    s0, qty = rng.uniform(1, 100, S), rng.uniform(0.1, 5, S)
    f, d, _ = engine.portfolio_bootstrap(table, log_returns, s0, qty, 777, 250, 11, block_len=block_len)
    fo, do, _, _ = mc_joint_ref.joint_bootstrap_paths(table, log_returns, s0, qty, 777, 250, 11, block_len=block_len)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-6)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)


def test_comonotone_var_percentile_points_add(engine):
    from functools import partial
    from ai_crypto_trader_b200.monte_carlo import _lerp, percentile_points

    def var_pct(x, initial):                        # risk_statistics' VaR: the 5th percentile of the percentage change
        [(lo, hi, g)] = percentile_points(partial(engine.select, x), int(x.numel()), [100 * (1 - 0.95)])
        return _lerp((lo / initial - 1) * 100, (hi / initial - 1) * 100, g)

    S = 4
    s0 = np.array([100.0, 20.0, 3.0, 0.7])
    qty = np.array([1.0, 4.0, 10.0, 50.0])
    mu = np.array([0.02, 0.05, -0.1, 0.0])
    sigma = np.array([0.3, 0.5, 0.7, 0.9])
    L = np.zeros((S, S), dtype=np.float32)
    L[:, 0] = 1.0                                   # every asset driven by the same normal
    f, _, af = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, 200_001, 29, 5, asset_finals=True)
    v0 = float(np.sum(qty * s0))
    joint = var_pct(f, v0)
    per_asset = [var_pct(af[i].contiguous(), s0[i]) for i in range(S)]
    assert all(v < 0 for v in per_asset)
    w = qty * s0 / v0
    assert joint == pytest.approx(float(np.dot(w, per_asset)), rel=1e-5)


def test_sample_correlation_hits_target(engine):
    target = np.array([[1.0, 0.6, -0.4, 0.2], [0.6, 1.0, -0.1, 0.3], [-0.4, -0.1, 1.0, 0.0], [0.2, 0.3, 0.0, 1.0]])
    L = np.linalg.cholesky(target).astype(np.float32)
    s0 = np.array([10.0, 20.0, 30.0, 40.0])
    _, _, af = engine.portfolio_gbm(s0, np.ones(4), [0.1, 0.0, -0.1, 0.2], [0.3, 0.6, 0.9, 0.2], DT, L, 1 << 20, 1, 8,
                                    asset_finals=True)
    x = np.log(af.cpu().numpy().astype(np.float64) / s0[:, None])
    assert np.abs(np.corrcoef(x) - target).max() < 0.01


def test_shards_concatenate_to_one_run(engine):
    import torch
    s0, qty, mu, sigma, L = _params(6, 7)
    one = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, 3000, 40, 31, asset_finals=True)
    a = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, 1100, 40, 31, path_offset=0, asset_finals=True)
    b = engine.portfolio_gbm(s0, qty, mu, sigma, DT, L, 1900, 40, 31, path_offset=1100, asset_finals=True)
    for whole, x, y in zip(one, a, b):
        assert torch.equal(torch.cat([x, y], dim=-1), whole)
    table = np.random.default_rng(2).normal(0, 0.02, (50, 6)).astype(np.float32)
    one = engine.portfolio_bootstrap(table, False, s0, qty, 3000, 40, 31, block_len=3, asset_finals=True)
    a = engine.portfolio_bootstrap(table, False, s0, qty, 1100, 40, 31, path_offset=0, block_len=3, asset_finals=True)
    b = engine.portfolio_bootstrap(table, False, s0, qty, 1900, 40, 31, path_offset=1100, block_len=3, asset_finals=True)
    for whole, x, y in zip(one, a, b):
        assert torch.equal(torch.cat([x, y], dim=-1), whole)


def test_zero_paths(engine):
    f, d, af = engine.portfolio_gbm([1.0, 2.0], [1, 1], [0, 0], [0.1, 0.1], DT, np.eye(2), 0, 10, 1, asset_finals=True)
    assert f.numel() == 0 and d.numel() == 0 and tuple(af.shape) == (2, 0)


def test_one_asset_service_equals_single_asset_statistics(engine):
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService, risk_statistics
    returns = np.random.default_rng(9).normal(8e-4, 0.025, 120)
    svc = MonteCarloService(seed=321)
    svc.mc_params.update(num_simulations=100_000, time_horizon_days=30)
    svc.set_returns("AAAUSDC", returns)
    holdings = {"total_value": 3000.0, "assets": {"AAA": {"value_usdc": 2500.0, "current_price": 10.0},
                                                  "USDC": {"value_usdc": 500.0, "current_price": 1.0}}}
    res = svc.run_joint_portfolio_monte_carlo(holdings, scenarios=["base"])
    assert res and res["assets"] == ["AAA"] and res["correlation_fallback"] is False
    assert res["quantities"] == {"AAA": 250.0} and res["weights"] == {"AAA": 1.0}
    got = res["scenarios"]["base"]
    mu, sigma = got["mu"]["AAA"], got["sigma"]["AAA"]
    f, d, _ = engine.gbm(10.0, mu, sigma, DT, 100_000, 29, 321)
    want = risk_statistics(engine, f, d, 10.0, 0.95)
    assert got["risk_metrics"]["var"] == pytest.approx(abs(want["var"]), rel=1e-5)
    assert got["risk_metrics"]["cvar"] == pytest.approx(abs(want["cvar"]), rel=1e-5)
    assert got["risk_metrics"]["prob_profit"] == pytest.approx(want["prob_profit"], abs=2e-5)
    for p, v in zip(("1", "5", "10", "25", "50", "75", "90", "95", "99"), want["percentile_values"]):
        assert got["percentiles"][p]["price"] == pytest.approx(250.0 * v, rel=1e-6)
    md = got["risk_metrics"]["max_drawdown"]
    assert md["mean"] == pytest.approx(want["mdd_mean"], abs=1e-6)
    assert md["median"] == pytest.approx(want["mdd_median"], abs=1e-6)
    assert md["max"] == pytest.approx(want["mdd_max"], abs=1e-6)
    assert got["undiversified_var"] == pytest.approx(got["risk_metrics"]["var"], rel=1e-5)


@pytest.mark.parametrize("method", ["geometric_brownian_motion", "historical"])
def test_fixture_portfolio_schema_and_diversification(native_lib, method):
    import pandas as pd
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService
    holdings = json.loads((GOLDEN / "mc_reference.json").read_text())["portfolio"]["holdings"]
    rng = np.random.default_rng(12)
    common = rng.normal(0, 0.015, 200)
    a = pd.Series(common + rng.normal(6e-4, 0.02, 200))
    b = pd.Series(0.5 * common + rng.normal(3e-4, 0.03, 200))[5:]          # a shorter series: aligned on the index
    svc = MonteCarloService(seed=7)
    svc.mc_params.update(num_simulations=200_000, simulation_method=method)
    svc.historical_data = {"AAAUSDC": pd.DataFrame({"returns": a}), "BBBUSDC": pd.DataFrame({"returns": b})}
    res = svc.run_joint_portfolio_monte_carlo(holdings)
    assert res["assets"] == ["AAA", "BBB"] and res["weights"] == pytest.approx({"AAA": 0.6, "BBB": 0.4})
    assert res["correlation_fallback"] is False
    want_corr = pd.DataFrame({"AAA": a, "BBB": b}).corr().to_numpy()
    assert res["correlation"]["AAA"]["BBB"] == pytest.approx(want_corr[0, 1], abs=1e-6)
    assert set(res["scenarios"]) == set(svc.mc_params["scenarios"])
    ref_keys = set(svc._calculate_portfolio_stats(holdings, {}).keys()) | {"scenario_stats"}
    assert set(res["portfolio_stats"].keys()) == ref_keys
    ps = res["portfolio_stats"]
    assert ps["var_loss_value"] == pytest.approx(holdings["total_value"] * ps["var"] / 100)
    for name, r in res["scenarios"].items():
        assert set(r["risk_metrics"]) == {"var", "cvar", "prob_profit", "prob_loss", "max_drawdown"}
        assert len(r["percentiles"]) == 9
        assert r["diversification_benefit"] == pytest.approx(r["undiversified_var"] - r["risk_metrics"]["var"])
        if method == "geometric_brownian_motion":
            assert r["diversification_benefit"] >= 0, name
