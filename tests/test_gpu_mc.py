"""GPU Monte-Carlo kernels vs the CPU Philox oracle and the reference's statistics."""
import json

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine(native_lib):
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    from ai_crypto_trader_b200.monte_carlo import PathEngine
    return PathEngine()


@pytest.mark.parametrize("n_paths,steps", [(1, 1), (7, 3), (1000, 29), (4096, 250), (333, 1001)] +
                         [(n, s) for n in (255, 256, 257) for s in (0, 2, 4, 5, 8)])
def test_gbm_matches_philox_oracle(engine, n_paths, steps):
    from oracle import mc_ref
    mu, sigma, dt, s0, seed = 0.126, 0.3175, 1 / 252, 100.0, 2024
    f, d, _ = engine.gbm(s0, mu, sigma, dt, n_paths, steps, seed)
    fo, do, _ = mc_ref.gbm_paths(s0, mu, sigma, dt, n_paths, steps, seed)
    # same Philox bits; normals go through logf/sincospif on the GPU and libm on the CPU (ulp-level)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=3e-5)
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=2e-4, atol=2e-6)


def test_gbm_sharding_invariance_and_path_store(engine):
    s0, mu, sigma, dt, seed, n, steps = 50.0, 0.05, 0.4, 1 / 252, 99, 2000, 64
    f, d, paths = engine.gbm(s0, mu, sigma, dt, n, steps, seed, store_paths=True)
    fa, da, _ = engine.gbm(s0, mu, sigma, dt, 800, steps, seed, path_offset=0)
    fb, db, _ = engine.gbm(s0, mu, sigma, dt, 1200, steps, seed, path_offset=800)
    f, d, paths = f.cpu().numpy(), d.cpu().numpy(), paths.cpu().numpy()
    assert np.array_equal(np.concatenate([fa.cpu().numpy(), fb.cpu().numpy()]), f)   # bit-identical under sharding
    assert np.array_equal(np.concatenate([da.cpu().numpy(), db.cpu().numpy()]), d)
    assert paths.shape == (steps + 1, n) and np.all(paths[0] == np.float32(s0))
    np.testing.assert_allclose(paths[-1], f, rtol=2e-6)
    runmax = np.maximum.accumulate(paths.astype(np.float64), axis=0)
    np.testing.assert_allclose(((runmax - paths) / runmax).max(axis=0), d, rtol=1e-4, atol=2e-6)


@pytest.mark.parametrize("log_returns,block_len", [(True, 1), (False, 1), (True, 5)])
def test_bootstrap_matches_oracle(engine, log_returns, block_len):
    from oracle import mc_ref
    rng = np.random.default_rng(3)
    ret = rng.normal(5e-4, 0.02, 60).astype(np.float32)
    f, d, _ = engine.bootstrap(ret, log_returns, 100.0, 3000, 45, 77, block_len=block_len)
    fo, do, _ = mc_ref.bootstrap_paths(ret, log_returns, 100.0, 3000, 45, 77, block_len=block_len)
    np.testing.assert_allclose(f.cpu().numpy(), fo, rtol=(1e-6 if log_returns else 3e-6))
    np.testing.assert_allclose(d.cpu().numpy(), do, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("n", [1, 2, 33, 1000, 1_000_003])
def test_select_is_exact(engine, n):
    import torch
    rng = np.random.default_rng(n)
    x = (rng.lognormal(0, 0.3, n) * 100).astype(np.float32)
    if n > 10:
        x[::7] = x[3]          # duplicates
        x[1::11] *= -1         # negatives
    xs = np.sort(x)
    ranks = sorted({0, n - 1, n // 2, (n - 1) // 2, n // 20, (n * 99) // 100, min(n - 1, 5)})
    got = engine.select(torch.from_numpy(x).cuda(), ranks)
    assert np.array_equal(got.astype(np.float32), xs[ranks])


def test_risk_statistics_match_reference_formulas(engine):
    from ai_crypto_trader_b200.monte_carlo import risk_statistics
    from oracle import mc_ref
    f, d, _ = engine.gbm(100.0, 0.1, 0.35, 1 / 252, 200_001, 29, 5)
    st = risk_statistics(engine, f, d, 100.0, 0.95)
    want = mc_ref.risk_statistics(f.cpu().numpy(), d.cpu().numpy(), 100.0, 0.95)
    got_pct = [st["percentile_values"][i] for i in range(9)]
    assert got_pct == pytest.approx([want["percentiles"][p]["price"] for p in ("1", "5", "10", "25", "50", "75", "90", "95", "99")], rel=1e-12)
    assert abs(st["var"]) == pytest.approx(want["risk_metrics"]["var"], rel=1e-12)
    assert abs(st["cvar"]) == pytest.approx(want["risk_metrics"]["cvar"], rel=1e-10)
    assert st["prob_profit"] == pytest.approx(want["risk_metrics"]["prob_profit"], rel=1e-12)
    assert st["expected_price"] == pytest.approx(want["expected"]["price"], rel=1e-10)
    assert st["mdd_mean"] == pytest.approx(want["risk_metrics"]["max_drawdown"]["mean"], rel=1e-10)
    assert st["mdd_median"] == pytest.approx(want["risk_metrics"]["max_drawdown"]["median"], rel=1e-12)
    assert st["mdd_max"] == pytest.approx(want["risk_metrics"]["max_drawdown"]["max"], rel=1e-12)


def test_service_schema_and_statistical_agreement_with_reference(native_lib):
    """MonteCarloService drop-in: same result schema as the reference run, same law."""
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService
    meta = json.loads((GOLDEN / "mc_reference.json").read_text())
    arrays = np.load(GOLDEN / "mc_reference.npz")
    for case in meta["cases"]:
        ref = case["result"]
        svc = MonteCarloService(seed=123)
        svc.mc_params.update(simulation_method=case["method"], num_simulations=200_000, time_horizon_days=case["days"])
        svc.set_returns("SYNUSDC", arrays["returns"])
        res = svc.run_monte_carlo_simulation("SYNUSDC", 100.0, scenario=case["scenario"])
        assert set(res.keys()) == set(ref.keys()) | {"paths", "timestamp"}
        assert res["mu"] == pytest.approx(ref["mu"], rel=1e-14) and res["sigma"] == pytest.approx(ref["sigma"], rel=1e-14)
        assert res["percentiles"].keys() == ref["percentiles"].keys()
        assert res["risk_metrics"].keys() == ref["risk_metrics"].keys()
        # the reference run has n = 120..400 paths: compare within its Monte-Carlo error
        n_ref = case["n"]
        sd_pct = np.std((arrays[f"paths_{case['key']}"][-1] / 100.0 - 1) * 100)
        assert res["expected"]["pct_change"] == pytest.approx(ref["expected"]["pct_change"], abs=4 * sd_pct / np.sqrt(n_ref))
        assert res["risk_metrics"]["var"] == pytest.approx(ref["risk_metrics"]["var"], rel=0.25)
        assert res["risk_metrics"]["max_drawdown"]["mean"] == pytest.approx(ref["risk_metrics"]["max_drawdown"]["mean"], rel=0.15)
    # error convention: unknown symbol -> {} (monte_carlo_service.py:232-233)
    assert MonteCarloService().run_monte_carlo_simulation("NOPE", 1.0) == {}


def test_portfolio_stats_match_reference(native_lib):
    from ai_crypto_trader_b200.monte_carlo import MonteCarloService
    meta = json.loads((GOLDEN / "mc_reference.json").read_text())["portfolio"]
    svc = MonteCarloService()
    got = svc._calculate_portfolio_stats(meta["holdings"], meta["simulations"])
    assert got == meta["stats"]
