"""Monte-Carlo risk projection on the GPU behind the reference's MonteCarloService surface.

Reference: services/monte_carlo_service.py (class MonteCarloService).  Same method
names, argument meaning, result schema (:339-374) and error convention (log and
return {} -- never raise, :392-394).  Differences, all deliberate (SURVEY.md 5, 8-a16):
  * no Binance client / Redis / matplotlib: return samples are supplied by the caller
    (`historical_data[symbol]` DataFrame with a 'returns' column, as the reference
    caches them at :223-227, or `set_returns`); holdings are passed in;
  * the constructor never rewrites config.json (the reference does, :98-101);
  * path generation, per-path drawdown, order statistics and moments run in the
    sm_90a kernels of csrc/montecarlo.cu (Philox4x32-10 instead of NumPy's MT19937:
    same distribution, different stream; `seed` makes runs reproducible);
  * `block_len` > 1 turns the 'historical' method into a block bootstrap (north-star
    extension; 1 reproduces the reference's iid resampling).
"""
from __future__ import annotations

import ctypes as C
import json
import logging
import math
from datetime import datetime
from functools import partial
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib

logger = logging.getLogger("b200bt.monte_carlo")

DEFAULT_MC_PARAMS = {  # monte_carlo_service.py:78-95
    "num_simulations": 1000,
    "time_horizon_days": 30,
    "confidence_level": 0.95,
    "lookback_days": 60,
    "return_method": "log",
    "simulation_method": "geometric_brownian_motion",
    "plot_chart": False,
    "generate_reports": True,
    "report_frequency": "daily",
    "scenarios": {
        "base": {},
        "bull": {"drift_factor": 1.5, "volatility_factor": 0.8},
        "bear": {"drift_factor": 0.5, "volatility_factor": 1.2},
        "volatile": {"drift_factor": 1.0, "volatility_factor": 2.0},
        "crab": {"drift_factor": 0.2, "volatility_factor": 0.5},
    },
}

PERCENTILES = [1, 5, 10, 25, 50, 75, 90, 95, 99]  # :308


def _lerp(a: float, b: float, t: float) -> float:
    """numpy.percentile(method='linear') interpolation, including its t >= 0.5 branch."""
    d = b - a
    return b - d * (1.0 - t) if t >= 0.5 else a + d * t


def _virtual_index(n: int, q_percent: float):
    """(floor index, next index, gamma) exactly as numpy's linear method derives them."""
    h = (n - 1) * np.true_divide(q_percent, 100)
    lo = int(math.floor(h))
    lo = min(max(lo, 0), n - 1)
    hi = min(lo + 1, n - 1)
    return lo, hi, float(h - math.floor(h))


def percentile_points(select, n: int, percentiles):
    """[(x_lo, x_hi, g)] for each percentile: numpy's linear percentile of n values is _lerp(x_lo, x_hi, g) of two exact
    order statistics.  `select(ranks)` returns the order statistics at ascending 0-based ranks; it is called once, over
    the union of the ranks every percentile needs."""
    idx = [_virtual_index(n, q) for q in percentiles]
    ranks = sorted({i for lo, hi, _ in idx for i in (lo, hi)})
    vals = dict(zip(ranks, select(ranks)))
    return [(vals[lo], vals[hi], g) for lo, hi, g in idx]


def _f64(x) -> np.ndarray:
    return np.atleast_1d(np.asarray(x, dtype=np.float64))


def _c_doubles(x: np.ndarray):
    return (C.c_double * len(x))(*x.tolist())


def joint_factor(corr: np.ndarray):
    """(correlation used, its float64 Cholesky factor, fallback taken) for a joint simulation.

    A matrix with a NaN entry (an asset without variance or without a common observation) or an eigenvalue <= 0 is
    replaced by the identity -- the policy of portfolio_risk_service.py:377-381 -- and the fallback is reported.  The
    diagonal is set to exactly 1, so that L_00 = 1 and asset 0 follows the single-asset generator's path."""
    c = np.array(corr, dtype=np.float64)
    S = c.shape[0]
    fallback = not np.all(np.isfinite(c))
    if not fallback:
        c = 0.5 * (c + c.T)
        np.fill_diagonal(c, 1.0)
        fallback = not np.all(np.linalg.eigvalsh(c) > 0)
    if not fallback:
        try:
            return c, np.linalg.cholesky(c), False
        except np.linalg.LinAlgError:
            fallback = True
    logger.warning("Correlation matrix is not positive definite, using identity matrix")
    return np.eye(S), np.eye(S), True


def joint_assets(holdings: Dict, historical_data: Dict):
    """The holdings a joint simulation can use: non-USDC assets with a current price and a return sample
    (historical_data[f"{asset}USDC"]), in holdings order.  -> [(asset, current_price, quantity, value_usdc, returns)]
    with quantity = value_usdc / current_price; the others are skipped with a warning (as :520-527 does)."""
    out = []
    for asset, h in holdings["assets"].items():
        if asset == "USDC":
            continue
        price = h.get("current_price", 0)
        if price == 0:
            logger.warning("No current price available for %s, skipping simulation", asset)
            continue
        df = historical_data.get(f"{asset}USDC")
        returns = df["returns"].dropna() if df is not None and not df.empty else None
        if returns is None or len(returns) < 2:
            logger.warning("No historical data available for %sUSDC, skipping simulation", asset)
            continue
        value = h.get("value_usdc", 0)
        out.append((asset, float(price), value / price, float(value), returns))
    return out


class PathEngine:
    """Device-side Monte-Carlo primitives (one instance per GPU)."""

    def __init__(self, device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("Monte-Carlo engine needs a CUDA device (sm_90); there is no CPU path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._ws = None

    def _generate(self, fn: str, args, n_paths, steps, seed, path_offset, rows=None):
        """Run the path generator `fn`(*args, n_paths, steps, seed, path_offset, finals, maxdd, block, stream) into new
        outputs: finals [n], maxdd [n] and, when `rows` is given, a [rows][n] block (stored paths or asset finals).
        A rank without paths (more ranks than paths) gets empty outputs and no launch."""
        out = lambda *shape: torch.empty(shape, dtype=torch.float32, device=self.device)
        finals, maxdd = out(n_paths), out(n_paths)
        block = out(rows, n_paths) if rows is not None else None
        if n_paths > 0:
            with torch.cuda.device(self.device):
                _lib.call(fn, *args, int(n_paths), int(steps), int(seed) & (2**64 - 1), int(path_offset),
                          finals.data_ptr(), maxdd.data_ptr(), _lib.ptr(block), _lib.current_stream())
        return finals, maxdd, block

    def gbm(self, s0, mu, sigma, dt, n_paths, steps, seed, path_offset=0, store_paths=False):
        return self._generate("b200bt_mc_gbm", (float(s0), float(mu), float(sigma), float(dt)), n_paths, steps, seed,
                              path_offset, steps + 1 if store_paths else None)

    def bootstrap(self, returns: np.ndarray, log_returns: bool, s0, n_paths, steps, seed, path_offset=0,
                  block_len=1, store_paths=False):
        r = torch.from_numpy(np.ascontiguousarray(returns, dtype=np.float32)).to(self.device)
        return self._generate("b200bt_mc_bootstrap", (r.data_ptr(), int(r.numel()), int(block_len),
                                                      1 if log_returns else 0, float(s0)),
                              n_paths, steps, seed, path_offset, steps + 1 if store_paths else None)

    def portfolio_gbm(self, s0, qty, mu, sigma, dt, chol, n_paths, steps, seed, path_offset=0, asset_finals=False):
        """Joint GBM of S assets: per-asset s0 / qty / mu / sigma (length S), `chol` the [S][S] lower Cholesky factor
        of their correlation.  -> (portfolio finals V_T [n], portfolio max drawdown [n], asset finals [S][n] or None)."""
        s0, qty = _f64(s0), _f64(qty)
        mu, sigma = _f64(mu), _f64(sigma)
        S = len(s0)
        drift = (mu - 0.5 * sigma * sigma) * dt     # as b200bt_mc_gbm derives them (:273)
        vol = sigma * np.sqrt(dt)
        L = np.ascontiguousarray(chol, dtype=np.float32).reshape(S, S)
        return self._generate("b200bt_mc_portfolio_gbm", (S, _c_doubles(s0), _c_doubles(qty), _c_doubles(drift),
                                                          _c_doubles(vol), (C.c_float * L.size)(*L.ravel().tolist())),
                              n_paths, steps, seed, path_offset, S if asset_finals else None)

    def portfolio_bootstrap(self, returns: np.ndarray, log_returns: bool, s0, qty, n_paths, steps, seed, path_offset=0,
                            block_len=1, asset_finals=False):
        """Joint bootstrap of whole days: `returns` [R][S], one row per day with a return for every asset."""
        s0, qty = _f64(s0), _f64(qty)
        S = len(s0)
        table = np.ascontiguousarray(returns, dtype=np.float32)
        if table.ndim != 2 or table.shape[1] != S:
            raise ValueError(f"return table of shape {table.shape} for {S} assets")
        r = torch.from_numpy(table).to(self.device)
        return self._generate("b200bt_mc_portfolio_bootstrap", (S, r.data_ptr(), int(table.shape[0]), int(block_len),
                                                                1 if log_returns else 0, _c_doubles(s0), _c_doubles(qty)),
                              n_paths, steps, seed, path_offset, S if asset_finals else None)

    def select(self, x: torch.Tensor, ranks) -> np.ndarray:
        """Exact order statistics x_(k) for ascending 0-based ranks (float32 values as float64)."""
        ranks = [int(k) for k in ranks]
        assert ranks == sorted(ranks) and len(ranks) <= 64
        dev = self.device
        need = int(_lib.load().b200bt_select_workspace_bytes(len(ranks)))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        rk = torch.tensor(ranks, dtype=torch.int64, device=dev)
        out = torch.empty(len(ranks), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.call("b200bt_select", x.data_ptr(), int(x.numel()), rk.data_ptr(), len(ranks), out.data_ptr(),
                      self._ws.data_ptr(), need, _lib.current_stream())
        return out.cpu().numpy().astype(np.float64)

    def moments(self, finals: torch.Tensor, maxdd: Optional[torch.Tensor], s0: float, var_threshold: float) -> np.ndarray:
        out = torch.empty(7, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("b200bt_mc_moments", finals.data_ptr(), _lib.ptr(maxdd), int(finals.numel()), float(s0),
                      float(var_threshold), out.data_ptr(), _lib.current_stream())
        return out.cpu().numpy()


def risk_statistics(engine: PathEngine, finals: torch.Tensor, maxdd: torch.Tensor, initial_price: float,
                    confidence: float, mdd_percentiles=()) -> Dict:
    """The statistics block of run_monte_carlo_simulation (:305-336) from device arrays, plus `mdd_p<q>`, the q-th
    percentile of the maximum drawdown, for each q in `mdd_percentiles`."""
    n = int(finals.numel())
    *points, (v_lo, v_hi, g) = percentile_points(partial(engine.select, finals), n,
                                                 PERCENTILES + [100 * (1 - confidence)])   # :308, :316
    pct = lambda v: (v / initial_price - 1) * 100                 # :312
    var = _lerp(pct(v_lo), pct(v_hi), g)                          # :317 on pct_changes (monotone in S_T)
    # the median is 50's order statistics: the middle one (g = 0, n odd) or the middle two (g = 0.5, n even)
    (d_lo, d_hi, d_g), *dd_points = percentile_points(partial(engine.select, maxdd), n, [50, *mdd_percentiles])
    m = engine.moments(finals, maxdd, initial_price, var)
    cvar = m[5] / m[6] if m[6] > 0 else float("nan")              # :320
    prob_profit = m[2] / n                                        # :323
    st = {
        "percentile_values": [_lerp(lo, hi, g) for lo, hi, g in points],
        "expected_price": m[0] / n, "expected_pct": m[1] / n,
        "var": var, "cvar": cvar, "prob_profit": prob_profit,
        "mdd_mean": m[3] / n, "mdd_median": float(np.mean([d_lo, d_hi] if d_g else [d_lo])), "mdd_max": float(m[4]),
    }
    for q, (lo, hi, g) in zip(mdd_percentiles, dd_points):
        st[f"mdd_p{q}"] = _lerp(lo, hi, g)
    return st


def statistics_blocks(st: Dict, initial: float, value_key: str) -> Dict:
    """The percentiles / expected / risk_metrics blocks of run_monte_carlo_simulation's result (:339-374) from
    risk_statistics' dict, the value under `value_key` ("price", or "equity" for a trade Monte-Carlo).  The drawdown
    block has `p95` when the statistics do."""
    drawdown = {"mean": float(st["mdd_mean"]), "median": float(st["mdd_median"])}
    if "mdd_p95" in st:
        drawdown["p95"] = float(st["mdd_p95"])
    drawdown["max"] = float(st["mdd_max"])
    return {
        "percentiles": {str(p): {value_key: float(v), "pct_change": float((v / initial - 1) * 100)}
                        for p, v in zip(PERCENTILES, st["percentile_values"])},
        "expected": {value_key: float(st["expected_price"]), "pct_change": float(st["expected_pct"])},
        "risk_metrics": {
            "var": float(abs(st["var"])), "cvar": float(abs(st["cvar"])),
            "prob_profit": float(st["prob_profit"]), "prob_loss": float(1 - st["prob_profit"]),
            "max_drawdown": drawdown,
        },
    }


def _world_rank():
    """(world size, rank) under torch.distributed, (1, 0) without it."""
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_world_size(), torch.distributed.get_rank()
    return 1, 0


class MonteCarloService:
    """Drop-in for services/monte_carlo_service.py:MonteCarloService (compute surface)."""

    def __init__(self, config: Optional[Dict] = None, config_path: Optional[str] = None, seed: int = 2024,
                 device: Optional[torch.device] = None, block_len: int = 1):
        if config is None and config_path is not None:
            with open(config_path, "r") as f:
                config = json.load(f)
        self.config = config or {}
        # the reference reads the TOP-LEVEL 'monte_carlo' key and falls back to in-code defaults (:75-95)
        self.mc_params = dict(self.config.get("monte_carlo", {})) or json.loads(json.dumps(DEFAULT_MC_PARAMS))
        self.historical_data: Dict = {}
        self.simulation_results: Dict = {}
        self.last_simulation_time: Dict = {}
        self.seed = int(seed)
        self.block_len = int(block_len)
        self._sim_counter = 0
        self._engine: Optional[PathEngine] = None
        self._device = device

    @property
    def engine(self) -> PathEngine:
        if self._engine is None:
            self._engine = PathEngine(self._device)
        return self._engine

    def set_returns(self, symbol: str, returns) -> None:
        """Install the historical return sample fetch_historical_prices would have produced (:186-189)."""
        import pandas as pd
        self.historical_data[symbol] = pd.DataFrame({"returns": np.asarray(returns, dtype=np.float64)})

    # -- the hot function ------------------------------------------------------
    def run_monte_carlo_simulation(self, symbol: str, initial_price: float, days: int = None,
                                   num_simulations: int = None, scenario: str = "base") -> Dict:
        try:
            if days is None:
                days = self.mc_params["time_horizon_days"]
            if num_simulations is None:
                num_simulations = self.mc_params["num_simulations"]
            if symbol not in self.historical_data:
                logger.error("No historical data available for %s", symbol)
                return {}
            df = self.historical_data[symbol]
            if df.empty:
                logger.error("No historical data available for %s", symbol)
                return {}
            returns = df["returns"].dropna()
            periods_per_year = 252
            mu = returns.mean() * periods_per_year                       # :243
            sigma = returns.std() * np.sqrt(periods_per_year)            # :244 (pandas ddof=1)
            drift_factor, volatility_factor = self._scenario_factors(scenario)
            mu = mu * drift_factor
            sigma = sigma * volatility_factor
            dt = 1 / periods_per_year
            method = self.mc_params["simulation_method"]
            store = bool(self.mc_params.get("store_all_paths", False))
            steps = int(days) - 1
            seed = self.seed + self._sim_counter
            self._sim_counter += 1
            eng = self.engine
            # under torch.distributed the paths are sharded over the ranks (Philox is keyed by the global path index:
            # the result does not depend on the number of GPUs) and gathered once for the statistics
            from .dist import gather_paths, shard_bounds
            world, rank = (1, 0) if store else _world_rank()
            lo, hi, _ = shard_bounds(int(num_simulations), world, rank)
            if method == "geometric_brownian_motion":
                finals, maxdd, paths = eng.gbm(initial_price, mu, sigma, dt, hi - lo, steps, seed, path_offset=lo,
                                               store_paths=store)
            elif method == "historical":
                finals, maxdd, paths = eng.bootstrap(returns.to_numpy(), self.mc_params["return_method"] == "log",
                                                     initial_price, hi - lo, steps, seed, path_offset=lo,
                                                     block_len=self.block_len, store_paths=store)
            else:
                logger.error("Unknown simulation method: %s", method)
                return {}
            if world > 1:
                finals, maxdd = gather_paths(finals, maxdd, int(num_simulations))
            st = risk_statistics(eng, finals, maxdd, initial_price, self.mc_params["confidence_level"])
            results = {
                "symbol": symbol, "initial_price": initial_price, "time_horizon_days": days,
                "num_simulations": num_simulations, "mu": mu, "sigma": sigma,
                "drift_factor": drift_factor, "volatility_factor": volatility_factor,
                "simulation_method": method, "scenario": scenario, "timestamp": datetime.now().isoformat(),
                **statistics_blocks(st, initial_price, "price"),
                "paths": paths.cpu().numpy().astype(np.float64).tolist() if store else None,
            }
            self.simulation_results[symbol] = results
            self.last_simulation_time[symbol] = datetime.now()
            if self.mc_params.get("plot_chart"):
                logger.info("plot_chart requested: charts are out of scope for the GPU engine, skipped")
            return results
        except Exception as e:  # reference convention: log, return {}
            logger.error("Error running Monte Carlo simulation for %s: %s", symbol, e, exc_info=True)
            return {}

    # -- portfolio layer (host arithmetic on a handful of numbers) -------------------
    async def run_portfolio_monte_carlo(self, holdings: Optional[Dict] = None) -> Dict:
        """:492-575 with the holdings passed in (the reference reads them from Redis)."""
        try:
            if not holdings or not holdings.get("assets"):
                return {}
            assets = [a for a in holdings["assets"].keys() if a != "USDC"]
            if not assets:
                return {}
            portfolio_simulations = {}
            for asset in assets:
                symbol = f"{asset}USDC"
                current_price = holdings["assets"][asset].get("current_price", 0)
                if current_price == 0:
                    continue
                for scenario in self.mc_params["scenarios"].keys():
                    key = f"{symbol}_{scenario}"
                    if (key in self.last_simulation_time
                            and (datetime.now() - self.last_simulation_time[key]).total_seconds() < 3600
                            and key in self.simulation_results):
                        portfolio_simulations[key] = self.simulation_results[key]
                        continue
                    results = self.run_monte_carlo_simulation(symbol, current_price, scenario=scenario)
                    if results:
                        portfolio_simulations[key] = results
                        self.simulation_results[key] = results
                        self.last_simulation_time[key] = datetime.now()
            stats = self._calculate_portfolio_stats(holdings, portfolio_simulations)
            return {"timestamp": datetime.now().isoformat(), "portfolio_value": holdings["total_value"],
                    "asset_simulations": portfolio_simulations, "portfolio_stats": stats}
        except Exception as e:
            logger.error("Error running portfolio Monte Carlo simulations: %s", e, exc_info=True)
            return {}

    def run_joint_portfolio_monte_carlo(self, holdings: Optional[Dict] = None, scenarios=None, days: int = None,
                                        num_simulations: int = None) -> Dict:
        """Simulate the holdings JOINTLY and read the risk off the distribution of the portfolio value.

        run_portfolio_monte_carlo simulates each asset on its own and _calculate_portfolio_stats adds up the weighted
        per-asset VaR / CVaR (:630-631 "ignores correlations"): the comonotone worst case, without diversification and
        without a portfolio drawdown.  Here the assets move together -- GBM with the assets' correlation (device
        b200bt_correlation on the return series aligned on their index, Cholesky factor on the host) or a bootstrap of
        whole days -- and the statistics of run_monte_carlo_simulation are taken on V_t = sum_i q_i P_i,t.
        Per scenario, `undiversified_var` is the weighted sum of the per-asset VaRs of the same run (what
        _calculate_portfolio_stats reports) and `diversification_benefit` is that minus the joint VaR.  `portfolio_stats`
        has the keys of _calculate_portfolio_stats, from the joint distribution.  Never raises: logs and returns {}."""
        try:
            if not holdings or not holdings.get("assets"):
                logger.debug("No holdings to analyze")
                return {}
            if days is None:
                days = self.mc_params["time_horizon_days"]
            if num_simulations is None:
                num_simulations = self.mc_params["num_simulations"]
            if scenarios is None:
                scenarios = list(self.mc_params["scenarios"].keys())
            used = joint_assets(holdings, self.historical_data)
            if not used:
                logger.warning("No assets with a price and historical data to simulate")
                return {}
            import pandas as pd
            from .dist import gather_path_rows, gather_paths, shard_bounds
            from .portfolio_risk import PortfolioRiskService, ReturnBank
            assets = [u[0] for u in used]
            s0 = np.array([u[1] for u in used])
            qty = np.array([u[2] for u in used])
            values = np.array([u[3] for u in used])
            v0 = sum(q * p for q, p in zip(qty.tolist(), s0.tolist()))    # V_0 as the kernel sums it
            if not values.sum() > 0:
                logger.warning("No non-USDC assets with value in portfolio")
                return {}
            weights = values / values.sum()
            frame = pd.DataFrame({u[0]: u[4] for u in used})             # aligned on the index (portfolio_risk_service.py:307)
            eng = self.engine
            x = torch.from_numpy(np.ascontiguousarray(frame.to_numpy(dtype=np.float64).T, dtype=np.float32)).to(eng.device)
            corr = PortfolioRiskService(ReturnBank(assets, x), device=eng.device).correlation_matrix()
            corr, chol, fallback = joint_factor(corr)
            method = self.mc_params["simulation_method"]
            if method == "historical":
                table = frame.dropna().to_numpy(dtype=np.float64)         # days with a return for every asset
                if len(table) == 0:
                    logger.error("No day with a return for every asset: cannot bootstrap the portfolio")
                    return {}
            elif method != "geometric_brownian_motion":
                logger.error("Unknown simulation method: %s", method)
                return {}
            periods_per_year, confidence = 252, self.mc_params["confidence_level"]
            steps = int(days) - 1
            world, rank = _world_rank()
            lo, hi, _ = shard_bounds(int(num_simulations), world, rank)
            results = {}
            for scenario in scenarios:
                drift_factor, volatility_factor = self._scenario_factors(scenario)
                mu = np.array([u[4].mean() * periods_per_year * drift_factor for u in used])                # :243
                sigma = np.array([u[4].std() * np.sqrt(periods_per_year) * volatility_factor for u in used])  # :244
                seed = self.seed + self._sim_counter
                self._sim_counter += 1
                if method == "geometric_brownian_motion":
                    finals, maxdd, af = eng.portfolio_gbm(s0, qty, mu, sigma, 1 / periods_per_year, chol.astype(np.float32),
                                                          hi - lo, steps, seed, path_offset=lo, asset_finals=True)
                else:
                    finals, maxdd, af = eng.portfolio_bootstrap(table, self.mc_params["return_method"] == "log", s0, qty,
                                                                hi - lo, steps, seed, path_offset=lo,
                                                                block_len=self.block_len, asset_finals=True)
                if world > 1:
                    finals, maxdd = gather_paths(finals, maxdd, int(num_simulations))
                    af = gather_path_rows(af, int(num_simulations))
                blocks = statistics_blocks(risk_statistics(eng, finals, maxdd, v0, confidence), v0, "price")
                asset_var = []
                for row, p0 in zip(af, s0):                              # risk_statistics' VaR (:316-317) of each asset
                    [(x_lo, x_hi, g)] = percentile_points(partial(eng.select, row), int(row.numel()),
                                                          [100 * (1 - confidence)])
                    asset_var.append(abs(_lerp((x_lo / p0 - 1) * 100, (x_hi / p0 - 1) * 100, g)))
                undiversified = float(sum(w * v for w, v in zip(weights.tolist(), asset_var)))
                var = blocks["risk_metrics"]["var"]
                results[scenario] = {
                    "scenario": scenario, "time_horizon_days": days, "num_simulations": num_simulations,
                    "simulation_method": method, "initial_value": v0,
                    "drift_factor": drift_factor, "volatility_factor": volatility_factor,
                    "mu": dict(zip(assets, mu.tolist())), "sigma": dict(zip(assets, sigma.tolist())),
                    **blocks,
                    "undiversified_var": undiversified,
                    "diversification_benefit": undiversified - var,
                }
            # _calculate_portfolio_stats' keys and conventions (:577-659), from the joint distribution
            scenario_stats = {s: {"expected_return": r["expected"]["pct_change"] / 100, "var": r["risk_metrics"]["var"] / 100,
                                  "cvar": r["risk_metrics"]["cvar"] / 100} for s, r in results.items()}
            base = scenario_stats.get("base", {})
            current = holdings["total_value"]
            return {
                "timestamp": datetime.now().isoformat(), "portfolio_value": current,
                "assets": assets, "weights": dict(zip(assets, weights.tolist())),
                "quantities": dict(zip(assets, qty.tolist())),
                "correlation": {a: {b: float(corr[i, j]) for j, b in enumerate(assets)} for i, a in enumerate(assets)},
                "correlation_fallback": bool(fallback),
                "scenarios": results,
                "portfolio_stats": {
                    "current_value": current,
                    "expected_value": current * (1 + base.get("expected_return", 0)),
                    "expected_change": base.get("expected_return", 0) * 100,
                    "var": base.get("var", 0) * 100,
                    "cvar": base.get("cvar", 0) * 100,
                    "var_loss_value": current * base.get("var", 0),
                    "scenario_stats": scenario_stats,
                },
            }
        except Exception as e:  # reference convention: log, return {}
            logger.error("Error running joint portfolio Monte Carlo simulation: %s", e, exc_info=True)
            return {}

    def _scenario_factors(self, scenario: str):
        """(drift_factor, volatility_factor) of a configured scenario, 1.0 for a factor it leaves out."""
        params = self.mc_params["scenarios"].get(scenario, {})
        return params.get("drift_factor", 1.0), params.get("volatility_factor", 1.0)

    def _calculate_portfolio_stats(self, holdings: Dict, simulations: Dict) -> Dict:
        """Value-weighted sums per scenario, correlations ignored (:577-659)."""
        try:
            assets = [a for a in holdings["assets"].keys() if a != "USDC"]
            non_usdc_value = sum(holdings["assets"][a]["value_usdc"] for a in assets)
            if non_usdc_value == 0:
                return {}
            weights = {a: holdings["assets"][a]["value_usdc"] / non_usdc_value for a in assets}
            scenario_stats = {}
            for scenario in self.mc_params["scenarios"].keys():
                er, vr, cv = [], [], []
                for a in assets:
                    key = f"{a}USDC_{scenario}"
                    if key in simulations:
                        w = weights.get(a, 0)
                        er.append(simulations[key]["expected"]["pct_change"] / 100 * w)
                        vr.append(simulations[key]["risk_metrics"]["var"] / 100 * w)
                        cv.append(simulations[key]["risk_metrics"]["cvar"] / 100 * w)
                if er:
                    scenario_stats[scenario] = {"expected_return": sum(er), "var": sum(vr), "cvar": sum(cv)}
            base = scenario_stats.get("base", {})
            current = holdings["total_value"]
            return {
                "current_value": current,
                "expected_value": current * (1 + base.get("expected_return", 0)),
                "expected_change": base.get("expected_return", 0) * 100,
                "var": base.get("var", 0) * 100,
                "cvar": base.get("cvar", 0) * 100,
                "var_loss_value": current * base.get("var", 0),
                "scenario_stats": scenario_stats,
            }
        except Exception as e:
            logger.error("Error calculating portfolio statistics: %s", e)
            return {}

    async def generate_monte_carlo_report(self, symbol: str = None, initial_price: float = None,
                                          holdings: Optional[Dict] = None) -> Dict:
        """:661-774; the live price / Redis lookups become arguments."""
        try:
            if symbol:
                sim = self.simulation_results.get(symbol)
                if sim is None:
                    if initial_price is None:
                        return {}
                    sim = self.run_monte_carlo_simulation(symbol, initial_price)
                    if not sim:
                        return {}
                return {
                    "symbol": symbol, "timestamp": datetime.now().isoformat(), "simulation": sim,
                    "risk_assessment": {
                        "time_horizon": f"{sim['time_horizon_days']} days",
                        "expected_return": f"{sim['expected']['pct_change']:.2f}%",
                        "price_range": {"low": f"${sim['percentiles']['5']['price']:.4f}",
                                        "median": f"${sim['percentiles']['50']['price']:.4f}",
                                        "high": f"${sim['percentiles']['95']['price']:.4f}"},
                        "risk_metrics": {
                            "var": f"{sim['risk_metrics']['var']:.2f}%",
                            "cvar": f"{sim['risk_metrics']['cvar']:.2f}%",
                            "probability_of_profit": f"{sim['risk_metrics']['prob_profit'] * 100:.1f}%",
                            "probability_of_loss": f"{sim['risk_metrics']['prob_loss'] * 100:.1f}%",
                            "max_drawdown": f"{sim['risk_metrics']['max_drawdown']['mean'] * 100:.2f}%"},
                    },
                }
            res = await self.run_portfolio_monte_carlo(holdings)
            ps = res.get("portfolio_stats", {}) if res else {}
            report = {
                "timestamp": datetime.now().isoformat(),
                "portfolio_value": ps.get("current_value", 0), "expected_value": ps.get("expected_value", 0),
                "expected_change": f"{ps.get('expected_change', 0):.2f}%",
                "value_at_risk": {"var_percent": f"{ps.get('var', 0):.2f}%",
                                  "var_amount": f"${ps.get('var_loss_value', 0):.2f}",
                                  "cvar_percent": f"{ps.get('cvar', 0):.2f}%"},
                "scenario_analysis": {s: {"expected_return": f"{v.get('expected_return', 0) * 100:.2f}%",
                                          "var": f"{v.get('var', 0) * 100:.2f}%",
                                          "cvar": f"{v.get('cvar', 0) * 100:.2f}%"}
                                      for s, v in ps.get("scenario_stats", {}).items()},
                "asset_analysis": {},
            }
            for key, sim in (res.get("asset_simulations", {}) if res else {}).items():
                if "_base" in key:
                    report["asset_analysis"][key.split("_base")[0]] = {
                        "expected_return": f"{sim['expected']['pct_change']:.2f}%",
                        "price_range": {"low": f"${sim['percentiles']['5']['price']:.4f}",
                                        "median": f"${sim['percentiles']['50']['price']:.4f}",
                                        "high": f"${sim['percentiles']['95']['price']:.4f}"},
                        "var": f"{sim['risk_metrics']['var']:.2f}%",
                        "prob_profit": f"{sim['risk_metrics']['prob_profit'] * 100:.1f}%"}
            return report
        except Exception as e:
            logger.error("Error generating Monte Carlo report: %s", e, exc_info=True)
            return {}
