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


class PathEngine:
    """Device-side Monte-Carlo primitives (one instance per GPU)."""

    def __init__(self, device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("Monte-Carlo engine needs a CUDA device (sm_90); there is no CPU path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._ws = None

    def gbm(self, s0, mu, sigma, dt, n_paths, steps, seed, path_offset=0, store_paths=False):
        dev = self.device
        if n_paths == 0:          # a rank without paths (more ranks than paths)
            e = torch.empty(0, dtype=torch.float32, device=dev)
            return e, e.clone(), None
        finals = torch.empty(n_paths, dtype=torch.float32, device=dev)
        maxdd = torch.empty(n_paths, dtype=torch.float32, device=dev)
        paths = torch.empty((steps + 1, n_paths), dtype=torch.float32, device=dev) if store_paths else None
        with torch.cuda.device(dev):
            _lib.call("b200bt_mc_gbm", float(s0), float(mu), float(sigma), float(dt), int(n_paths), int(steps),
                      int(seed) & (2**64 - 1), int(path_offset), finals.data_ptr(), maxdd.data_ptr(), _lib.ptr(paths),
                      _lib.current_stream())
        return finals, maxdd, paths

    def bootstrap(self, returns: np.ndarray, log_returns: bool, s0, n_paths, steps, seed, path_offset=0,
                  block_len=1, store_paths=False):
        dev = self.device
        if n_paths == 0:          # a rank without paths (more ranks than paths), as in gbm()
            e = torch.empty(0, dtype=torch.float32, device=dev)
            return e, e.clone(), None
        r = torch.from_numpy(np.ascontiguousarray(returns, dtype=np.float32)).to(dev)
        finals = torch.empty(n_paths, dtype=torch.float32, device=dev)
        maxdd = torch.empty(n_paths, dtype=torch.float32, device=dev)
        paths = torch.empty((steps + 1, n_paths), dtype=torch.float32, device=dev) if store_paths else None
        with torch.cuda.device(dev):
            _lib.call("b200bt_mc_bootstrap", r.data_ptr(), int(r.numel()), int(block_len), 1 if log_returns else 0,
                      float(s0), int(n_paths), int(steps), int(seed) & (2**64 - 1), int(path_offset),
                      finals.data_ptr(), maxdd.data_ptr(), _lib.ptr(paths), _lib.current_stream())
        return finals, maxdd, paths

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
                    confidence: float) -> Dict:
    """The statistics block of run_monte_carlo_simulation (:305-336) from device arrays."""
    n = int(finals.numel())
    var_percentile = 100 * (1 - confidence)                       # :316
    idx = [_virtual_index(n, p) for p in PERCENTILES] + [_virtual_index(n, var_percentile)]
    ranks = sorted({i for lo, hi, _ in idx for i in (lo, hi)})
    vals = dict(zip(ranks, engine.select(finals, ranks)))
    percentile_values = [_lerp(vals[lo], vals[hi], g) for lo, hi, g in idx[:-1]]
    lo, hi, g = idx[-1]
    pct = lambda v: (v / initial_price - 1) * 100                 # :312
    var = _lerp(pct(vals[lo]), pct(vals[hi]), g)                  # :317 on pct_changes (monotone in S_T)
    mid = sorted({(n - 1) // 2, n // 2})
    dd_mid = engine.select(maxdd, mid)
    m = engine.moments(finals, maxdd, initial_price, var)
    cvar = m[5] / m[6] if m[6] > 0 else float("nan")              # :320
    prob_profit = m[2] / n                                        # :323
    return {
        "percentile_values": percentile_values,
        "expected_price": m[0] / n, "expected_pct": m[1] / n,
        "var": var, "cvar": cvar, "prob_profit": prob_profit,
        "mdd_mean": m[3] / n, "mdd_median": float(np.mean(dd_mid)), "mdd_max": float(m[4]),
    }


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
            scenario_params = self.mc_params["scenarios"].get(scenario, {})
            drift_factor = scenario_params.get("drift_factor", 1.0)
            volatility_factor = scenario_params.get("volatility_factor", 1.0)
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
            world, rank = 1, 0
            if torch.distributed.is_available() and torch.distributed.is_initialized() and not store:
                world, rank = torch.distributed.get_world_size(), torch.distributed.get_rank()
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
                "percentiles": {str(p): {"price": float(v), "pct_change": float((v / initial_price - 1) * 100)}
                                for p, v in zip(PERCENTILES, st["percentile_values"])},
                "expected": {"price": float(st["expected_price"]), "pct_change": float(st["expected_pct"])},
                "risk_metrics": {
                    "var": float(abs(st["var"])), "cvar": float(abs(st["cvar"])),
                    "prob_profit": float(st["prob_profit"]), "prob_loss": float(1 - st["prob_profit"]),
                    "max_drawdown": {"mean": float(st["mdd_mean"]), "median": float(st["mdd_median"]),
                                     "max": float(st["mdd_max"])},
                },
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
