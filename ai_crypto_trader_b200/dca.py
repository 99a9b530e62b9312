"""Dollar-cost averaging on the GPU engine: backtest a population of DCA parameter sets over a market's bars, and evolve
them.

Reference: services/dca_strategy.py (DCAStrategy).  The reference evaluates the service only in "simulation mode": its live
loop run() (:140-239) against the exchange ticker, once per update_interval, for as long as one waits.  Here one
individual is ONE service instance trading all of the market's symbols (the rebalance couples them), run over history by
b200bt_dca_sweep (csrc/dca.cu; the rule restated in include/b200bt.h and DESIGN.md section 3.14): a tick per bar, the bar's
close as the ticker price, the bar's label as market_regime_history.

    dca_param_ranges()     genes of the config keys the service reads (nested keys flattened, booleans as 0 / 1)
    quantity_precision()   _get_quantity_precision (:1094-1100) of a LOT_SIZE step
    DCASweep               population fitness / stats / service stats / objectives / per-day PnL rows on the device
    DCAStrategy            one parameter set, in the reference's result shape

The host turns each individual into exact lookup tables -- interval lengths in microseconds from Python's own timedelta,
the clamped order sizes, the rebalance targets after the last-symbol quirk, the dip cooldown and the rebalance period in
ticks -- so that the device does integer time arithmetic and the reference's float64 operations only.
"""
from __future__ import annotations

import copy
import ctypes as C
import logging
import math
from datetime import datetime, timedelta
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .population import StrategySweep, iso_minute

logger = logging.getLogger("b200bt.dca")

FIELDS = _lib.DCA_STATS_FIELDS
OBJECTIVE_FIELDS = FIELDS[:-3]          # purchase_hash, n_ticks and reserved describe the run, not the strategy
SERVICE_FIELDS = _lib.DCA_SERVICE_FIELDS
REGIMES = _lib.REGIMES
BEAR = REGIMES.index("bear")
DEFAULT_PRECISION = 6                   # _get_quantity_precision without a LOT_SIZE filter

# DCAStrategy.__init__ defaults (:63-136) of the keys the backtest reads, by their flattened gene name
DEFAULTS = {
    "interval_hours": 24, "base_order_size_usdc": 100, "min_order_size_usdc": 20, "max_order_size_usdc": 500,
    "price_dip_detection": True, "dip_threshold_pct": 5.0, "additional_dip_allocation": 0.5,
    "max_dip_frequency_days": 7, "adaptive_scheduling": True,
}
# flattened gene -> its path in the dca_strategy block (the reference's own default applies when the path is missing)
NESTED = {
    "bull_interval_hours": ("scheduling_strategies", "market_regime_based", "bull_interval_hours"),
    "bear_interval_hours": ("scheduling_strategies", "market_regime_based", "bear_interval_hours"),
    "volatile_interval_hours": ("scheduling_strategies", "market_regime_based", "volatile_interval_hours"),
    "day_of_week_weight": ("scheduling_strategies", "weighted_scheduling", "weight_factors", "day_of_week"),
    "increase_in_bear_market": ("market_condition_rules", "increase_in_bear_market"),
    "bear_market_adjustment": ("market_condition_rules", "bear_market_adjustment"),
    "periodic_rebalancing": ("periodic_rebalancing", "enabled"),
    "rebalance_interval_days": ("periodic_rebalancing", "rebalance_interval_days"),
    "max_deviation_pct": ("periodic_rebalancing", "max_deviation_pct"),
}
BOOLEAN_GENES = ("price_dip_detection", "adaptive_scheduling", "increase_in_bear_market", "periodic_rebalancing")


def dca_param_ranges() -> Dict[str, Tuple]:
    """GA genes of the DCA service's parameters (integer ranges where the reference's value is an integer or a flag)."""
    return {
        "interval_hours": (1.0, 168.0),
        "base_order_size_usdc": (20.0, 500.0),
        "price_dip_detection": (0, 1),
        "dip_threshold_pct": (1.0, 20.0),
        "additional_dip_allocation": (0.0, 2.0),
        "max_dip_frequency_days": (1, 30),
        "adaptive_scheduling": (0, 1),
        "bull_interval_hours": (1.0, 168.0),
        "bear_interval_hours": (1.0, 168.0),
        "volatile_interval_hours": (1.0, 168.0),
        "day_of_week_weight": (0.0, 1.0),
        "increase_in_bear_market": (0, 1),
        "bear_market_adjustment": (1.0, 3.0),
        "periodic_rebalancing": (0, 1),
        "rebalance_interval_days": (1, 90),
        "max_deviation_pct": (1.0, 50.0),
    }


def dca_block(config: Optional[Dict]) -> Dict:
    """The dca_strategy block of a config (a whole config.json dict, or the block itself)."""
    config = config or {}
    return config.get("dca_strategy", config) if isinstance(config, dict) else {}


def quantity_precision(step_size=None) -> int:
    """_get_quantity_precision (:1094-1100) of a LOT_SIZE stepSize (None: no LOT_SIZE filter, 6): the decimals of
    str(float(step)), so a step of 1e-05 (scientific notation) gives 0."""
    if step_size is None:
        return DEFAULT_PRECISION
    step = float(step_size)
    return len(str(step).rstrip('0').split('.')[1]) if '.' in str(step) else 0


def hours_to_us(hours) -> int:
    """timedelta(hours=x) in microseconds (Python's own rounding)."""
    return timedelta(hours=hours) // timedelta(microseconds=1)


def effective_block(block: Dict, params: Dict) -> Dict:
    """The dca_strategy block with an individual's genes written into their (nested) keys."""
    out = copy.deepcopy(block)
    for k, v in params.items():
        if k in NESTED:
            node = out
            *path, leaf = NESTED[k]
            for p in path:
                node = node.setdefault(p, {})
            node[leaf] = bool(int(v)) if k in BOOLEAN_GENES else v
        else:
            out[k] = bool(int(v)) if k in BOOLEAN_GENES else v
    return out


class Service:
    """The parameters DCAStrategy.__init__ (:63-136) reads from a dca_strategy block, with its defaults."""

    def __init__(self, b: Dict, symbols: Sequence[str]):
        self.symbols = list(symbols)
        self.interval_hours = b.get("interval_hours", DEFAULTS["interval_hours"])
        self.base_order_size_usdc = b.get("base_order_size_usdc", DEFAULTS["base_order_size_usdc"])
        self.min_order_size_usdc = b.get("min_order_size_usdc", DEFAULTS["min_order_size_usdc"])
        self.max_order_size_usdc = b.get("max_order_size_usdc", DEFAULTS["max_order_size_usdc"])
        self.price_dip_detection = b.get("price_dip_detection", DEFAULTS["price_dip_detection"])
        self.dip_threshold_pct = b.get("dip_threshold_pct", DEFAULTS["dip_threshold_pct"])
        self.additional_dip_allocation = b.get("additional_dip_allocation", DEFAULTS["additional_dip_allocation"])
        self.max_dip_frequency_days = b.get("max_dip_frequency_days", DEFAULTS["max_dip_frequency_days"])
        self.adaptive_scheduling = b.get("adaptive_scheduling", DEFAULTS["adaptive_scheduling"])
        strategies = b.get("scheduling_strategies", {})
        self.market_regime_scheduling = strategies.get("market_regime_based", {})
        self.weighted_scheduling = strategies.get("weighted_scheduling", {}).get("enabled", False)
        self.weighted_factors = strategies.get("weighted_scheduling", {}).get("weight_factors", {})
        self.periodic_rebalancing = b.get("periodic_rebalancing", {}).get("enabled", True)
        self.rebalance_interval_days = b.get("periodic_rebalancing", {}).get("rebalance_interval_days", 30)
        self.max_deviation_pct = b.get("periodic_rebalancing", {}).get("max_deviation_pct", 5.0)
        self.market_condition_rules = b.get("market_condition_rules", {})
        self.symbol_settings = b.get("symbol_settings", []) or []

    def settings(self, symbol: str) -> Dict:
        """symbols_config[symbol] as _get_symbol_specific_settings (:322-345) sets it."""
        s = next((s for s in self.symbol_settings if s.get("symbol") == symbol), None)
        if s:
            return {"allocation": s.get("allocation", 1.0 / len(self.symbols)),
                    "interval_hours": s.get("interval_hours", self.interval_hours),
                    "base_order_size_usdc": s.get("base_order_size_usdc", self.base_order_size_usdc)}
        return {"allocation": 1.0 / len(self.symbols), "interval_hours": self.interval_hours,
                "base_order_size_usdc": self.base_order_size_usdc}

    def interval_hours_at(self, interval_hours, label: Optional[int], weekday: int):
        """_calculate_next_purchase_time (:347-450) in hours, with no market_volatility / sentiment data."""
        if not self.adaptive_scheduling:
            return interval_hours
        if self.adaptive_scheduling and self.market_regime_scheduling and label is not None and label < len(REGIMES):
            regime = REGIMES[label]
            if regime == 'bull':
                interval_hours = self.market_regime_scheduling.get('bull_interval_hours', interval_hours)
            elif regime == 'bear':
                interval_hours = self.market_regime_scheduling.get('bear_interval_hours', interval_hours)
            elif regime == 'crab':
                interval_hours = self.market_regime_scheduling.get('crab_interval_hours', interval_hours)
            elif regime == 'volatile':
                interval_hours = self.market_regime_scheduling.get('volatile_interval_hours', interval_hours)
        if self.adaptive_scheduling and self.weighted_scheduling:
            day_weight = self.weighted_factors.get('day_of_week', 0.0)
            day_factor = 1.0 + (0.2 * day_weight * (weekday >= 5))
            volatility_factor = 1.0
            sentiment_factor = 1.0
            combined_factor = day_factor * volatility_factor * sentiment_factor
            interval_hours = max(interval_hours * 0.5, min(interval_hours * 1.5, interval_hours * combined_factor))
        return interval_hours

    def interval_table(self, interval_hours) -> np.ndarray:
        """int64 [5][2]: the interval in microseconds by [label][weekend] (label 4 = unknown = no label source)."""
        return np.array([[hours_to_us(self.interval_hours_at(interval_hours, lab, 5 if wk else 0)) for wk in (0, 1)]
                         for lab in range(len(REGIMES))], dtype=np.int64)

    def order_size(self, base, dip: bool, bear: bool):
        """_calculate_adjusted_order_size (:651-740) with no volatility / sentiment data."""
        adjusted_size = base
        if dip and self.price_dip_detection:
            adjusted_size = base * (1.0 + self.additional_dip_allocation)
        if self.market_condition_rules.get('increase_in_bear_market', False) and bear:
            adjusted_size *= self.market_condition_rules.get('bear_market_adjustment', 1.5)
        return max(self.min_order_size_usdc, min(self.max_order_size_usdc, adjusted_size))


def rebalance_period(days, bar_minutes: int) -> int:
    """Ticks between two rebalance checks (:191-200): (now - last).days >= R with last = now after each run."""
    if float(days) != int(days):
        raise ValueError(f"rebalance_interval_days = {days}: an integer number of days is needed")
    days = int(days)
    if days <= 0:
        return 1
    return max(1, -(-days * 1440 // int(bar_minutes)))


def decode_individual(params: Dict, block: Dict, symbols: Sequence[str], bar_minutes: int) -> Dict:
    """One parameter dict (genes, or keys of the block; missing keys from the block, then __init__'s defaults) -> the
    kernel's tables: {individual: DcaIndividual, first_us: int64 [S][5][2], target: float64 [S], service: Service}."""
    svc = Service(effective_block(block, params), symbols)
    S = len(symbols)
    last = svc.settings(symbols[-1])                     # what symbols_config holds after initialisation
    for h in [svc.interval_hours, last["interval_hours"]] + [svc.settings(s)["interval_hours"] for s in symbols]:
        if not float(h) >= 0.0:
            raise ValueError(f"interval_hours = {h}: must be >= 0")
    iv = _lib.DcaIndividual()
    for j, hours in enumerate((svc.interval_hours, last["interval_hours"])):
        table = svc.interval_table(hours)
        for lab in range(5):
            for wk in range(2):
                iv.later_us[j][lab][wk] = int(table[lab, wk])
    for j, base in enumerate((svc.base_order_size_usdc, last["base_order_size_usdc"])):
        for dip in range(2):
            for bear in range(2):
                iv.order[j][dip][bear] = float(svc.order_size(base, bool(dip), bool(bear)))
    iv.dip_threshold_pct = float(svc.dip_threshold_pct)
    iv.max_deviation_pct = float(svc.max_deviation_pct)
    f = float(svc.max_dip_frequency_days)
    iv.dip_cooldown_minutes = int(math.ceil(f)) * 1440 if f > 0 else 0
    iv.rebalance_first = 0
    iv.rebalance_period = rebalance_period(svc.rebalance_interval_days, bar_minutes)
    iv.flags = (_lib.DCA_DIP if svc.price_dip_detection else 0) | (_lib.DCA_REBALANCE if svc.periodic_rebalancing else 0)
    first = np.stack([svc.interval_table(svc.settings(s)["interval_hours"]) for s in symbols])
    target = np.full(S, 1.0 / S)
    target[-1] = float(last["allocation"])
    return {"individual": iv, "first_us": first, "target": target, "service": svc}


class DCASweep(StrategySweep):
    """b200bt_dca_sweep for populations of DCA parameter dicts on one market.

    market              MarketData (device closes and highs, bar clock); every close from start_bar on must be > 0
    config              config.json dict or its dca_strategy block: the keys an individual does not set, symbol_settings
    regime              None (no regime source), a device uint8 label tensor [S or 1][N] (B200BT_REGIME_*), or True for
                        regime.regime_labels(market)
    start_bar           tick 0 (the dip rule's klines reach back into the bars before it)
    usdc_balance        get_account's USDC balance, constant (simulation mode places no orders)
    quantity_precision  decimals of the quantities: None (6, no LOT_SIZE filter), one int, or one per symbol (see
                        quantity_precision() for a LOT_SIZE step)
    objective           the stats field (mean over the symbols) or service field evaluate() returns

    The rebalance targets depend on the config alone, so they are the same for every individual.  Individuals that
    decode alike are evaluated once."""

    FIELDS, OBJECTIVE_FIELDS, SERVICE_FIELDS = FIELDS, OBJECTIVE_FIELDS, SERVICE_FIELDS
    SERVICE_OBJECTIVE_FIELDS = SERVICE_FIELDS
    service = True

    def __init__(self, market, config: Optional[Dict] = None, regime=None, start_bar: int = 0, usdc_balance: float = 0.0,
                 quantity_precision: Union[None, int, Sequence[int]] = None, objective: str = "total_profit_pct"):
        self.market = market
        self.block = dca_block(config)
        S, N = market.S, market.N
        if not 0 <= int(start_bar) < N:
            raise ValueError(f"start_bar = {start_bar} outside [0, {N})")
        self.start_bar = int(start_bar)
        if not bool((market.close[:, self.start_bar:] > 0).all()):
            raise ValueError("every close from the start bar on must be > 0 (the quantity is order / price)")
        if quantity_precision is None:
            prec = [DEFAULT_PRECISION] * S
        elif np.ndim(quantity_precision) == 0:
            prec = [int(quantity_precision)] * S
        else:
            prec = [int(p) for p in quantity_precision]
        if len(prec) != S or not all(0 <= p <= 22 for p in prec):
            raise ValueError(f"quantity_precision: {S} values in 0 .. 22 needed")
        self.precision = prec
        self._pow10 = torch.tensor([float(10 ** p) for p in prec], dtype=torch.float64, device=market.device)
        self.usdc_balance = float(usdc_balance)
        from .regime import label_rows, regime_labels
        if regime is True:
            regime = regime_labels(market)[0]
        self.labels, self.ld_labels = None, 0
        if regime is not None:
            self.labels, self.ld_labels = label_rows(regime, S, N)
        self.objective = objective
        self._column(objective)
        self.dip = dip_pct(market)
        self._ws = torch.empty(max(1, _lib.load().b200bt_dca_workspace_bytes(S, N)), dtype=torch.uint8,
                               device=market.device)

    # -- host decoding --------------------------------------------------------------------------------------------
    def decode(self, population: List[Dict]) -> Tuple[np.ndarray, np.ndarray, np.ndarray, bool]:
        """(individuals: DcaIndividual bytes [pop], first_us int64 [pop][S][5][2], target float64 [S], rebalance_any)."""
        m = self.market
        rows = (_lib.DcaIndividual * len(population))()
        first = np.empty((len(population), m.S, 5, 2), dtype=np.int64)
        target = None
        for i, params in enumerate(population):
            d = decode_individual(params, self.block, m.symbols, m.bar_minutes)
            rows[i] = d["individual"]
            first[i] = d["first_us"]
            target = d["target"]
        packed = np.frombuffer(bytes(rows), dtype=np.uint8).reshape(len(population), C.sizeof(_lib.DcaIndividual))
        flags = np.array([r.flags for r in rows])
        return packed, first, target, bool(np.any(flags & _lib.DCA_REBALANCE))

    def _inputs(self, population: List[Dict]):
        packed, first, target, reb = self.decode(population)
        return [packed, first], {"target": torch.from_numpy(target).to(self.market.device), "rebalance_any": reb}

    def launch(self, indiv: torch.Tensor, first_us: torch.Tensor, stats: torch.Tensor, service: Optional[torch.Tensor],
               rows: Optional[torch.Tensor] = None, *, target: torch.Tensor, rebalance_any: bool) -> None:
        """b200bt_dca_sweep on the current stream for the decoded individuals `indiv` (DcaIndividual bytes [U]), their
        first intervals `first_us` [U][S][5][2] and the rebalance targets `target` [S], writing `stats` [U][S][20],
        `service` [U][5] and, when given, the per-day rows `rows` [U][D]."""
        m = self.market
        _lib.call("b200bt_dca_sweep", m.close.data_ptr(), _lib.ld(m.close), self.dip.data_ptr(), m.N, m.S, m.N,
                  self.start_bar, m.bar_minutes, m.minute0, self._ws.data_ptr(), self._ws.numel(), indiv.data_ptr(),
                  first_us.data_ptr(), indiv.shape[0], int(rebalance_any), target.data_ptr(), self._pow10.data_ptr(),
                  _lib.ptr(self.labels), self.ld_labels, self.usdc_balance, stats.data_ptr(), _lib.ptr(service),
                  _lib.ptr(rows), 0 if rows is None else rows.shape[1], _lib.current_stream())

    dca_stats = StrategySweep.stats_dict

    def day_pnl(self, population: List[Dict]) -> Tuple[torch.Tensor, int]:
        """(rows float64 [pop][D] on the device, first_day): row i, column d = the change of individual i's
        sum_s (Q_s * c_s - I_s) over calendar day first_day + d -- the row shape b200bt_cscv takes."""
        return self.day_rows(population)


def dip_pct(market) -> torch.Tensor:
    """b200bt_dca_dip_pct of a market: float64 [S][N] on the device, the drop from the 7-day high in percent (NaN where
    _check_for_dips makes no check)."""
    out = torch.empty((market.S, market.N), dtype=torch.float64, device=market.device)
    high, close = market.high, market.close
    if _lib.ld(high) != _lib.ld(close):
        high = high.contiguous()
        close = close.contiguous()
    with torch.cuda.device(market.device):
        _lib.call("b200bt_dca_dip_pct", high.data_ptr(), close.data_ptr(), _lib.ld(close), market.S, market.N,
                  market.minute0, market.bar_minutes, out.data_ptr(), market.N, _lib.current_stream())
    return out


class DCAStrategy:
    """The DCA service's evaluation on the GPU engine, one parameter set at a time.  config: config.json dict (or its
    dca_strategy block), as the reference reads it."""

    def __init__(self, config: Optional[Dict] = None):
        self.config = config or {}
        self.dca_config = dca_block(self.config)

    def backtest(self, market, params: Optional[Dict] = None, start_bar: int = 0, regime=None, usdc_balance: float = 0.0,
                 quantity_precision=None) -> Optional[Dict]:
        """Run the service over the market's bars (its symbols) from start_bar with `params` (genes or keys of the
        dca_strategy block; the config fills the rest).  Returns {"dca_positions": per symbol the reference's position
        dict without the purchase list, "dca_performance": the _update_performance_metrics dict at the last tick,
        "stats": per symbol every b200bt_dca_stats field}.  Errors are logged and give None (the reference's convention)."""
        try:
            sweep = DCASweep(market, config=self.dca_config, regime=regime, start_bar=start_bar,
                             usdc_balance=usdc_balance, quantity_precision=quantity_precision)
            st = sweep.dca_stats([dict(params or {})])
            sv = {k: float(v[0]) for k, v in sweep.service_stats().items()}
            t0 = market.minute0 + sweep.start_bar * market.bar_minutes
            t1 = market.minute0 + (market.N - 1) * market.bar_minutes
            last_close = market.close[:, -1].double().cpu().numpy()
            positions, stats = {}, {}
            for s, sym in enumerate(market.symbols):
                v = {k: float(a[0, s]) for k, a in st.items()}
                stats[sym] = v
                k = int(v["last_purchase_tick"])
                positions[sym] = {
                    "symbol": sym, "total_invested": v["total_invested"], "total_quantity": v["total_quantity"],
                    "average_price": v["average_price"],
                    "last_purchase_time": iso_minute(t0 + k * market.bar_minutes) if k >= 0 else None,
                    "last_purchase_price": v["last_purchase_price"], "current_price": float(last_close[s]),
                    "current_value": v["current_value"], "profit_loss": v["profit_loss"],
                    "profit_loss_pct": v["profit_loss_pct"],
                }
            next_buys = {sym: (datetime(1970, 1, 1) + timedelta(minutes=t0, microseconds=int(stats[sym]["next_scheduled_us"])))
                         .isoformat() for sym in market.symbols}
            performance = {
                "timestamp": iso_minute(t1), "start_time": iso_minute(t0), "running_time_hours": (t1 - t0) * 60 / 3600,
                "total_purchases": int(sv["total_purchases"]), "total_invested": sv["total_invested"],
                "total_value": sv["total_value"], "total_profit": sv["total_profit"],
                "total_profit_pct": sv["total_profit_pct"], "symbols": list(market.symbols),
                "avg_costs": {sym: {"average_price": p["average_price"], "total_quantity": p["total_quantity"],
                                    "current_price": p["current_price"], "profit_loss_pct": p["profit_loss_pct"]}
                              for sym, p in positions.items() if p["total_quantity"] > 0},
                "simulation_mode": True, "next_scheduled_buys": next_buys,
            }
            return {"dca_positions": positions, "dca_performance": performance, "stats": stats}
        except Exception as e:
            logger.error("Error backtesting DCA: %s", e)
            return None
