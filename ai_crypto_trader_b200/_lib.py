"""ctypes binding of the C-ABI in include/b200bt.h (libb200bt.so, built in-tree).

There is no fallback: if the shared library is missing, or a compute entry
point is called without an sm_90 device, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("B200BT_LIB", _HERE / "libb200bt.so"))


class B200btError(RuntimeError):
    """Non-zero status from the C-ABI."""

    def __init__(self, fn: str, status: int, message: str):
        super().__init__(f"{fn} failed with status {status}: {message}")
        self.status = status


class Individual(C.Structure):
    _fields_ = [
        ("rsi_row", C.c_int32),
        ("rsi_lo", C.c_float),
        ("rsi_hi", C.c_float),
        ("reserved", C.c_int32),
        ("take_profit", C.c_double),
        ("stop_loss", C.c_double),
        ("position_size", C.c_double),
    ]


class BtParams(C.Structure):
    _fields_ = [
        ("initial_balance", C.c_double), ("position_pct", C.c_double), ("stop_loss_pct", C.c_double),
        ("take_profit_pct", C.c_double), ("volume_factor", C.c_double), ("max_risk_per_trade", C.c_double),
        ("can_enter", C.c_int32), ("skip", C.c_int32),
    ]


class SweepConfig(C.Structure):
    _fields_ = [
        ("initial_capital", C.c_double),
        ("minute0", C.c_int64),
        ("bar_minutes", C.c_int32),
        ("primary", C.c_int32),
        ("secondary_mask", C.c_int32),
        ("variant", C.c_int32),
        ("gap_bar", C.c_int32),
        ("gap_minutes", C.c_int32),
    ]


class RegimeParams(C.Structure):
    """b200bt_regime_params: the point clock and the thresholds of detect_regime_from_data
    (services/market_regime_service.py:100-118, at their defaults)."""
    _fields_ = [
        ("sample_minutes", C.c_int32), ("reserved", C.c_int32),
        ("volatile_volatility", C.c_double), ("bull_price_change", C.c_double), ("bull_trend_strength", C.c_double),
        ("bear_price_change", C.c_double), ("bear_trend_strength", C.c_double), ("ranging_price_range", C.c_double),
        ("ranging_trend_strength", C.c_double),
    ]


class GridIndividual(C.Structure):
    """b200bt_grid_individual: one grid parameter set, decoded by the host (grid.py)."""
    _fields_ = [
        ("num_grids", C.c_int32), ("grid_type", C.c_int32), ("rebalance_ticks", C.c_int32), ("adjust_ticks", C.c_int32),
        ("flags", C.c_int32), ("reserved", C.c_int32), ("lower_pct", C.c_double), ("upper_pct", C.c_double),
    ]


class GridRegimeRule(C.Structure):
    """b200bt_grid_regime_rule: what the adjustment's regime rule sets for one label."""
    _fields_ = [("apply", C.c_int32), ("num_grids", C.c_int32), ("lower_pct", C.c_double), ("upper_pct", C.c_double)]


class DcaIndividual(C.Structure):
    """b200bt_dca_individual: one DCA parameter set as the host's lookup tables (dca.py)."""
    _fields_ = [
        ("later_us", (C.c_int64 * 2) * 5 * 2), ("order", (C.c_double * 2) * 2 * 2), ("dip_threshold_pct", C.c_double),
        ("max_deviation_pct", C.c_double), ("dip_cooldown_minutes", C.c_int64), ("rebalance_first", C.c_int64),
        ("rebalance_period", C.c_int64), ("flags", C.c_int32), ("reserved", C.c_int32),
    ]


DCA_STATS_FIELDS = (
    "total_invested", "total_quantity", "average_price", "current_value", "profit_loss", "profit_loss_pct",
    "n_scheduled", "n_dip", "n_rebalance", "order_usdc", "last_purchase_price", "last_purchase_tick",
    "next_scheduled_us", "last_dip_tick", "n_zero_quantity", "n_rebalance_checks", "min_day_profit_loss",
    "purchase_hash", "n_ticks", "reserved",
)                                                                     # b200bt_dca_stats, 160 bytes
DCA_SERVICE_FIELDS = ("total_purchases", "total_invested", "total_value", "total_profit", "total_profit_pct")
DCA_DIP = 1
DCA_REBALANCE = 2
DCA_MAX_COUPLED = 32

GRID_STATS_FIELDS = (
    "total_profit", "total_trades", "profitable_trades", "win_rate", "profit_per_day", "up_crossings", "down_crossings",
    "n_regenerations", "num_grids", "lower", "upper", "cash", "position", "mark_to_market", "max_position",
    "min_position", "n_rebalance_checks", "n_adjustments", "n_ticks", "near_ties",
)                                                                     # b200bt_grid_stats, 160 bytes
GRID_SERVICE_FIELDS = (
    "total_profit", "total_trades", "profitable_trades", "win_rate", "profit_per_day", "num_grids", "lower_pct",
    "upper_pct", "n_adjustments", "n_num_grids_changes", "min_num_grids", "max_num_grids",
)                                                                     # b200bt_grid_service_stats, 96 bytes
GRID_ADAPT_REGIME = 1
GRID_AUTO_BOUNDARIES = 2
GRID_MAX_GRIDS = 127
GRID_TYPES = ("arithmetic", "geometric")                              # B200BT_GRID_* = index

class RlAgent(C.Structure):
    """b200bt_rl_agent: one agent's seed, symbol and hyperparameters."""
    _fields_ = [
        ("seed", C.c_uint64), ("symbol", C.c_int32), ("batch_size", C.c_int32), ("memory_size", C.c_int32),
        ("update_target_every", C.c_int32), ("learning_rate", C.c_double), ("gamma", C.c_double),
        ("epsilon_start", C.c_double), ("epsilon_end", C.c_double), ("epsilon_decay", C.c_double),
    ]


RL_STATE_DTYPE = [("initialized", "<i8"), ("n_transitions", "<i8"), ("replays", "<i8"), ("epsilon", "<f8"),
                  ("act_words", "<u8"), ("sample_words", "<u8"), ("mean_q", "<f8"), ("reserved", "<i8")]
                                                                      # b200bt_rl_agent_state, 64 bytes
RL_FEATURES = 16
RL_PARAMS = 1083
RL_MAX_BATCH = 128
RL_MAX_MEMORY = 1 << 20

REGIMES = ("bull", "bear", "ranging", "volatile", "unknown")          # B200BT_REGIME_* = index
REGIME_WINDOW_DTYPE = [("start_minute", "<i8"), ("n_points", "<i4"), ("label", "<i4"), ("volatility", "<f8"),
                       ("change_pct", "<f8"), ("mean_strength", "<f8"), ("up_frac", "<f8"), ("down_frac", "<f8"),
                       ("sideways_frac", "<f8")]                      # b200bt_regime_window, 64 bytes

LANE_STATS_FIELDS = (
    "n_records", "n_wins", "n_losses", "total_profit", "total_loss", "net_profit",
    "max_drawdown", "sharpe_ratio", "n_days", "largest_profit", "largest_loss",
    "sum_duration_bars", "score", "win_rate", "profit_factor",
    "sortino_ratio", "n_negative_days", "downside_deviation", "mean_daily_pnl", "trade_hash",
)
LANE_STATS_WORDS = len(LANE_STATS_FIELDS)

ANALYZER_COLUMNS = ("sma_20", "sma_50", "sma_200", "ema_12", "ema_26", "macd", "macd_signal", "macd_diff", "ichimoku_a",
                    "ichimoku_b", "rsi", "bb_high", "bb_mid", "bb_low", "bb_width", "atr", "vwap", "stoch_k", "stoch_d",
                    "williams_r", "bb_position")      # enum b200bt_analyzer_column

EVENT_EXIT = 0x40000000
EVENT_SELL = 0x80000000
EVENT_BAR_MASK = 0x3FFFFFFF

TRADE_MC_METHODS = {"bootstrap": 0, "shuffle": 1}     # B200BT_TRADE_MC_*

PRIMARY = {"sharpe_ratio": 0, "return_pct": 1, "profit_factor": 2, "win_rate": 3, "net_profit": 4, "total_trades": 5,
           "max_drawdown": 6, "total_profit": 7, "total_loss": 8, "largest_profit": 9, "largest_loss": 10,
           "average_profit": 11, "average_loss": 12}
PRIMARY_ADVANCED = {"sortino_ratio": 13, "expectancy": 14, "calmar_ratio": 15, "profit_per_day": 16, "recovery_factor": 17}
PRIMARY_ZERO = 99
SECONDARY = {"max_drawdown": 1, "win_rate": 2, "profit_factor": 4}
SECONDARY_ADVANCED = {"expectancy": 8}


def score_codes(goals: dict, advanced: bool = False):
    """(primary code, secondary mask) of `_calculate_strategy_score` (strategy_evaluation.py:579-633) for the kernels.

    `advanced` = the score is taken on calculate_advanced_metrics' dict (evaluate_strategy :545-557) instead of the plain
    calculate_metrics dict (cross_validate_strategy :683-691).  The reference reads `metrics.get(primary, 0)` and walks
    an if / elif chain over the secondary names, so a key the dict does not hold scores 0 and an unknown secondary
    name (or `expectancy` on the plain dict, where the key is absent and the factor is 1) changes nothing."""
    name = goals.get("primary", "sharpe_ratio")
    table = dict(PRIMARY, **PRIMARY_ADVANCED) if advanced else PRIMARY
    primary = table.get(name, PRIMARY_ZERO)
    sec = dict(SECONDARY, **SECONDARY_ADVANCED) if advanced else SECONDARY
    mask = 0
    for m in goals.get("secondary", []):
        mask |= sec.get(m, 0)
    return primary, mask

_vp, _i, _i64 = C.c_void_p, C.c_int, C.c_int64

_SIGNATURES = {
    "b200bt_abi_version": (C.c_int, []),
    "b200bt_last_error": (C.c_char_p, []),
    "b200bt_launch_count": (C.c_int64, []),
    "b200bt_rsi_bank": (C.c_int, [_vp, _i, _i64, _i64, C.POINTER(C.c_int), _i, _i, _vp, _vp]),
    "b200bt_rsi_bank_zones": (C.c_int, [_vp, _i, _i64, _i64, C.POINTER(C.c_int), _i, _vp, _vp, _i, _i, _vp]),
    "b200bt_ema_bank": (C.c_int, [_vp, _i, _i64, _i64, C.POINTER(C.c_int), _i, _vp, _vp]),
    "b200bt_sma_bank": (C.c_int, [_vp, _i, _i64, _i64, C.POINTER(C.c_int), _i, _vp, _vp]),
    "b200bt_macd": (C.c_int, [_vp, _i, _i64, _i64, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "b200bt_bollinger": (C.c_int, [_vp, _i, _i64, _i64, _i, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200bt_stochastic": (C.c_int, [_vp, _vp, _vp, _i, _i64, _i64, _i, _i, _vp, _vp, _vp]),
    "b200bt_williams_r": (C.c_int, [_vp, _vp, _vp, _i, _i64, _i64, _i, _vp, _vp]),
    "b200bt_ichimoku": (C.c_int, [_vp, _vp, _i, _i64, _i64, _i, _i, _i, _vp, _vp, _vp]),
    "b200bt_atr_bank": (C.c_int, [_vp, _vp, _vp, _i, _i64, _i64, C.POINTER(C.c_int), _i, _vp, _vp]),
    "b200bt_vwap": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i64, _i64, _i, _vp, _vp]),
    "b200bt_analyzer_workspace_floats": (C.c_int64, [_i, _i64]),
    "b200bt_analyzer": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i64, _i64, _vp, _vp, _vp]),
    "b200bt_resample_bars": (C.c_int64, [_i64, _i64, _i, _i]),
    "b200bt_resample": (C.c_int, [_vp, _i, _i64, _i64, _i, _i, _vp, _i64, _vp]),
    "b200bt_align": (C.c_int, [_vp, _i, _i64, _i64, _i64, _i, _i, _vp, _vp]),
    "b200bt_nanfill_workspace_floats": (C.c_int64, [_i64, _i64]),
    "b200bt_nanfill": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "b200bt_sweep": (C.c_int, [_vp, _i64, _vp, _i64, _i, _i, _i64, _vp, _vp, _i,
                               C.POINTER(SweepConfig), _vp, _vp, _i64, _vp]),
    "b200bt_sweep_chunked_workspace_bytes": (C.c_int64, [_i, _i, _i]),
    "b200bt_sweep_chunked": (C.c_int, [_vp, _i64, _vp, _i64, _i, _i, _i64, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i,
                                       _vp, _i64, C.POINTER(SweepConfig), _vp, _vp, _i64, _vp, _vp, _vp]),
    "b200bt_sweep_tiled_workspace_bytes": (C.c_int64, [_i, _i, _i, _i]),
    "b200bt_sweep_scan_timing": (C.c_int, [_vp, _vp]),
    "b200bt_sweep_scan_wait_cycles": (C.c_int, [_i64]),
    "b200bt_zone_map_floats": (C.c_int64, [_i, _i, _i64]),
    "b200bt_zone_map": (C.c_int, [_vp, _i64, _vp, _i64, _i, _i, _i64, _vp, _vp]),
    "b200bt_sweep_tiled": (C.c_int, [_vp, _i64, _vp, _i64, _i, _i, _i64, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i,
                                     _vp, _i64, C.POINTER(SweepConfig), _vp, _vp, _i64, _vp, _vp, _vp]),
    "b200bt_fitness_reduce": (C.c_int, [_vp, _i, _i, _vp, _vp]),
    "b200bt_book_metrics": (C.c_int, [_vp, _i64, _i, _i64, _vp, _i, C.POINTER(SweepConfig), _vp, _vp, _i64, _vp, _vp,
                                      _vp]),
    "b200bt_backtest_ref": (C.c_int, [_vp, _i64, _i, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _vp]),
    "b200bt_mc_gbm": (C.c_int, [C.c_double, C.c_double, C.c_double, C.c_double, _i64, _i, C.c_uint64, C.c_uint64,
                                _vp, _vp, _vp, _vp]),
    "b200bt_mc_bootstrap": (C.c_int, [_vp, _i, _i, _i, C.c_double, _i64, _i, C.c_uint64, C.c_uint64,
                                      _vp, _vp, _vp, _vp]),
    "b200bt_select_workspace_bytes": (C.c_int64, [_i]),
    "b200bt_select": (C.c_int, [_vp, _i64, _vp, _i, _vp, _vp, _i64, _vp]),
    "b200bt_mc_moments": (C.c_int, [_vp, _vp, _i64, C.c_double, C.c_double, _vp, _vp]),
    "b200bt_mc_portfolio_gbm": (C.c_int, [_i, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                          C.POINTER(C.c_double), C.POINTER(C.c_float), _i64, _i, C.c_uint64, C.c_uint64,
                                          _vp, _vp, _vp, _vp]),
    "b200bt_mc_portfolio_bootstrap": (C.c_int, [_i, _vp, _i, _i, _i, C.POINTER(C.c_double), C.POINTER(C.c_double), _i64,
                                                _i, C.c_uint64, C.c_uint64, _vp, _vp, _vp, _vp]),
    "b200bt_trade_pnl": (C.c_int, [_vp, _i64, _i, _i64, _vp, _i, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp]),
    "b200bt_trade_mc": (C.c_int, [_vp, _i64, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_uint32), _i, _i,
                                  _i, C.c_double, _i64, C.c_uint64, C.c_uint64, _vp, _vp, _vp]),
    "b200bt_ga_init": (C.c_int, [_vp, _i, _i, _i, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int),
                                 C.c_uint64, _vp]),
    "b200bt_ga_next_generation": (C.c_int, [_vp, _vp, _vp, _i, _i, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                            C.POINTER(C.c_int), C.c_double, _i, C.c_double, C.c_double, C.c_uint64,
                                            C.c_uint32, _vp, _vp, _vp]),
    "b200bt_objective_matrix": (C.c_int, [_vp, _i, _i, C.POINTER(C.c_int), _i, _vp, _i64, _vp]),
    "b200bt_pareto_workspace_bytes": (C.c_int64, [_i, _i]),
    "b200bt_pareto_rank": (C.c_int, [_vp, _i64, _i, _i, C.POINTER(C.c_int), _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "b200bt_daily_pnl": (C.c_int, [_vp, _i64, _i, _i64, _vp, _i, C.POINTER(SweepConfig), _vp, _vp, _i64, _vp, _i64, _vp,
                                   _vp]),
    "b200bt_cscv_workspace_bytes": (C.c_int64, [_i, _i64, _i]),
    "b200bt_cscv": (C.c_int, [_vp, _i64, _i, _i64, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200bt_regime_max_windows": (C.c_int64, [_i64, _i]),
    "b200bt_regime_labels": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i64, _i64, _i64, _i, C.POINTER(RegimeParams), _vp, _i64,
                                       _vp, _i64, _vp]),
    "b200bt_class_stats": (C.c_int, [_vp, _i64, _i, _i64, _vp, _i, C.POINTER(SweepConfig), _vp, _vp, _i64, _vp, _i64, _i,
                                     _vp, _vp]),
    "b200bt_grid_sweep": (C.c_int, [_vp, _i64, _i, _i64, _i64, _i, _i64, _vp, _i, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64,
                                    _vp]),
    "b200bt_grid_service_sweep": (C.c_int, [_vp, _i64, _i, _i64, _i64, _i, _i64, _vp, _i, _vp, _vp, _vp, _i64, _vp, _vp,
                                            _vp, _vp, _i64, _vp]),
    "b200bt_dca_dip_pct": (C.c_int, [_vp, _vp, _i64, _i, _i64, _i64, _i, _vp, _i64, _vp]),
    "b200bt_dca_workspace_bytes": (C.c_int64, [_i, _i64]),
    "b200bt_dca_sweep": (C.c_int, [_vp, _i64, _vp, _i64, _i, _i64, _i64, _i, _i64, _vp, _i64, _vp, _vp, _i, _i, _vp, _vp,
                                   _vp, _i64, C.c_double, _vp, _vp, _vp, _i64, _vp]),
    "b200bt_rl_states": (C.c_int, [_vp, _vp, _vp, _i64, _i, _i64, _i, _vp, _vp]),
    "b200bt_rl_workspace_bytes": (C.c_int64, [_i, _i]),
    "b200bt_rl_train": (C.c_int, [_vp, _i, _i64, _vp, _i, _i64, _i, _vp, _i64, _vp, _i, _i, _vp, _vp, _vp, _vp, _i64, _vp]),
    "b200bt_pct_change": (C.c_int, [_vp, _i64, _i, _i64, _vp, _i64, _vp]),
    "b200bt_tail_stats_workspace_bytes": (C.c_int64, [_i64]),
    "b200bt_tail_stats": (C.c_int, [_vp, _i64, C.c_double, _vp, _vp, _i64, _vp]),
    "b200bt_correlation_workspace_bytes": (C.c_int64, [_i, _i64]),
    "b200bt_correlation": (C.c_int, [_vp, _i64, _i, _i64, _vp, _vp, _i64, _vp]),
}

_lib = None


def exported_symbols():
    """Names the header declares (used by the CPU-side ABI test)."""
    return sorted(_SIGNATURES)


def load():
    """Load libb200bt.so (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU or PyTorch fallback for this engine)")
    lib = C.CDLL(str(LIB_PATH), mode=getattr(os, "RTLD_NOW", 2))
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.b200bt_abi_version() != 1:
        raise ImportError("libb200bt.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def call(name: str, *args):
    lib = load()
    status = getattr(lib, name)(*args)
    if status != 0:
        raise B200btError(name, status, lib.b200bt_last_error().decode("utf-8", "replace"))


def launch_count() -> int:
    return int(load().b200bt_launch_count())


def ptr(t) -> int:
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def ld(t) -> int:
    """Row stride (in elements) of the last-but-one axis; a size-1 axis may carry any stride."""
    return int(t.stride(-2)) if t.shape[-2] > 1 else int(t.shape[-1])


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
