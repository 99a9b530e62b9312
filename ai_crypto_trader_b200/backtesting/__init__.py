"""Drop-in for the reference's `backtesting` package (run_backtest.py:11:
`from backtesting import BacktestEngine, ResultAnalyzer`)."""
import sys as _sys

from . import backtest_engine, data_manager, result_analyzer, strategy_tester
from .backtest_engine import BacktestEngine
from .data_manager import HistoricalDataManager
from .result_analyzer import ResultAnalyzer
from .strategy_tester import StrategyTester

__all__ = ["BacktestEngine", "HistoricalDataManager", "ResultAnalyzer", "StrategyTester", "install_as_backtesting"]


def install_as_backtesting() -> None:
    """Make `import backtesting` (and `backtesting.data_manager`, ... as run_backtest.py:11-12 imports them) resolve to
    this package, so that the reference's CLI runs unmodified on the H100 path:

        import ai_crypto_trader_b200.backtesting as b; b.install_as_backtesting(); runpy.run_path("run_backtest.py")
    """
    me = _sys.modules[__name__]
    _sys.modules["backtesting"] = me
    for name in ("backtest_engine", "data_manager", "result_analyzer", "strategy_tester"):
        _sys.modules[f"backtesting.{name}"] = getattr(me, name)
