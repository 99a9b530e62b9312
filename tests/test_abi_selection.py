"""CPU-side checks of the strategy selection entry points (csrc/selection.cu): every argument refusal, which happens before
the device is touched (so these run without a GPU; the dummy device pointers are never dereferenced), and the header's slot
and column macros against their _lib names."""
import ctypes as C

import pytest

import abi_header
from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

M0 = 28_401_120


def _params(**kw):
    from ai_crypto_trader_b200 import _lib
    vals = dict(start_bar=0, check_bars=5, cache_expiry=3600, w_market_regime=0.3, w_historical_performance=0.25,
                w_risk_profile=0.15, w_social_sentiment=0.15, w_market_volatility=0.1, w_feature_importance=0.05,
                min_improvement=0.15, min_confidence=0.7, risk_max_drawdown=0.1, risk_min_sharpe=1.2, risk_volatility=1,
                high_vol_start=14, high_vol_end=22, low_activity_start=0, low_activity_end=8)
    vals.update(kw)
    return (C.c_double * len(_lib.SEL_PARAMS))(*[float(vals[n]) for n in _lib.SEL_PARAMS])


def _replay(price=DEV, ld_price=10_000, S=2, N=10_000, indiv=DEV, n_indiv=4, cfg="ok", stats=DEV, events=DEV,
            event_cap=64, labels=DEV, ld_labels=0, cand_row=DEV, cand_index=DEV, genes=DEV, n_cand=4, K=4, params=None,
            n_checks=2000, merge=0, rows=DEV, scores=None, locks=DEV):
    from ai_crypto_trader_b200 import _lib
    c = _lib.SweepConfig(initial_capital=10000.0, minute0=M0, bar_minutes=1, primary=0, secondary_mask=7, variant=0)
    return status("b200bt_selection_replay", price, ld_price, S, N, indiv, n_indiv, None if cfg is None else C.byref(c),
                  stats, events, event_cap, labels, ld_labels, cand_row, cand_index, genes, n_cand, K,
                  _params() if params is None else params, n_checks, merge, rows, scores, locks, None)


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")


def test_selection_replay_refusals(native_lib):
    _no_gpu()
    assert _replay() == ENODEVICE                                       # every check passed
    assert _replay(scores=DEV, merge=1, ld_labels=10_000, n_cand=2) == ENODEVICE
    assert _replay(params=_params(start_bar=9_999), n_checks=1) == ENODEVICE
    assert _replay(params=_params(check_bars=10_000), n_checks=1) == ENODEVICE
    for kw in ({"price": None}, {"indiv": None}, {"cfg": None}, {"stats": None}, {"events": None}, {"labels": None},
               {"cand_row": None}, {"cand_index": None}, {"genes": None}, {"rows": None}, {"locks": None}):
        assert _replay(**kw) == EINVAL, kw
    for kw in ({"event_cap": 0}, {"ld_labels": 9_999}, {"n_cand": 0}, {"K": 3}, {"merge": 2}, {"n_checks": 0},
               {"n_checks": 2001}, {"ld_price": 9_999}, {"n_indiv": 0},
               {"params": _params(check_bars=0)}, {"params": _params(check_bars=2.5)},
               {"params": _params(check_bars=10_001)}, {"params": _params(check_bars=1e300)},
               {"params": _params(start_bar=-1)}, {"params": _params(start_bar=10_000)},
               {"params": _params(start_bar=1.5)}, {"params": _params(cache_expiry=0)},
               {"params": _params(cache_expiry=float("inf"))}, {"params": _params(risk_max_drawdown=0)},
               {"params": _params(risk_min_sharpe=0)}, {"params": _params(risk_volatility=3)},
               {"params": _params(high_vol_start=14.5)}):
        assert _replay(**kw) == EINVAL, kw
    assert _replay(S=65, n_cand=4) == ELIMIT
    assert _replay(N=1 << 30, ld_price=1 << 30) == ELIMIT


def test_selection_switch_refusals(native_lib):
    _no_gpu()
    p = _params()
    assert status("b200bt_selection_switch", DEV, 100, p, DEV, DEV, None) == ENODEVICE
    for args in ((None, 100, p, DEV, DEV), (DEV, 100, None, DEV, DEV), (DEV, 100, p, None, DEV), (DEV, 100, p, DEV, None),
                 (DEV, 0, p, DEV, DEV)):
        assert status("b200bt_selection_switch", *args, None) == EINVAL, args
    assert status("b200bt_selection_switch", DEV, 1 << 31, p, DEV, DEV, None) == ELIMIT


def test_slot_and_column_macros_match_lib():
    from ai_crypto_trader_b200 import _lib
    d = abi_header.parse().defines
    for prefix, names, count in (("B200BT_SEL_P_", _lib.SEL_PARAMS, "B200BT_SEL_PARAMS"),
                                 ("B200BT_SEL_G_", _lib.SEL_GENES, "B200BT_SEL_GENES"),
                                 ("B200BT_SEL_R_", _lib.SEL_ROW, "B200BT_SEL_ROW_WORDS")):
        assert {m: v for m, v in d.items() if m.startswith(prefix)} == {prefix + n.upper(): i for i, n in enumerate(names)}
        assert d[count] == len(names)
