"""CPU-side checks of the market-regime entry points (csrc/regime.cu): the window bound and every argument refusal,
which happens before the device is touched (so these run without a GPU; the dummy device pointers are never
dereferenced)."""
import ctypes as C

import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status


def _params(sample_minutes=60):
    from ai_crypto_trader_b200 import regime
    return regime.regime_params(sample_minutes)


def _labels(params=None, close=DEV, S=2, N=10_000, ld=10_000, minute0=28_401_120, bar_minutes=1, labels=DEV,
            ld_labels=10_000, rows=None, max_windows=0):
    p = _params() if params is None else params
    return status("b200bt_regime_labels", close, DEV, DEV, DEV, S, N, ld, minute0, bar_minutes, C.byref(p), labels,
                  ld_labels, rows, max_windows, None)


def _classes(R=5, labels=DEV, ld_labels=10_000, N=10_000, class_stats=DEV, events=DEV, event_cap=64):
    from ai_crypto_trader_b200 import _lib
    cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=28_401_120, bar_minutes=1)
    return status("b200bt_class_stats", DEV, N, 2, N, DEV, 4, C.byref(cfg), DEV, events, event_cap, labels, ld_labels,
                  R, class_stats, None)


def test_window_bound(native_lib):
    mw = native_lib.b200bt_regime_max_windows
    assert mw(1, 1) == 1
    assert mw(1441, 1) == 2
    assert mw(1442, 1) == 3
    assert mw(1_000_000, 1) == (999_999 + 1439) // 1440 + 1
    assert mw(0, 1) == 0 and mw(10, 0) == 0


def test_regime_labels_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    assert _labels() == ENODEVICE                                     # every check passed
    assert _labels(close=None) == EINVAL
    assert _labels(labels=None) == EINVAL
    assert status("b200bt_regime_labels", DEV, DEV, DEV, DEV, 1, 100, 100, 0, 1, None, DEV, 100, None, 0, None) == EINVAL
    assert _labels(minute0=-1) == EINVAL                               # glued / negative clocks: refused
    assert _labels(params=_params(7)) == EINVAL                        # not a multiple of 5
    assert _labels(params=_params(0)) == EINVAL
    assert _labels(params=_params(-60)) == EINVAL
    assert _labels(params=_params(15), bar_minutes=10) == EINVAL       # not a multiple of bar_minutes
    assert _labels(params=_params(30), bar_minutes=10) == ENODEVICE
    assert _labels(params=_params(5), bar_minutes=5) == ENODEVICE
    assert _labels(bar_minutes=0) == EINVAL
    assert _labels(ld=9_999) == EINVAL
    assert _labels(ld_labels=9_999) == EINVAL
    assert _labels(S=1, ld_labels=0) == ENODEVICE                     # one symbol: any label stride
    assert _labels(N=1 << 30, ld=1 << 30, ld_labels=1 << 30) == ELIMIT
    assert _labels(rows=DEV, max_windows=7) == EINVAL                  # fewer rows than windows
    assert _labels(rows=DEV, max_windows=int(native_lib.b200bt_regime_max_windows(10_000, 1))) == ENODEVICE


def test_class_stats_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    for R in range(1, 9):
        assert _classes(R=R) == ENODEVICE
    assert _classes(R=0) == EINVAL
    assert _classes(R=-1) == EINVAL
    assert _classes(R=9) == ELIMIT
    assert _classes(labels=None) == EINVAL
    assert _classes(class_stats=None) == EINVAL
    assert _classes(events=None) == EINVAL
    assert _classes(events=None, event_cap=0) == ENODEVICE
    assert _classes(ld_labels=0) == ENODEVICE                         # one shared label row
    assert _classes(ld_labels=9_999) == EINVAL
    assert _classes(N=1 << 30, ld_labels=0) == ELIMIT
