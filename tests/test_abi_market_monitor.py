"""CPU-side checks of b200bt_market_monitor / b200bt_indicator_combinations (csrc/market_monitor.cu): every argument
refusal, which happens before the device is touched (so these run without a GPU; the dummy device pointers are never
dereferenced)."""
import ctypes as C

import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status


def _bars(N, minute0, k):
    from ai_crypto_trader_b200 import _lib
    return int(_lib.load().b200bt_resample_bars(N, minute0, 1, k))


def _mm(S=2, N=10_000, minute0=28_401_127, bar_minutes=1, M=None, ohlcv=DEV, k3=DEV, k5=DEV, k15=DEV, params=None,
        rows=DEV, labels=None, **kw):
    from ai_crypto_trader_b200 import market_monitor as mm
    p = mm.monitor_params(**kw) if params is None else params
    M3, M5, M15 = M or tuple(_bars(N, max(minute0, 0), k) for k in (3, 5, 15))
    return status("b200bt_market_monitor", ohlcv, S, N, minute0, bar_minutes, k3, M3, k5, M5, k15, M15,
                  C.byref(p) if p is not False else None, rows, labels, None)


def test_market_monitor_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    assert _mm() == ENODEVICE                                            # every check passed
    assert _mm(rows=None, labels=DEV) == ENODEVICE
    assert _mm(rows=None) == EINVAL                                      # no output
    for null in ("ohlcv", "k3", "k5", "k15"):
        assert _mm(**{null: None}) == EINVAL, null
    assert _mm(params=False) == EINVAL
    assert _mm(S=0) == EINVAL and _mm(N=0, M=(1, 1, 1)) == EINVAL
    assert _mm(bar_minutes=3) == EINVAL and _mm(bar_minutes=0) == EINVAL
    assert _mm(minute0=-1, M=(3334, 2001, 667)) == EINVAL
    good = tuple(_bars(10_000, 28_401_127, k) for k in (3, 5, 15))
    for i in range(3):
        bad = list(good)
        bad[i] += 1
        assert _mm(M=tuple(bad)) == EINVAL, i
    assert _mm(frame_bars=0) == EINVAL and _mm(frame_bars=-1) == EINVAL
    assert _mm(frame_bars=1) == ENODEVICE and _mm(frame_bars=100_000) == ENODEVICE
    assert _mm(label_field=-1) == EINVAL and _mm(label_field=9) == EINVAL and _mm(label_field=8) == ENODEVICE
    assert _mm(N=1 << 30) == ELIMIT
    assert _mm(S=65_536) == ELIMIT


def test_indicator_combinations_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    assert status("b200bt_indicator_combinations", DEV, 5, None) == ENODEVICE
    assert status("b200bt_indicator_combinations", None, 5, None) == EINVAL
    assert status("b200bt_indicator_combinations", DEV, 0, None) == EINVAL
    assert status("b200bt_indicator_combinations", DEV, 1 << 31, None) == ELIMIT
