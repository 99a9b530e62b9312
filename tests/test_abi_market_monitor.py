"""CPU-side checks of b200bt_market_monitor / b200bt_indicator_combinations (csrc/market_monitor.cu): struct layouts, the
name tuples, and every argument refusal, which happens before the device is touched (so these run without a GPU; the
dummy device pointers are never dereferenced)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

_EINVAL, _ENODEVICE, _ELIMIT = 10001, 10002, 10003
DEV = 1 << 20
HEADER = (Path(__file__).resolve().parents[1] / "include" / "b200bt.h").read_text()


def _status(fn, *args):
    from ai_crypto_trader_b200 import _lib
    try:
        _lib.call(fn, *args)
    except _lib.B200btError as e:
        return e.status
    return 0


def _bars(N, minute0, k):
    from ai_crypto_trader_b200 import _lib
    return int(_lib.load().b200bt_resample_bars(N, minute0, 1, k))


def _mm(S=2, N=10_000, minute0=28_401_127, bar_minutes=1, M=None, ohlcv=DEV, k3=DEV, k5=DEV, k15=DEV, params=None,
        rows=DEV, labels=None, **kw):
    from ai_crypto_trader_b200 import market_monitor as mm
    p = mm.monitor_params(**kw) if params is None else params
    M3, M5, M15 = M or tuple(_bars(N, max(minute0, 0), k) for k in (3, 5, 15))
    return _status("b200bt_market_monitor", ohlcv, S, N, minute0, bar_minutes, k3, M3, k5, M5, k15, M15,
                   C.byref(p) if p is not False else None, rows, labels, None)


def test_header_row_fields_match_dtype(native_lib):
    """The header's b200bt_monitor_row declares the dtype's fields in the dtype's order; sizes and constants agree."""
    from ai_crypto_trader_b200 import _lib
    body = HEADER[HEADER.index("typedef struct b200bt_monitor_row {"):HEADER.index("} b200bt_monitor_row;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in re.findall(r"(?:int32_t|double)\s+([^;]+);", body):
        names += [n.strip().split("[")[0] for n in decl.split(",")]
    assert names == [f[0] for f in _lib.MONITOR_ROW_DTYPE]
    assert np.dtype(_lib.MONITOR_ROW_DTYPE).itemsize == 352 and C.sizeof(_lib.MonitorParams) == 24
    for name in ("NO_LABEL", "LABEL_FIELDS", "COMBINATIONS"):
        want = getattr(_lib, "MM_" + name)
        assert int(re.search(rf"#define B200BT_MM_{name} (\d+)", HEADER).group(1)) == (want if name == "NO_LABEL" else len(want))
    for name, bit in _lib.MM_HAS.items():
        assert int(re.search(rf"#define B200BT_MM_HAS_{name.upper()} (\d+)", HEADER).group(1)) == bit


def test_market_monitor_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    assert _mm() == _ENODEVICE                                            # every check passed
    assert _mm(rows=None, labels=DEV) == _ENODEVICE
    assert _mm(rows=None) == _EINVAL                                      # no output
    for null in ("ohlcv", "k3", "k5", "k15"):
        assert _mm(**{null: None}) == _EINVAL, null
    assert _mm(params=False) == _EINVAL
    assert _mm(S=0) == _EINVAL and _mm(N=0, M=(1, 1, 1)) == _EINVAL
    assert _mm(bar_minutes=3) == _EINVAL and _mm(bar_minutes=0) == _EINVAL
    assert _mm(minute0=-1, M=(3334, 2001, 667)) == _EINVAL
    good = tuple(_bars(10_000, 28_401_127, k) for k in (3, 5, 15))
    for i in range(3):
        bad = list(good)
        bad[i] += 1
        assert _mm(M=tuple(bad)) == _EINVAL, i
    assert _mm(frame_bars=0) == _EINVAL and _mm(frame_bars=-1) == _EINVAL
    assert _mm(frame_bars=1) == _ENODEVICE and _mm(frame_bars=100_000) == _ENODEVICE
    assert _mm(label_field=-1) == _EINVAL and _mm(label_field=9) == _EINVAL and _mm(label_field=8) == _ENODEVICE
    assert _mm(N=1 << 30) == _ELIMIT
    assert _mm(S=65_536) == _ELIMIT


def test_indicator_combinations_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    assert _status("b200bt_indicator_combinations", DEV, 5, None) == _ENODEVICE
    assert _status("b200bt_indicator_combinations", None, 5, None) == _EINVAL
    assert _status("b200bt_indicator_combinations", DEV, 0, None) == _EINVAL
    assert _status("b200bt_indicator_combinations", DEV, 1 << 31, None) == _ELIMIT
