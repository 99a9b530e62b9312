"""CPU-side checks of b200bt_volume_profile (csrc/volume_profile.cu): struct layouts, the name tuples, and every argument
refusal, which happens before the device is touched (so these run without a GPU; the dummy device pointers are never
dereferenced)."""
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


def _vp(params=None, ohlcv=DEV, ld=10_000, S=2, N=10_000, rows=DEV, bins=None, labels=None, ld_rows=10_000, **kw):
    from ai_crypto_trader_b200 import volume_profile as vp
    p = vp.vp_params(**dict(dict(frame_bars=100), **kw)) if params is None else params
    return _status("b200bt_volume_profile", ohlcv, ld, S, N, C.byref(p) if p is not False else None, rows, bins,
                   labels, ld_rows, None)


def test_struct_layouts(native_lib):
    from ai_crypto_trader_b200 import _lib
    assert C.sizeof(_lib.VpParams) == 32
    row = np.dtype(_lib.VP_ROW_DTYPE)
    assert row.itemsize == 384
    assert row.fields["price_min"][1] == 120 and row.fields["recent_significance"][1] == 384 - 40
    assert re.search(r"#define B200BT_VP_MAX_BINS (\d+)", HEADER).group(1) == str(_lib.VP_MAX_BINS)
    assert _lib.VP_MAX_BINS >= 64 and _lib.VP_NO_LABEL == 255
    assert len(_lib.VP_SIGNALS) == 6 and _lib.VP_SIGNALS[-1] == "neutral"
    assert len(_lib.VP_POC_CODES) == 4 and len(_lib.VP_VALUE_AREA_CODES) == 7
    assert len(_lib.VP_PRESSURES) == 5 and len(_lib.VP_DIVERGENCES) == 3


def test_header_row_fields_match_dtype(native_lib):
    """The header's b200bt_vp_row declares the dtype's fields in the dtype's order."""
    from ai_crypto_trader_b200 import _lib
    body = HEADER[HEADER.index("typedef struct b200bt_vp_row {"):HEADER.index("} b200bt_vp_row;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in re.findall(r"(?:int32_t|double)\s+([^;]+);", body):
        names += [n.strip().split("[")[0] for n in decl.split(",")]
    assert names == [f[0] for f in _lib.VP_ROW_DTYPE]


def test_volume_profile_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    from ai_crypto_trader_b200 import _lib
    assert _vp() == _ENODEVICE                                            # every check passed
    assert _vp(rows=None, labels=DEV) == _ENODEVICE
    assert _vp(rows=None, bins=DEV) == _ENODEVICE
    assert _vp(rows=None) == _EINVAL                                     # no output
    assert _vp(ohlcv=None) == _EINVAL
    assert _vp(params=False) == _EINVAL
    assert _vp(ld=9_999) == _EINVAL
    assert _vp(ld_rows=9_999) == _EINVAL
    assert _vp(S=0) == _EINVAL and _vp(N=0) == _EINVAL
    assert _vp(N=1 << 30, ld=1 << 30, ld_rows=1 << 30) == _ELIMIT
    assert _vp(S=65_536) == _ELIMIT
    assert _vp(frame_bars=0) == _EINVAL and _vp(frame_bars=-3) == _EINVAL
    assert _vp(frame_bars=1) == _ENODEVICE and _vp(frame_bars=20_000) == _ENODEVICE    # longer than the series: no frame
    assert _vp(num_bins=0) == _EINVAL
    assert _vp(num_bins=1) == _ENODEVICE and _vp(num_bins=_lib.VP_MAX_BINS) == _ENODEVICE
    assert _vp(num_bins=_lib.VP_MAX_BINS + 1) == _ELIMIT
    assert _vp(anomaly_window=1) == _EINVAL and _vp(anomaly_window=2) == _ENODEVICE
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert _vp(value_area_pct=bad) == _EINVAL
        assert _vp(std_threshold=bad) == _EINVAL
