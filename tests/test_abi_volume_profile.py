"""CPU-side checks of b200bt_volume_profile (csrc/volume_profile.cu): the name tuples and every argument refusal, which
happens before the device is touched (so these run without a GPU; the dummy device pointers are never dereferenced)."""
import ctypes as C

import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status


def _vp(params=None, ohlcv=DEV, ld=10_000, S=2, N=10_000, rows=DEV, bins=None, labels=None, ld_rows=10_000, **kw):
    from ai_crypto_trader_b200 import volume_profile as vp
    p = vp.vp_params(**dict(dict(frame_bars=100), **kw)) if params is None else params
    return status("b200bt_volume_profile", ohlcv, ld, S, N, C.byref(p) if p is not False else None, rows, bins,
                  labels, ld_rows, None)


def test_struct_layouts(native_lib):
    """The row's codes and their name tuples (the struct layouts are checked against the header in
    tests/test_abi_header.py)."""
    from ai_crypto_trader_b200 import _lib
    assert _lib.VP_MAX_BINS >= 64 and _lib.VP_NO_LABEL == 255
    assert len(_lib.VP_SIGNALS) == 6 and _lib.VP_SIGNALS[-1] == "neutral"
    assert len(_lib.VP_POC_CODES) == 4 and len(_lib.VP_VALUE_AREA_CODES) == 7
    assert len(_lib.VP_PRESSURES) == 5 and len(_lib.VP_DIVERGENCES) == 3


def test_volume_profile_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    from ai_crypto_trader_b200 import _lib
    assert _vp() == ENODEVICE                                            # every check passed
    assert _vp(rows=None, labels=DEV) == ENODEVICE
    assert _vp(rows=None, bins=DEV) == ENODEVICE
    assert _vp(rows=None) == EINVAL                                     # no output
    assert _vp(ohlcv=None) == EINVAL
    assert _vp(params=False) == EINVAL
    assert _vp(ld=9_999) == EINVAL
    assert _vp(ld_rows=9_999) == EINVAL
    assert _vp(S=0) == EINVAL and _vp(N=0) == EINVAL
    assert _vp(N=1 << 30, ld=1 << 30, ld_rows=1 << 30) == ELIMIT
    assert _vp(S=65_536) == ELIMIT
    assert _vp(frame_bars=0) == EINVAL and _vp(frame_bars=-3) == EINVAL
    assert _vp(frame_bars=1) == ENODEVICE and _vp(frame_bars=20_000) == ENODEVICE    # longer than the series: no frame
    assert _vp(num_bins=0) == EINVAL
    assert _vp(num_bins=1) == ENODEVICE and _vp(num_bins=_lib.VP_MAX_BINS) == ENODEVICE
    assert _vp(num_bins=_lib.VP_MAX_BINS + 1) == ELIMIT
    assert _vp(anomaly_window=1) == EINVAL and _vp(anomaly_window=2) == ENODEVICE
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert _vp(value_area_pct=bad) == EINVAL
        assert _vp(std_threshold=bad) == EINVAL
