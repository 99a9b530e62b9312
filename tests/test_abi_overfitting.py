"""Status codes of the backtest-overfitting entry points (b200bt_daily_pnl, b200bt_cscv): argument checks come before
the device check, so EINVAL and ELIMIT are exercised with or without a GPU; ENODEVICE without one."""
import ctypes as C

import pytest

from abi_header import EINVAL, ELIMIT, ENODEVICE, status

MINUTE0 = 1440 * 19_000 + 600


def _cfg(minute0=MINUTE0, bar_minutes=1, gap_bar=0, gap_minutes=0):
    from ai_crypto_trader_b200 import _lib
    return _lib.SweepConfig(initial_capital=1e4, minute0=minute0, bar_minutes=bar_minutes, primary=0, secondary_mask=0,
                            variant=0, gap_bar=gap_bar, gap_minutes=gap_minutes)


def _daily(S=1, pop=1, N=2000, ld=None, D=4, events=True, event_cap=4, out=True, cfg=None):
    buf = (C.c_double * 64)()
    dev = C.addressof(buf)
    return ("b200bt_daily_pnl", dev, ld if ld is not None else N, S, N, dev, pop, C.byref(cfg or _cfg()), dev,
            dev if events else None, event_cap, dev if out else None, D, None, None)


def _cscv(N=4, T=40, B=4, ld=None, ws=True, ws_bytes=None, out=True):
    from ai_crypto_trader_b200 import _lib
    buf = (C.c_double * 64)()
    dev = C.addressof(buf)
    need = int(_lib.load().b200bt_cscv_workspace_bytes(N, T, B))
    return ("b200bt_cscv", dev, ld if ld is not None else T, N, T, B, dev if ws else None,
            need if ws_bytes is None else ws_bytes, dev if out else None, dev, dev, dev, dev, dev, dev, dev, dev, dev, None)


def test_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    # 2000 one-minute bars from 10:00 end on the next calendar day: D = 2 columns cover them
    assert status(*_daily(D=2)) == ENODEVICE
    assert status(*_cscv()) == ENODEVICE


def test_daily_pnl_validates_arguments(native_lib):
    assert status(*_daily(S=0)) == EINVAL
    assert status(*_daily(pop=0)) == EINVAL
    assert status(*_daily(ld=100)) == EINVAL                    # row stride below N
    assert status(*_daily(events=False)) == EINVAL
    assert status(*_daily(out=False)) == EINVAL
    assert status(*_daily(D=1)) == EINVAL                       # the series spans two calendar days
    assert status(*_daily(D=5, cfg=_cfg(gap_bar=10, gap_minutes=4 * 1440))) == EINVAL    # the gap adds four more
    assert status(*_daily(N=1 << 30, ld=1 << 30, D=1 << 20)) == ELIMIT
    assert status(*_daily(cfg=_cfg(bar_minutes=0))) == EINVAL   # the sweeps' clock check
    assert status(*_daily(cfg=_cfg(minute0=-1))) == EINVAL
    assert status(*_daily(cfg=_cfg(minute0=(1 << 32) - 1440))) == ELIMIT


def test_cscv_validates_arguments(native_lib):
    from ai_crypto_trader_b200 import _lib
    lib = _lib.load()
    assert status(*_cscv(B=3)) == EINVAL                        # odd
    assert status(*_cscv(B=0)) == EINVAL
    assert status(*_cscv(B=22, T=440)) == ELIMIT                # more than 20 blocks
    assert status(*_cscv(T=7, B=4)) == EINVAL                   # L = 1
    assert status(*_cscv(N=1)) == EINVAL
    assert status(*_cscv(ws=False)) == EINVAL
    assert status(*_cscv(out=False)) == EINVAL
    assert status(*_cscv(ld=30)) == EINVAL                      # row stride below T
    assert status(*_cscv(ws_bytes=8)) == EINVAL                 # workspace too small
    for args in ((4, 7, 4), (1, 40, 4), (4, 40, 3), (4, 440, 22)):
        assert lib.b200bt_cscv_workspace_bytes(*args) == 0, args
    assert lib.b200bt_cscv_workspace_bytes(1000, 700, 16) >= 2 * 16 * 1000 * 8 + 12870 * 4 * 12
