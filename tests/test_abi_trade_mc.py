"""Status codes of the trade-sequence Monte-Carlo entry points: argument checks come before the device check, so EINVAL
and ELIMIT are exercised with or without a GPU; ENODEVICE without one."""
import ctypes as C

import pytest

from abi_header import EINVAL, ELIMIT, ENODEVICE, status


def _mc(T=4, L=1, block_len=1, n_paths=8, method=0, trips=True, counts=True, fees=True, out=True, ld=None, capital=1e4):
    buf = (C.c_double * 64)()
    res = (C.c_float * 64)()
    nt = (C.c_int32 * L)(*[T] * L)
    fee = (C.c_double * L)(*[1.0] * L)
    return ("b200bt_trade_mc", C.addressof(buf) if trips else None, ld if ld is not None else max(T, 1),
            nt if counts else None, fee if fees else None, None, L, method, block_len, capital, n_paths, 1, 0,
            C.addressof(res) if out else None, C.addressof(res), None)


def _pnl(S=1, pop=1, N=16, ld=None, event_cap=4, ld_trip=2, events=True):
    buf = (C.c_double * 64)()
    return ("b200bt_trade_pnl", C.addressof(buf), ld if ld is not None else N, S, N, C.addressof(buf), pop,
            C.addressof(buf), C.addressof(buf) if events else None, event_cap, C.addressof(buf), ld_trip,
            C.addressof(buf), C.addressof(buf), None)


def test_trade_mc_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    assert status(*_mc()) == ENODEVICE
    assert status(*_mc(method=1)) == ENODEVICE
    assert status(*_pnl()) == ENODEVICE


def test_trade_mc_validates_arguments(native_lib):
    assert status(*_mc(trips=False)) == EINVAL
    assert status(*_mc(counts=False)) == EINVAL
    assert status(*_mc(fees=False)) == EINVAL
    assert status(*_mc(out=False)) == EINVAL
    assert status(*_mc(L=0)) == EINVAL
    assert status(*_mc(method=2)) == EINVAL
    assert status(*_mc(block_len=0)) == EINVAL
    assert status(*_mc(n_paths=0)) == EINVAL
    assert status(*_mc(T=-1)) == EINVAL
    assert status(*_mc(T=5, ld=4)) == EINVAL                # more trips than the row stride holds
    assert status(*_mc(capital=0.0)) == EINVAL


def test_trade_mc_limits(native_lib):
    assert status(*_mc(T=1 << 30, ld=1 << 30)) == ELIMIT
    assert status(*_mc(n_paths=(1 << 38) + 1)) == ELIMIT


def test_trade_pnl_validates_arguments(native_lib):
    assert status(*_pnl(S=0)) == EINVAL
    assert status(*_pnl(pop=0)) == EINVAL
    assert status(*_pnl(ld=8)) == EINVAL                    # row stride below N
    assert status(*_pnl(events=False)) == EINVAL
    assert status(*_pnl(event_cap=6, ld_trip=2)) == EINVAL  # event_cap / 2 trips do not fit a row
    assert status(*_pnl(N=1 << 30, ld=1 << 30)) == ELIMIT
