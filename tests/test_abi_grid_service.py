"""CPU-side checks of b200bt_grid_service_sweep (csrc/grid.cu): every argument refusal, which happens before the device
is touched (so these run without a GPU; the dummy device pointers are never dereferenced)."""
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

M0 = 28_401_120


def _table(n=15):
    from ai_crypto_trader_b200 import _lib
    t = (_lib.GridRegimeRule * 5)()
    t[2] = _lib.GridRegimeRule(1, n, 3.0, 3.0)
    return t


def _svc(price=DEV, ld=10_000, S=3, N=10_000, start_bar=100, bar_minutes=1, minute0=M0, indiv=DEV, pop=4, qty=DEV,
         bounds=DEV, labels=None, ld_labels=0, table=None, stats=DEV, service=DEV, day=None, D=0):
    return status("b200bt_grid_service_sweep", price, ld, S, N, start_bar, bar_minutes, minute0, indiv, pop, qty, bounds,
                  labels, ld_labels, table, stats, service, day, D, None)


def test_grid_service_sweep_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    days = (M0 + 9_999) // 1440 - M0 // 1440 + 1
    assert _svc() == ENODEVICE                                          # every check passed
    assert _svc(service=None) == ENODEVICE                              # the service record is optional
    assert _svc(labels=DEV, ld_labels=0, table=_table()) == ENODEVICE
    assert _svc(day=DEV, D=days) == ENODEVICE
    assert _svc(S=40) == ENODEVICE and _svc(S=1) == ENODEVICE
    assert _svc(start_bar=0) == ENODEVICE and _svc(start_bar=9_999) == ENODEVICE
    for kw in ({"price": None}, {"indiv": None}, {"qty": None}, {"bounds": None}, {"stats": None}):
        assert _svc(**kw) == EINVAL, kw
    assert _svc(S=0) == EINVAL
    assert _svc(pop=0) == EINVAL
    assert _svc(N=0) == EINVAL
    assert _svc(ld=9_999) == EINVAL
    assert _svc(start_bar=-1) == EINVAL
    assert _svc(start_bar=10_000) == EINVAL
    assert _svc(bar_minutes=0) == EINVAL
    assert _svc(minute0=-1) == EINVAL
    assert _svc(labels=DEV, ld_labels=10_000) == EINVAL                 # per-symbol label rows: the service reads one
    assert _svc(labels=DEV, ld_labels=9_999) == EINVAL
    assert _svc(day=DEV, D=days - 1) == EINVAL
    assert _svc(table=_table(0)) == EINVAL
    assert _svc(table=_table(128)) == EINVAL
    assert _svc(table=_table(127)) == ENODEVICE
    assert _svc(N=1 << 30, ld=1 << 30) == ELIMIT
