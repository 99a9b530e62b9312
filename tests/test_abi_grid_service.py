"""CPU-side checks of b200bt_grid_service_sweep (csrc/grid.cu): the service record's layout and every argument refusal,
which happens before the device is touched (so these run without a GPU; the dummy device pointers are never
dereferenced)."""
import pytest

_EINVAL, _ENODEVICE, _ELIMIT = 10001, 10002, 10003
DEV = 1 << 20
M0 = 28_401_120


def _status(fn, *args):
    from ai_crypto_trader_b200 import _lib
    try:
        _lib.call(fn, *args)
    except _lib.B200btError as e:
        return e.status
    return 0


def _table(n=15):
    from ai_crypto_trader_b200 import _lib
    t = (_lib.GridRegimeRule * 5)()
    t[2] = _lib.GridRegimeRule(1, n, 3.0, 3.0)
    return t


def _svc(price=DEV, ld=10_000, S=3, N=10_000, start_bar=100, bar_minutes=1, minute0=M0, indiv=DEV, pop=4, qty=DEV,
         bounds=DEV, labels=None, ld_labels=0, table=None, stats=DEV, service=DEV, day=None, D=0):
    return _status("b200bt_grid_service_sweep", price, ld, S, N, start_bar, bar_minutes, minute0, indiv, pop, qty, bounds,
                   labels, ld_labels, table, stats, service, day, D, None)


def test_service_record_layout(native_lib):
    from ai_crypto_trader_b200 import _lib
    assert len(_lib.GRID_SERVICE_FIELDS) * 8 == 96
    assert _lib.GRID_SERVICE_FIELDS[:4] == ("total_profit", "total_trades", "profitable_trades", "win_rate")
    assert _lib.GRID_SERVICE_FIELDS[-1] == "max_num_grids"


def test_grid_service_sweep_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    days = (M0 + 9_999) // 1440 - M0 // 1440 + 1
    assert _svc() == _ENODEVICE                                          # every check passed
    assert _svc(service=None) == _ENODEVICE                              # the service record is optional
    assert _svc(labels=DEV, ld_labels=0, table=_table()) == _ENODEVICE
    assert _svc(day=DEV, D=days) == _ENODEVICE
    assert _svc(S=40) == _ENODEVICE and _svc(S=1) == _ENODEVICE
    assert _svc(start_bar=0) == _ENODEVICE and _svc(start_bar=9_999) == _ENODEVICE
    for kw in ({"price": None}, {"indiv": None}, {"qty": None}, {"bounds": None}, {"stats": None}):
        assert _svc(**kw) == _EINVAL, kw
    assert _svc(S=0) == _EINVAL
    assert _svc(pop=0) == _EINVAL
    assert _svc(N=0) == _EINVAL
    assert _svc(ld=9_999) == _EINVAL
    assert _svc(start_bar=-1) == _EINVAL
    assert _svc(start_bar=10_000) == _EINVAL
    assert _svc(bar_minutes=0) == _EINVAL
    assert _svc(minute0=-1) == _EINVAL
    assert _svc(labels=DEV, ld_labels=10_000) == _EINVAL                 # per-symbol label rows: the service reads one
    assert _svc(labels=DEV, ld_labels=9_999) == _EINVAL
    assert _svc(day=DEV, D=days - 1) == _EINVAL
    assert _svc(table=_table(0)) == _EINVAL
    assert _svc(table=_table(128)) == _EINVAL
    assert _svc(table=_table(127)) == _ENODEVICE
    assert _svc(N=1 << 30, ld=1 << 30) == _ELIMIT
