"""CPU-side checks of the grid-trading entry point (csrc/grid.cu): every argument refusal, which happens before the
device is touched (so these run without a GPU; the dummy device pointers are never dereferenced)."""
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

M0 = 28_401_120


def _table(n=15):
    from ai_crypto_trader_b200 import _lib
    t = (_lib.GridRegimeRule * 5)()
    t[2] = _lib.GridRegimeRule(1, n, 3.0, 3.0)
    return t


def _grid(price=DEV, ld=10_000, S=2, N=10_000, start_bar=100, bar_minutes=1, minute0=M0, indiv=DEV, pop=4, qty=DEV,
          bounds=DEV, labels=None, ld_labels=0, table=None, stats=DEV, day=None, D=0):
    return status("b200bt_grid_sweep", price, ld, S, N, start_bar, bar_minutes, minute0, indiv, pop, qty, bounds, labels,
                  ld_labels, table, stats, day, D, None)


def test_grid_sweep_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    days = (M0 + 9_999) // 1440 - M0 // 1440 + 1
    assert _grid() == ENODEVICE                                         # every check passed
    assert _grid(labels=DEV, ld_labels=0, table=_table()) == ENODEVICE
    assert _grid(labels=DEV, ld_labels=10_000) == ENODEVICE
    assert _grid(day=DEV, D=days) == ENODEVICE
    assert _grid(start_bar=0) == ENODEVICE and _grid(start_bar=9_999) == ENODEVICE
    for kw in ({"price": None}, {"indiv": None}, {"qty": None}, {"bounds": None}, {"stats": None}):
        assert _grid(**kw) == EINVAL, kw
    assert _grid(S=0) == EINVAL
    assert _grid(pop=0) == EINVAL
    assert _grid(N=0) == EINVAL
    assert _grid(ld=9_999) == EINVAL
    assert _grid(start_bar=-1) == EINVAL
    assert _grid(start_bar=10_000) == EINVAL
    assert _grid(bar_minutes=0) == EINVAL
    assert _grid(minute0=-1) == EINVAL
    assert _grid(labels=DEV, ld_labels=9_999) == EINVAL
    assert _grid(day=DEV, D=days - 1) == EINVAL
    assert _grid(table=_table(0)) == EINVAL
    assert _grid(table=_table(128)) == EINVAL
    assert _grid(table=_table(127)) == ENODEVICE
    assert _grid(N=1 << 30, ld=1 << 30) == ELIMIT
