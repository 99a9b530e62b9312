"""CPU-side checks of the DCA entry points (csrc/dca.cu): workspace sizing and every argument refusal, which happens
before the device is touched (so these run without a GPU; the dummy device pointers are never dereferenced)."""
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

M0 = 28_401_120


def _ws(S=2, N=10_000):
    from ai_crypto_trader_b200 import _lib
    return int(_lib.load().b200bt_dca_workspace_bytes(S, N))


def _sweep(close=DEV, ld=10_000, dip=DEV, ld_dip=10_000, S=2, N=10_000, start_bar=100, bar_minutes=1, minute0=M0, ws=DEV,
           ws_bytes=None, indiv=DEV, first=DEV, pop=4, reb=1, target=DEV, pow10=DEV, labels=None, ld_labels=0, usdc=0.0,
           stats=DEV, service=None, day=None, D=0):
    if ws_bytes is None:
        ws_bytes = _ws(S, N)
    return status("b200bt_dca_sweep", close, ld, dip, ld_dip, S, N, start_bar, bar_minutes, minute0, ws, ws_bytes, indiv,
                  first, pop, reb, target, pow10, labels, ld_labels, usdc, stats, service, day, D, None)


def _dip(high=DEV, close=DEV, ld=10_000, S=2, N=10_000, minute0=M0, bar_minutes=1, out=DEV, ld_out=10_000):
    return status("b200bt_dca_dip_pct", high, close, ld, S, N, minute0, bar_minutes, out, ld_out, None)


def test_workspace_bytes(native_lib):
    from ai_crypto_trader_b200 import _lib
    f = _lib.load().b200bt_dca_workspace_bytes
    even = lambda n: (n + 1) & ~1
    for S, N in ((1, 1), (3, 1000), (10, 1_000_000)):
        want = S * 8 * sum(even(-(-N // 32 ** l)) for l in (1, 2, 3))
        assert f(S, N) == want
    assert f(0, 10) == 0 and f(1, 0) == 0


def test_dca_refusals(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")
    days = (M0 + 9_999) // 1440 - M0 // 1440 + 1
    assert _sweep() == ENODEVICE                                         # every check passed
    assert _sweep(labels=DEV, ld_labels=0) == ENODEVICE and _sweep(labels=DEV, ld_labels=10_000) == ENODEVICE
    assert _sweep(day=DEV, D=days, service=DEV) == ENODEVICE
    assert _sweep(start_bar=0) == ENODEVICE and _sweep(start_bar=9_999) == ENODEVICE
    for kw in ({"close": None}, {"dip": None}, {"ws": None}, {"indiv": None}, {"first": None}, {"target": None},
               {"pow10": None}, {"stats": None}):
        assert _sweep(**kw) == EINVAL, kw
    assert _sweep(S=0) == EINVAL
    assert _sweep(pop=0) == EINVAL
    assert _sweep(N=0) == EINVAL
    assert _sweep(ld=9_999) == EINVAL and _sweep(ld_dip=9_999) == EINVAL
    assert _sweep(start_bar=-1) == EINVAL and _sweep(start_bar=10_000) == EINVAL
    assert _sweep(bar_minutes=0) == EINVAL and _sweep(minute0=-1) == EINVAL
    assert _sweep(bar_minutes=1 << 26, ws_bytes=_ws()) == EINVAL                     # the clock in us overflows
    assert _sweep(labels=DEV, ld_labels=9_999) == EINVAL
    assert _sweep(day=DEV, D=days - 1) == EINVAL
    assert _sweep(ws_bytes=_ws() - 1) == EINVAL
    assert _sweep(N=1 << 30, ld=1 << 30, ld_dip=1 << 30, ws_bytes=1 << 40) == ELIMIT
    # S > 32: refused with rebalancing or day rows, accepted without
    assert _sweep(S=33, reb=1) == ELIMIT
    assert _sweep(S=33, reb=0, day=DEV, D=days) == ELIMIT
    assert _sweep(S=33, reb=0) == ENODEVICE
    assert _sweep(S=32, reb=1, day=DEV, D=days) == ENODEVICE
    # the drop series
    assert _dip() == ENODEVICE
    for kw in ({"high": None}, {"close": None}, {"out": None}, {"S": 0}, {"N": 0}, {"ld": 9_999}, {"ld_out": 9_999},
               {"bar_minutes": 0}, {"minute0": -1}):
        assert _dip(**kw) == EINVAL, kw
    assert _dip(N=1 << 30, ld=1 << 30, ld_out=1 << 30) == ELIMIT
