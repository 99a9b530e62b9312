"""CPU-side checks of the walk-forward entry points (csrc/walk_forward.cu): every argument refusal, which happens before the
device is touched (so these run without a GPU; the dummy device pointers are never dereferenced), and their header
declarations."""
import ctypes as C

import pytest

import abi_header
from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

M0 = 28_401_120


def _cfg(**kw):
    from ai_crypto_trader_b200 import _lib
    c = _lib.SweepConfig(initial_capital=10000.0, minute0=M0, bar_minutes=1, primary=0, secondary_mask=7, variant=0)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _segments(price=DEV, ld_price=10_000, rsi=DEV, ld_rsi=10_000, P=26, S=2, N=10_000, indiv=DEV, n_indiv=4,
              segments=DEV, seg_begin=DEV, J=3, cfg=None, stats=DEV, events=None, event_cap=0):
    cfg = _cfg() if cfg is None else cfg
    return status("b200bt_sweep_segments", price, ld_price, rsi, ld_rsi, P, S, N, indiv, n_indiv, segments, seg_begin, J,
                  C.byref(cfg), stats, events, event_cap, None)


def _decode(params=DEV, ld=18, n=20, cols=(0, 2, 1, 17, 16, -1), table=None, n_table=None, out=DEV):
    table = list(range(-1, 30)) if table is None else table
    n_table = len(table) if n_table is None else n_table
    cols_arr = None if cols is None else (C.c_int * 6)(*cols)
    tab = (C.c_int32 * max(1, len(table)))(*table)
    return status("b200bt_decode_individuals", params, ld, n, cols_arr, tab, n_table, out, None)


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the accepted call would run")


def test_sweep_segments_refusals(native_lib):
    _no_gpu()
    assert _segments() == ENODEVICE                                     # every check passed
    assert _segments(events=DEV, event_cap=64) == ENODEVICE
    assert _segments(ld_price=10_001, ld_rsi=10_003) == ENODEVICE
    for kw in ({"price": None}, {"rsi": None}, {"indiv": None}, {"segments": None}, {"seg_begin": None},
               {"stats": None}):
        assert _segments(**kw) == EINVAL, kw
    assert _segments(n_indiv=0) == EINVAL
    assert _segments(J=0) == EINVAL
    assert _segments(S=0) == EINVAL
    assert _segments(P=0) == EINVAL
    assert _segments(N=0) == EINVAL
    assert _segments(ld_price=9_999) == EINVAL
    assert _segments(ld_rsi=9_999) == EINVAL
    assert _segments(events=DEV, event_cap=0) == EINVAL
    assert _segments(N=1 << 30, ld_price=1 << 30, ld_rsi=1 << 30) == ELIMIT
    # the calendar clock, as the sweeps check it
    assert _segments(cfg=_cfg(bar_minutes=0)) == EINVAL
    assert _segments(cfg=_cfg(minute0=-1)) == EINVAL
    assert _segments(cfg=_cfg(minute0=(1 << 32) - 1440 - 10_000)) == ELIMIT
    assert _segments(cfg=_cfg(minute0=(1 << 32) - 1441 - 10_000)) == ENODEVICE
    # a glued series is not combined with segments
    assert _segments(cfg=_cfg(gap_bar=5_000)) == EINVAL
    assert _segments(cfg=_cfg(gap_minutes=60)) == ENODEVICE             # no gap bar: the minutes are never added


def test_decode_individuals_refusals(native_lib):
    _no_gpu()
    assert _decode() == ENODEVICE
    assert _decode(cols=(-1,) * 6) == ENODEVICE
    assert _decode(table=[0] * 256) == ENODEVICE
    for kw in ({"params": None}, {"cols": None}, {"out": None}):
        assert _decode(**kw) == EINVAL, kw
    assert status("b200bt_decode_individuals", DEV, 18, 20, (C.c_int * 6)(0, 1, 2, 3, 4, 5), None, 31, DEV, None) == EINVAL
    assert _decode(n=0) == EINVAL
    assert _decode(ld=0) == EINVAL
    assert _decode(n_table=0) == EINVAL
    assert _decode(table=[0] * 257) == ELIMIT
    assert _decode(cols=(18, 2, 1, 17, 16, -1)) == EINVAL               # column outside [-1, ld)
    assert _decode(cols=(0, -2, 1, 17, 16, -1)) == EINVAL
    assert _decode(ld=6, cols=(0, 1, 2, 3, 4, 5)) == ENODEVICE


def test_header_declares_both_entries():
    header = abi_header.parse()
    ret, params = header.prototypes["b200bt_sweep_segments"]
    assert ret == abi_header.CType("int")
    assert params[9] == abi_header.CType("int64_t", 1) and params[10] == abi_header.CType("int32_t", 1)
    assert params[7] == abi_header.CType("b200bt_individual", 1)
    ret, params = header.prototypes["b200bt_decode_individuals"]
    assert ret == abi_header.CType("int")
    assert params[0] == abi_header.CType("double", 1) and params[6] == abi_header.CType("b200bt_individual", 1)


def test_segment_record_mirror_matches_header():
    """The 24-byte segment record: the header's B200BT_SEGMENT_* offsets against _lib.SEGMENT_DTYPE, the dtype the
    driver builds its tables with."""
    import numpy as np
    from ai_crypto_trader_b200 import _lib, walk_forward
    d = abi_header.parse().defines
    dt = np.dtype(_lib.SEGMENT_DTYPE)
    assert dt.itemsize == d["B200BT_SEGMENT_BYTES"] == 24
    want = {"start": ("<i8", "B200BT_SEGMENT_START"), "end": ("<i8", "B200BT_SEGMENT_END"),
            "individual": ("<i4", "B200BT_SEGMENT_INDIVIDUAL"), "reserved": ("<i4", "B200BT_SEGMENT_RESERVED")}
    assert list(dt.names) == list(want)
    for name, (kind, macro) in want.items():
        assert dt.fields[name][0] == np.dtype(kind) and dt.fields[name][1] == d[macro], name
    seg, _ = walk_forward.segment_tables([[(3, 9, 1)], [(0, 4, 0), (4, 8, 2)]])
    assert seg.dtype == dt and seg.tolist() == [(3, 9, 1, 0), (0, 4, 0, 0), (4, 8, 2, 0)]
