"""Status codes of the risk entry points (joint Monte-Carlo, bootstrap paths, order statistics, returns, tail sums and
correlation): argument checks come before the device check, so EINVAL and ELIMIT are exercised with or without a GPU;
ENODEVICE without one."""
import ctypes as C

import pytest

from abi_header import EINVAL, ELIMIT, ENODEVICE, status


def _d(*v):
    return (C.c_double * len(v))(*v)


def _gbm(S=2, s0=None, qty=None, chol=None, n_paths=8, steps=4, finals=True):
    buf = (C.c_float * 64)()
    out = C.addressof(buf) if finals else None
    s0 = s0 if s0 is not None else _d(*[1.0] * S)
    qty = qty if qty is not None else _d(*[1.0] * S)
    chol = chol if chol is not None else (C.c_float * (S * S))(*[1.0 if i % (S + 1) == 0 else 0.0 for i in range(S * S)])
    return ("b200bt_mc_portfolio_gbm", S, s0, qty, _d(*[0.0] * S), _d(*[0.01] * S), chol, n_paths, steps, 1, 0,
            out, out, None, None)


def _boot(S=2, R=16, block_len=1, returns=True, n_paths=8):
    buf = (C.c_float * 64)()
    return ("b200bt_mc_portfolio_bootstrap", S, C.addressof(buf) if returns else None, R, block_len, 1,
            _d(*[1.0] * S), _d(*[1.0] * S), n_paths, 4, 1, 0, C.addressof(buf), C.addressof(buf), None, None)


def test_portfolio_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    assert status(*_gbm()) == ENODEVICE
    assert status(*_boot()) == ENODEVICE


def test_portfolio_entry_points_validate_arguments(native_lib):
    assert status(*_gbm(S=0)) == EINVAL
    assert status(*_gbm(n_paths=0)) == EINVAL
    assert status(*_gbm(steps=-1)) == EINVAL
    assert status(*_gbm(finals=False)) == EINVAL
    assert status(*_gbm(s0=_d(1.0, 0.0))) == EINVAL                  # a price must be positive
    assert status(*_gbm(qty=_d(1.0, -1.0))) == EINVAL                # no short positions
    assert status(*_gbm(qty=_d(0.0, 0.0))) == EINVAL                 # V_0 = 0
    assert status(*_gbm(chol=(C.c_float * 4)(1.0, 0.0, float("nan"), 1.0))) == EINVAL
    assert status(*_boot(returns=False)) == EINVAL
    assert status(*_boot(R=0)) == EINVAL
    assert status(*_boot(block_len=0)) == EINVAL


def test_portfolio_entry_points_limits(native_lib):
    assert status(*_gbm(S=33)) == ELIMIT
    assert status(*_boot(S=33)) == ELIMIT
    assert status(*_boot(S=4, R=3073)) == ELIMIT                      # R x S > 12288 table entries


_BUF = (C.c_float * 64)()
_P = C.addressof(_BUF)           # any non-null pointer: the arguments are refused before anything is read


def test_risk_entry_points_validate_arguments(native_lib):
    lib = native_lib
    ws = int(lib.b200bt_correlation_workspace_bytes(4, 100))
    assert status(*("b200bt_correlation", _P, 100, 513, 100, _P, _P, 1 << 40, None)) == EINVAL      # S > 512
    assert status(*("b200bt_correlation", _P, 99, 4, 100, _P, _P, ws, None)) == EINVAL              # ld < N
    assert status(*("b200bt_correlation", _P, 100, 4, 100, _P, _P, ws - 8, None)) == EINVAL         # workspace
    need = int(lib.b200bt_select_workspace_bytes(3))
    assert status(*("b200bt_select", _P, 10, _P, 0, _P, _P, 1 << 40, None)) == EINVAL               # no rank
    assert status(*("b200bt_select", _P, 10, _P, 65, _P, _P, 1 << 40, None)) == EINVAL              # > 64 ranks
    assert status(*("b200bt_select", _P, 10, _P, 3, _P, _P, need - 1, None)) == EINVAL              # workspace
    assert status(*("b200bt_tail_stats", _P, 0, 0.0, _P, _P, 1 << 20, None)) == EINVAL              # empty input
    assert status(*("b200bt_pct_change", _P, 99, 2, 100, _P, 100, None)) == EINVAL                  # ld < N


def test_risk_entry_points_limits(native_lib):
    def boot(R):
        return ("b200bt_mc_bootstrap", _P, R, 1, 1, 100.0, 8, 4, 1, 0, _P, _P, None, None)
    assert status(*boot(12289)) == ELIMIT                                # more than 48 KB of table
    assert status(*("b200bt_pct_change", _P, 10, 65536, 10, _P, 10, None)) == ELIMIT   # S rides on gridDim.y
