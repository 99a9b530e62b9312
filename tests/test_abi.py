"""CPU-side checks of the drop-in boundary: the library builds for sm_90a, loads,
exports every symbol include/b200bt.h declares, and refuses to compute without a GPU."""
import ctypes as C
import re
from pathlib import Path

import pytest

import abi_header
from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE


def test_library_exports_every_declared_symbol(native_lib):
    header = abi_header.parse()
    for name in header.prototypes:
        assert hasattr(native_lib, name), name
    assert native_lib.b200bt_abi_version() == header.defines["B200BT_ABI_VERSION"]


def test_library_holds_sm90a_code_only(native_lib):
    import shutil
    import subprocess
    import __graft_entry__
    nvcc = shutil.which(__graft_entry__._nvcc())          # cuobjdump sits beside the nvcc the build uses
    tool = Path(nvcc).with_name("cuobjdump") if nvcc else None
    if tool is None or not tool.exists():
        pytest.skip("cuobjdump not available")
    from ai_crypto_trader_b200 import _lib
    out = subprocess.run([tool, "--list-elf", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    assert set(re.findall(r"\.(sm_\w+)\.cubin", out)) == {"sm_90a"}, out


def test_no_cpu_fallback(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    from ai_crypto_trader_b200 import _lib
    periods = (C.c_int * 1)(14)
    buf = (C.c_float * 64)()
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_rsi_bank", C.addressof(buf), 1, 64, 64, periods, 1, 1, C.addressof(buf), None)
    assert ei.value.status == ENODEVICE
    from ai_crypto_trader_b200.sweep import MarketData
    import numpy as np
    with pytest.raises(RuntimeError):
        MarketData(np.zeros((5, 1, 8), dtype=np.float32))


def test_argument_validation(native_lib):
    from ai_crypto_trader_b200 import _lib
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_rsi_bank", None, 1, 64, 64, (C.c_int * 1)(14), 1, 1, None, None)
    assert ei.value.status == EINVAL


_CPU_TENSOR_CALLS = """
import torch
from ai_crypto_trader_b200 import indicators, sweep
x = torch.zeros((2, 64), dtype=torch.float32)
for name, call in (("nanfill_", lambda: indicators.nanfill_(x)), ("rsi_bank", lambda: sweep.rsi_bank(x, [14])),
                   ("from_close", lambda: sweep.MarketData.from_close(x))):
    try:
        call()
    except ValueError:
        continue
    raise SystemExit(name + " accepted a host tensor")
"""


def test_host_wrappers_refuse_host_tensors_under_python_O():
    """The wrappers check a tensor's device and dtype before its pointer goes to C with raises, not assert statements,
    which `python -O` strips."""
    import subprocess
    import sys
    subprocess.run([sys.executable, "-O", "-c", _CPU_TENSOR_CALLS], cwd=Path(__file__).resolve().parents[1], check=True)


_CLOCK_N, _CLOCK_BAR = 200_000, 7
_CLOCK_END = (1 << 32) - 1440          # minute0 + N * bar_minutes + gap_minutes must stay below this


def _sweep_calls(cfg):
    """The three sweep entry points with real sizes (P = 26 periods, S = 2 symbols, N = 200 000 7-minute bars, 64
    individuals) and the host config `cfg`.  The clock in cfg_host is checked before the device is touched; every config
    passed here is rejected there, so the non-null dummy device pointers are never dereferenced and nothing is launched."""
    from ai_crypto_trader_b200 import _lib
    lib = _lib.load()
    P, S, N, pop, K, n_seg, pool = 26, 2, _CLOCK_N, 64, 8, 64 * 8, 4096
    ws_c = int(lib.b200bt_sweep_chunked_workspace_bytes(pool, S, n_seg))
    ws_t = int(lib.b200bt_sweep_tiled_workspace_bytes(pool, S, pop, K))
    ref = C.byref(cfg)
    return {
        "b200bt_sweep": (DEV, N, DEV, N, P, S, N, DEV, None, pop, ref, DEV, None, 0, None),
        "b200bt_sweep_chunked": (DEV, N, DEV, N, P, S, N, DEV, None, pop, DEV, n_seg, DEV, DEV, n_seg, 2048, 8, pool, DEV,
                                 ws_c, ref, DEV, None, 0, DEV, None, None),
        "b200bt_sweep_tiled": (DEV, N, DEV, N, P, S, N, None, DEV, DEV, pop, None, pop, K, 1536, 2, pool, DEV, ws_t, ref,
                               DEV, None, 0, DEV, None, None),
    }


@pytest.mark.parametrize("case, minute0, gap_minutes, bar_minutes, status", [
    ("sum at 2^32 - 1440", _CLOCK_END - _CLOCK_N * _CLOCK_BAR - 1441, 1441, _CLOCK_BAR, ELIMIT),
    ("minute0 at 2^32 - 1440", _CLOCK_END, 0, _CLOCK_BAR, ELIMIT),
    ("minute0 near 2^62", 1 << 62, 0, _CLOCK_BAR, ELIMIT),
    ("negative minute0", -1, 0, _CLOCK_BAR, EINVAL),
    ("negative gap_minutes", 0, -1, _CLOCK_BAR, EINVAL),
    ("negative gap_minutes, large minute0", _CLOCK_END - _CLOCK_N * _CLOCK_BAR, -1, _CLOCK_BAR, EINVAL),
    ("zero bar_minutes", 0, 0, 0, EINVAL),
])
def test_sweep_entry_points_reject_an_out_of_range_calendar(native_lib, case, minute0, gap_minutes, bar_minutes, status):
    """The kernels form calendar minutes in unsigned 32 bits: the three sweep entry points refuse a clock that leaves that
    range (ELIMIT) and a negative clock field (EINVAL) alike.  The largest accepted clock, one minute lower than the
    first case, is swept on the GPU in tests/test_gpu_sweep_calendar.py."""
    from ai_crypto_trader_b200 import _lib
    cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=minute0, bar_minutes=bar_minutes, primary=0, secondary_mask=7,
                           variant=0, gap_bar=_CLOCK_N // 2, gap_minutes=gap_minutes)
    for name, args in _sweep_calls(cfg).items():
        with pytest.raises(_lib.B200btError) as ei:
            _lib.call(name, *args)
        assert ei.value.status == status, (case, name, str(ei.value))
        assert "minute0" in str(ei.value) or "bar_minutes" in str(ei.value), (case, name, str(ei.value))


@pytest.mark.parametrize("minute0", [-1, -1439, -(1 << 40)])
def test_resample_and_align_reject_a_negative_clock(native_lib, minute0):
    """The derived clocks bucket minute0 + t * bar_minutes with truncating division, which floors only from 0 up: a negative
    minute0 would start the first bucket on the wrong minute.  Both entry points refuse it (checked before the device is
    touched; the dummy pointers are never read) and b200bt_resample_bars reports no bars."""
    from ai_crypto_trader_b200 import _lib
    lib = _lib.load()
    N, bar, k = 1000, 5, 15
    assert lib.b200bt_resample_bars(N, minute0, bar, k) == 0
    assert lib.b200bt_resample_bars(N, 0, bar, k) == (N * bar + k - 1) // k
    M = int(lib.b200bt_resample_bars(N, 0, bar, k))
    for name, args in (("b200bt_resample", (DEV, 2, N, minute0, bar, k, DEV, M, None)),
                       ("b200bt_align", (DEV, 2, M, N, minute0, bar, k, DEV, None))):
        with pytest.raises(_lib.B200btError) as ei:
            _lib.call(name, *args)
        assert ei.value.status == EINVAL and "minute0" in str(ei.value), (name, str(ei.value))
