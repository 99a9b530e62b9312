"""CPU-side checks of the drop-in boundary: the library builds for sm_90a, loads,
exports every symbol include/b200bt.h declares, and refuses to compute without a GPU."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol(native_lib):
    header = (ROOT / "include" / "b200bt.h").read_text()
    declared = set(re.findall(r"\b(b200bt_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    from ai_crypto_trader_b200 import _lib
    assert set(_lib.exported_symbols()) == declared
    for name in declared:
        assert hasattr(native_lib, name), name
    assert native_lib.b200bt_abi_version() == 1


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


def test_struct_layouts_match_header(native_lib):
    from ai_crypto_trader_b200 import _lib
    assert C.sizeof(_lib.Individual) == 40
    assert C.sizeof(_lib.SweepConfig) == 40
    assert len(_lib.LANE_STATS_FIELDS) * 8 == 160


def test_no_cpu_fallback(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    from ai_crypto_trader_b200 import _lib
    periods = (C.c_int * 1)(14)
    buf = (C.c_float * 64)()
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_rsi_bank", C.addressof(buf), 1, 64, 64, periods, 1, 1, C.addressof(buf), None)
    assert ei.value.status == 10002  # B200BT_ENODEVICE
    from ai_crypto_trader_b200.sweep import MarketData
    import numpy as np
    with pytest.raises(RuntimeError):
        MarketData(np.zeros((5, 1, 8), dtype=np.float32))


def test_argument_validation(native_lib):
    from ai_crypto_trader_b200 import _lib
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_rsi_bank", None, 1, 64, 64, (C.c_int * 1)(14), 1, 1, None, None)
    assert ei.value.status == 10001
