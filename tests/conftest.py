import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
GOLDEN = Path(__file__).resolve().parent / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def sim_golden():
    meta = json.loads((GOLDEN / "sim_cases.json").read_text())
    arrays = np.load(GOLDEN / "sim_cases.npz")
    return meta, arrays


@pytest.fixture(scope="session")
def native_lib():
    """The in-tree C-ABI library; built on demand (nvcc cross-compiles without a GPU)."""
    from ai_crypto_trader_b200 import _lib
    if not _lib.LIB_PATH.exists():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


def unjson(x):
    if isinstance(x, str):
        return float(x)
    return x
