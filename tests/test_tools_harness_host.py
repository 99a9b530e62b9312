"""tools/harness.py without a GPU: the card query names its device, never raises, the clock sampler's child ends with the
block, and the resource table reads the library; every tool compiles, and bench.py can still load evolution_c4.py."""
import importlib.util
import py_compile
import subprocess
import types
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
TOOLS = ROOT / "tools"


def _load(name):
    spec = importlib.util.spec_from_file_location(name, str(TOOLS / f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def harness():
    return _load("harness")


def test_card_queries_the_named_device(harness, monkeypatch):
    calls = []

    def run(argv, **kw):
        calls.append(argv)
        return subprocess.CompletedProcess(argv, 0, stdout="NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n", stderr="")

    monkeypatch.setattr(subprocess, "run", run)
    assert harness.card(3) == {"card": "NVIDIA H100 80GB HBM3", "power_limit": "700.00 W", "sm_max_mhz": "1980 MHz"}
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 5)
    harness.card()
    assert [argv[argv.index("-i") + 1] for argv in calls] == ["3", "5"]
    assert all(argv[0] == "nvidia-smi" for argv in calls)


def test_card_falls_back_without_nvidia_smi(harness, monkeypatch):
    def missing(argv, **kw):
        raise FileNotFoundError(argv[0])

    def no_device(index=None):
        raise RuntimeError("no CUDA device")

    monkeypatch.setattr(subprocess, "run", missing)
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda index=None: "stand-in device")
    assert harness.card(0) == {"card": "stand-in device", "power_limit": "unavailable", "sm_max_mhz": "unavailable"}
    monkeypatch.setattr(torch.cuda, "get_device_name", no_device)
    monkeypatch.setattr(torch.cuda, "current_device", no_device)
    assert harness.card() == {"card": "unavailable", "power_limit": "unavailable", "sm_max_mhz": "unavailable"}


def test_sampled_clocks_ends_its_child_when_the_body_raises(harness, monkeypatch):
    import bench
    children = []

    class StandIn:
        def __init__(self, argv, **kw):
            self.argv, self.stdout, self.terminated, self.waited = argv, iter(()), False, False
            children.append(self)

        def terminate(self):
            self.terminated = True

        def wait(self, timeout=None):
            self.waited = True
            return 0

    monkeypatch.setattr(bench.subprocess, "Popen", StandIn)
    with pytest.raises(RuntimeError, match="body failed"):
        with harness.sampled_clocks(0) as clocks:
            raise RuntimeError("body failed")
    assert len(children) == 1 and children[0].argv[0] == "nvidia-smi"
    assert children[0].terminated and children[0].waited
    assert clocks.sm_clock is not None and "sm_mhz" in clocks.sm_clock


def test_kernel_resources_reads_the_built_library(harness, native_lib):
    res = harness.kernel_resources(["book_kernel", "trade_mc_kernel"])
    assert res is not None, "cuobjdump not found"
    assert set(res) == {"book_kernel", "trade_mc_kernel"}
    for entry in res.values():
        assert isinstance(entry["registers"], int) and entry["registers"] > 0


@pytest.mark.parametrize("path", sorted(TOOLS.glob("*.py")), ids=lambda p: p.name)
def test_tool_compiles(path, tmp_path):
    py_compile.compile(str(path), cfile=str(tmp_path / (path.name + "c")), doraise=True)


def test_evolution_c4_loads_by_file_path():
    mod = _load("evolution_c4")
    assert isinstance(mod, types.ModuleType) and callable(mod.run)
