"""Fixtures of the GPU tests.  A test module registers one by importing it: `from gpu_fixtures import torch_cuda`."""
import pytest


@pytest.fixture(scope="module")
def torch_cuda(native_lib):
    """torch, with cuda:0 as the current device."""
    import torch
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    torch.cuda.set_device(0)
    return torch
