"""GPU parity tests (`pytest -m gpu`).  Each group compares the sm_90a kernels / the drop-in
MIDIModel -- called through the C ABI -- with the PyTorch composite / the oracle, judged by the bound table each check
carries; see gpu_checks.py."""
import pytest

import gpu_checks as G
from parity_metrics import assert_within


@pytest.mark.gpu
def test_native_library_is_loaded():
    """The product path must be the CUDA extension (no eager fallback): the .so is mapped into this process."""
    from midi_b200 import lib
    lib.load()
    maps = open("/proc/self/maps").read()
    assert "libmidi_b200.so" in maps
    assert lib.query("b200_abi_version") == 1


@pytest.mark.gpu
@pytest.mark.parametrize("group", list(G.GROUPS))
def test_gpu_group(group):
    import torch
    assert torch.cuda.is_available(), "needs an H100"
    g = G.GROUPS[group]
    metrics = g()
    torch.cuda.synchronize()
    assert_within(metrics, g.bounds, g.info)
