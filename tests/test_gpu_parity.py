"""GPU parity tests (`pytest -m gpu`).  Each group compares the sm_90a kernels / the drop-in
MIDIModel -- called through the C ABI -- with the PyTorch composite / the oracle; see gpu_checks.py."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

GROUP_NAMES = ["gemm_fwd", "gemm_swiglu", "gemm_dgrad", "gemm_wgrad", "elementwise", "fused_rope", "attn_flash", "attn_wgmma", "attn_tiny", "loss_optim", "decode",
               "model_forward", "model_layer_tf", "model_train", "model_generate", "model_peaked_greedy", "model_large",
               "gemm_exact", "decode_paged", "lora_train", "model_vs_hf", "model_medium_long"]


@pytest.mark.gpu
def test_native_library_is_loaded():
    """The product path must be the CUDA extension (no eager fallback): the .so is mapped into this process."""
    from midi_b200 import lib
    lib.load()
    maps = open("/proc/self/maps").read()
    assert "libmidi_b200.so" in maps
    assert lib.query("b200_abi_version") == 1


@pytest.mark.gpu
@pytest.mark.parametrize("group", GROUP_NAMES)
def test_gpu_group(group):
    import torch
    assert torch.cuda.is_available(), "needs an H100"
    import gpu_checks as G
    metrics = G.GROUPS[group]()
    torch.cuda.synchronize()
    bad = [(k, v, b) for k, v, b, ok in G.verdict(metrics) if not ok]
    assert not bad, f"{group}: out of tolerance: {bad}"
