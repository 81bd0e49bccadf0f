"""Shared fixtures of the GPU tests that train the real-width model through the sm_90a kernels: the seeded model, train.py's
--sample-seq indices, and the step runner and comparisons of two fused steps that must agree bit for bit."""
import random

import torch

from host_model import BF, global_rel


def config(name=None):
    """A named MIDIModelConfig, by default 4 event-level layers at the real width (H = 1024, 16 heads, 4096 inner)."""
    import midi_model as mm
    return (mm.MIDIModelConfig.from_name(name) if name else
            mm.MIDIModelConfig.get_config("v2", True, n_layer=4, n_head=16, n_embd=1024, n_inner=4096))


def cpu_model(cfg=None):
    """The fp32 MIDIModel of `cfg` (default: config()) on the CPU, initialised from seed 0."""
    import midi_model as mm
    torch.manual_seed(0)
    return mm.MIDIModel(cfg or config())


def cuda_model(cfg=None):
    """cpu_model in bf16 on the GPU, in training mode."""
    assert torch.cuda.is_available(), "needs an H100"
    return cpu_model(cfg).to("cuda", dtype=BF).train()


def rand_idx(S, seed=0):
    random.seed(seed)
    return [-1] + random.sample(list(range(S - 2)), min(127, (S - 2) // 2))      # train.py:173


def atomic(name):
    """Gradients summed with fp32 atomics in a run-dependent order (csrc/elementwise.cu rmsnorm_bwd_warp_kernel,
    embed_bwd): RMSNorm weights and embedding tables.  Every other gradient comes out of a deterministic GEMM."""
    return name.endswith("norm.weight") or name.endswith("layernorm.weight") or name.endswith("embed_tokens.weight")


def step(model, fn):
    """fn(grad_ready) on cleared gradients -> (loss, {name: gradient}, [(lo, hi) grad_ready calls])."""
    for p in model.parameters():
        p.grad = None
    calls = []
    loss = fn(lambda lo, hi: calls.append((lo, hi)))
    torch.cuda.synchronize()
    return loss.detach().float().clone(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}, calls


def exact(a, b, tag):
    """Metrics of two steps that must agree bit for bit up to the fp32-atomic gradients."""
    (l0, g0, _), (l1, g1, _) = a, b
    assert g0 and g0.keys() == g1.keys()
    gemm = [n for n in g0 if not atomic(n)]
    atomics = [n for n in g0 if atomic(n)]
    m = {f"loss_mismatch_{tag}": float(not torch.equal(l0, l1)),
         f"gemm_grad_mismatch_{tag}": float(sum(int((g0[n] != g1[n]).sum()) for n in gemm))}
    if atomics:
        m[f"atomic_grad_rel_{tag}"] = global_rel(g1, {n: g0[n] for n in atomics})
    return m


def cover(model, calls, tag):
    """How many elements grad_ready did not hand over exactly once: everything in full training, the adapter tail in
    LoRA."""
    store = model._rt().store
    got, want = (torch.zeros(store.numel, dtype=torch.int32) for _ in range(2))
    want[store.train_lo:store.train_hi] = 1
    for lo, hi in calls:
        got[lo:hi] += 1
    return {f"grad_ready_cover_error_{tag}": float((got != want).sum())}
