"""GPU tests (`pytest -m gpu`) of activation checkpointing (`model.gradient_checkpointing_enable()`) through the sm_90a
kernels: a checkpointed step against the same step without checkpointing, on the same weights and batch.

The recompute runs the forward's own deterministic kernels with the same GEMM plans, so the loss must agree bit for bit
and so must every gradient a GEMM produces (q/k/v/o/gate/up/down weights, lm_head, LoRA A and B).  RMSNorm-weight and
embedding-table gradients are summed with fp32 atomics whose order varies between any two runs (csrc/elementwise.cu
rmsnorm_bwd_warp_kernel, embed_bwd); they get the 1e-3 global relative bound the other trainer tests use for that spread.
The memory test measures what checkpointing is for: activation memory of a tv2o-medium step."""
import pytest

import gpu_model as GM
from host_model import TARGETS, make_batch
from parity_metrics import assert_within

# metric-name prefix -> upper bound.  Every metric a test reports must match one.
BOUNDS = [
    ("loss_mismatch", 0.0),               # checkpointed loss vs default loss, bitwise
    ("gemm_grad_mismatch", 0.0),          # differing elements of GEMM-produced gradients
    ("atomic_grad_rel", 1e-3),            # norm weights + embedding tables: global relative difference
    ("grad_ready_mismatch", 0.0),         # grad_ready call sequence differs from the default step's
    ("grad_ready_cover_error", 0.0),      # [0, numel) handed over exactly once
    ("act_mem_ratio", 0.5),               # activation memory, checkpointed / default (tv2o-medium, B = 4 x 2048)
]


@pytest.fixture(scope="module")
def model():
    return GM.cuda_model()


def _batch(model, S1, seed, B=2):
    return make_batch(model, B, S1, seed=seed).to("cuda")


def _compare(model, step, tag):
    """step(grad_ready) with checkpointing off, then on -> metrics."""
    runs = []
    for on in (False, True):
        if on:
            model.gradient_checkpointing_enable()
        else:
            model.gradient_checkpointing_disable()
        runs.append(GM.step(model, step))
    model.gradient_checkpointing_disable()
    (l0, g0, c0), (_, _, c1) = runs
    m = GM.exact(*runs, tag)
    m[f"grad_ready_mismatch_{tag}"] = float(c0 != c1)
    if c1:
        m.update(GM.cover(model, c1, tag))
    n_atomic = sum(map(GM.atomic, g0))
    print(tag, "loss", float(l0), "gemm grads", len(g0) - n_atomic, "atomic grads", n_atomic, "grad_ready calls", len(c1))
    return m


@pytest.mark.gpu
def test_checkpointed_training_step(model):
    import torch
    m = {}
    for S1 in (2049, 130):
        batch = _batch(model, S1, seed=3)
        m.update(_compare(model, lambda gr: model.training_loss(batch, grad_ready=gr), f"full_S{S1 - 1}"))
    batch = _batch(model, 2049, seed=4)
    idx = GM.rand_idx(2048)
    m.update(_compare(model, lambda gr: model.training_loss(batch, sample_idx=idx, grad_ready=gr), "sample_idx"))
    a, b = _batch(model, 2049, seed=5), _batch(model, 2049, seed=6)

    def accumulate(gr):
        model.training_loss(a)
        return model.training_loss(b, accumulate=True, grad_ready=gr)
    m.update(_compare(model, accumulate, "accumulate"))
    a16 = a.to(torch.int16)
    m.update(_compare(model, lambda gr: model.training_loss(a16, grad_ready=gr), "int16"))
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_checkpointed_dropin_path(model):
    """train.py:169-185 on the drop-in autograd path: forward -> forward_token -> F.cross_entropy -> backward."""
    import torch.nn.functional as F
    tok = model.tokenizer
    m = {}
    for S1 in (2049, 130):
        batch = _batch(model, S1, seed=7)

        def step(_gr):
            x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
            hidden = model.forward(x)
            hidden = hidden.reshape(-1, hidden.shape[-1])
            y = y.reshape(-1, y.shape[-1])
            logits = model.forward_token(hidden, y[:, :-1])
            loss = F.cross_entropy(logits.view(-1, tok.vocab_size), y.view(-1), reduction="mean", ignore_index=tok.pad_id)
            loss.backward()
            return loss
        m.update(_compare(model, step, f"dropin_S{S1 - 1}"))
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_checkpointed_lora_step():
    import torch
    from midi_b200 import lora
    model = GM.cuda_model()
    model.requires_grad_(False)                                                          # train.py:440
    model.add_adapter(lora.LoraAdapterConfig(r=64, lora_alpha=128, target_modules=TARGETS, lora_dropout=0, bias="none",
                                             task_type="CAUSAL_LM"))                    # train.py:441-449
    g = torch.Generator(device="cuda").manual_seed(5)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(torch.bfloat16))
    m = {}
    for S1 in (2049, 130):
        batch = _batch(model, S1, seed=8)
        m.update(_compare(model, lambda gr: model.training_loss(batch, grad_ready=gr), f"lora_S{S1 - 1}"))
    assert_within(m, BOUNDS)
    del model
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_checkpointing_halves_activation_memory():
    """tv2o-medium (12 + 3 layers) at B = 4 x 2048: allocator peak during a fused step minus what was allocated before it."""
    import torch
    model = GM.cuda_model(GM.config("tv2o-medium"))
    batch = _batch(model, 2049, seed=9, B=4)
    dev = batch.device
    act, losses = {}, {}
    for on in (False, True, False, True):               # first round warms up workspaces and plan caches
        if on:
            model.gradient_checkpointing_enable()
        else:
            model.gradient_checkpointing_disable()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        before = torch.cuda.memory_allocated(dev)
        loss = model.training_loss(batch)
        torch.cuda.synchronize()
        act[on] = torch.cuda.max_memory_allocated(dev) - before
        losses[on] = loss.detach().clone()
        del loss
    model.gradient_checkpointing_disable()
    ratio = act[True] / act[False]
    print(f"activation memory, tv2o-medium B=4x2048: default {act[False] / 2 ** 30:.2f} GiB, checkpointed "
          f"{act[True] / 2 ** 30:.2f} GiB, ratio {ratio:.3f}")
    m = {"act_mem_ratio": ratio, "loss_mismatch_medium": float(not torch.equal(losses[False], losses[True]))}
    del model, batch
    torch.cuda.empty_cache()
    assert_within(m, BOUNDS)
