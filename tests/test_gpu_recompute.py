"""GPU tests (`pytest -m gpu`) of activation checkpointing (`model.gradient_checkpointing_enable()`) through the sm_90a
kernels: a checkpointed step against the same step without checkpointing, on the same weights and batch.

The recompute runs the forward's own deterministic kernels with the same GEMM plans, so the loss must agree bit for bit
and so must every gradient a GEMM produces (q/k/v/o/gate/up/down weights, lm_head, LoRA A and B).  RMSNorm-weight and
embedding-table gradients are summed with fp32 atomics whose order varies between any two runs (csrc/elementwise.cu
rmsnorm_bwd_warp_kernel, embed_bwd); they get the 1e-3 global relative bound the other trainer tests use for that spread.
The memory test measures what checkpointing is for: activation memory of a tv2o-medium step."""
import math
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

# metric-name prefix -> upper bound.  Every metric a test reports must match one.
BOUNDS = [
    ("loss_mismatch", 0.0),               # checkpointed loss vs default loss, bitwise
    ("gemm_grad_mismatch", 0.0),          # differing elements of GEMM-produced gradients
    ("atomic_grad_rel", 1e-3),            # norm weights + embedding tables: global relative difference
    ("grad_ready_mismatch", 0.0),         # grad_ready call sequence differs from the default step's
    ("grad_ready_cover_error", 0.0),      # [0, numel) handed over exactly once
    ("act_mem_ratio", 0.5),               # activation memory, checkpointed / default (tv2o-medium, B = 4 x 2048)
]
TARGETS = ["q_proj", "o_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "down_proj"]      # train.py:443


def _assert_within(metrics):
    bad, unbounded = [], []
    for k, v in metrics.items():
        b = next((b for p, b in BOUNDS if k.startswith(p)), None)
        if b is None:
            unbounded.append(k)
        elif math.isnan(v) or v > b:
            bad.append((k, v, b))
    print(metrics)
    assert not unbounded, unbounded
    assert not bad, bad


def _model(n_layer=4, name=None):
    import torch
    import midi_model as mm
    assert torch.cuda.is_available(), "needs an H100"
    torch.manual_seed(0)
    cfg = (mm.MIDIModelConfig.from_name(name) if name else
           mm.MIDIModelConfig.get_config("v2", True, n_layer=n_layer, n_head=16, n_embd=1024, n_inner=4096))
    return mm.MIDIModel(cfg).to("cuda", dtype=torch.bfloat16).train()


@pytest.fixture(scope="module")
def model():
    return _model()


def _batch(model, S1, seed, B=2):
    from midi_b200.synth import synth_batch
    return synth_batch(model.tokenizer, B, S1, seed=seed).to("cuda")


def _rand_idx(S, seed=0):
    random.seed(seed)
    return [-1] + random.sample(list(range(S - 2)), min(127, (S - 2) // 2))      # train.py:173


def _atomic(name):
    return name.endswith("norm.weight") or name.endswith("layernorm.weight") or name.endswith("embed_tokens.weight")


def _compare(model, step, tag):
    """step(grad_ready) with checkpointing off, then on -> metrics."""
    import torch
    out = []
    for on in (False, True):
        if on:
            model.gradient_checkpointing_enable()
        else:
            model.gradient_checkpointing_disable()
        for p in model.parameters():
            p.grad = None
        calls = []
        loss = step(lambda lo, hi: calls.append((lo, hi)))
        torch.cuda.synchronize()
        grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
        out.append((loss.detach().float().clone(), grads, calls))
    model.gradient_checkpointing_disable()
    (l0, g0, c0), (l1, g1, c1) = out
    assert g0 and g0.keys() == g1.keys()
    gemm = [n for n in g0 if not _atomic(n)]
    atomic = [n for n in g0 if _atomic(n)]
    m = {f"loss_mismatch_{tag}": float(not torch.equal(l0, l1)),
         f"gemm_grad_mismatch_{tag}": float(sum(int((g0[n] != g1[n]).sum()) for n in gemm)),
         f"grad_ready_mismatch_{tag}": float(c0 != c1)}
    if atomic:
        num = sum(float((g1[n].double() - g0[n].double()).pow(2).sum()) for n in atomic)
        den = sum(float(g0[n].double().pow(2).sum()) for n in atomic)
        m[f"atomic_grad_rel_{tag}"] = math.sqrt(num / den)
    if c1:
        store = model._rt().store
        cover, want = (torch.zeros(store.numel, dtype=torch.int32) for _ in range(2))
        want[store.train_lo:store.train_hi] = 1                  # everything in full training, the adapter tail in LoRA
        for lo, hi in c1:
            cover[lo:hi] += 1
        m[f"grad_ready_cover_error_{tag}"] = float((cover != want).sum())
    print(tag, "loss", float(l0), "gemm grads", len(gemm), "atomic grads", len(atomic), "grad_ready calls", len(c1))
    return m


@pytest.mark.gpu
def test_checkpointed_training_step(model):
    import torch
    m = {}
    for S1 in (2049, 130):
        batch = _batch(model, S1, seed=3)
        m.update(_compare(model, lambda gr: model.training_loss(batch, grad_ready=gr), f"full_S{S1 - 1}"))
    batch = _batch(model, 2049, seed=4)
    idx = _rand_idx(2048)
    m.update(_compare(model, lambda gr: model.training_loss(batch, sample_idx=idx, grad_ready=gr), "sample_idx"))
    a, b = _batch(model, 2049, seed=5), _batch(model, 2049, seed=6)

    def accumulate(gr):
        model.training_loss(a)
        return model.training_loss(b, accumulate=True, grad_ready=gr)
    m.update(_compare(model, accumulate, "accumulate"))
    a16 = a.to(torch.int16)
    m.update(_compare(model, lambda gr: model.training_loss(a16, grad_ready=gr), "int16"))
    _assert_within(m)


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
    _assert_within(m)


@pytest.mark.gpu
def test_checkpointed_lora_step():
    import torch
    from midi_b200 import lora
    model = _model()
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
    _assert_within(m)
    del model
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_checkpointing_halves_activation_memory():
    """tv2o-medium (12 + 3 layers) at B = 4 x 2048: allocator peak during a fused step minus what was allocated before it."""
    import torch
    model = _model(name="tv2o-medium")
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
    _assert_within(m)
