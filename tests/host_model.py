"""Shared fixtures of the CPU tests that run host logic over the mock kernel layer (tests/mock_kernels.py): a tiny model,
synthetic batches, LoRA set-up, gradient read-out and the oracle's autograd for the fused trainer; the installed layer, a
generate loop and prompts for the generate tests."""
import torch

BF = torch.bfloat16
TARGETS = ["q_proj", "o_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "down_proj"]      # train.py:443


def tiny_model(seed=0):
    """A 4-layer, H = 256 MIDIModel in bf16, training mode."""
    import midi_model as mm
    torch.manual_seed(seed)
    cfg = mm.MIDIModelConfig.get_config("v2", True, n_layer=4, n_head=4, n_embd=256, n_inner=512)
    return mm.MIDIModel(cfg).to(BF).train()


def generate_model(monkeypatch, loop):
    """The tiny model in eval mode over the mock kernel layer, generating on `loop` (B200_GENERATE): "nograph" for the
    host-issued loop, "persist" for the persistent kernel's launch protocol."""
    import mock_kernels
    mock_kernels.install(monkeypatch, persist=loop == "persist")
    monkeypatch.setenv("B200_GENERATE", loop)
    return tiny_model(0).eval()


def prompts(model, lengths, seed):
    """Prompts of `lengths` events (int64 [L, T] arrays), cut from one synthetic batch."""
    from midi_b200.synth import synth_batch
    batch = synth_batch(model.tokenizer, len(lengths), max(lengths), seed=seed).numpy()
    return [batch[i, :L] for i, L in enumerate(lengths)]


def make_batch(model, B=2, S1=10, seed=1, pad_tail=0, lengths=None):
    """A synthetic [B, S1, T] int64 batch (midi_b200.synth); with `lengths` a right-padded one (train.py:86-90 collate_fn):
    sample b holds lengths[b] events, then pad_id, and B = len(lengths)."""
    from midi_b200.synth import synth_batch
    b = synth_batch(model.tokenizer, B if lengths is None else len(lengths), S1, seed=seed, pad_tail=pad_tail)
    for i, L in enumerate(lengths or ()):
        b[i, L:] = model.tokenizer.pad_id
    return b


def add_lora(model):
    """train.py:440-449: freeze the base, inject r = 8 adapters on every projection, and make B non-zero (B = 0 at init
    would zero the gradient of A)."""
    from midi_b200 import lora
    model.requires_grad_(False)
    model.add_adapter(lora.LoraAdapterConfig(r=8, lora_alpha=16, target_modules=TARGETS, lora_dropout=0, bias="none",
                                             task_type="CAUSAL_LM"))
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(BF))
    return model


def grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def oracle_padded(model, batch, lora_scale=None):
    """train.py:169-185 on the (padded) batch under the oracle's fp32 autograd over the bf16-rounded weights: (loss,
    {name: gradient}).  With adapters the effective weight W + scale * B A is formed differentiably, so the gradients of
    A and B are those of peft's unmerged forward."""
    from oracle import midi_oracle as O
    leaf = {n: p.detach().float().requires_grad_(True) for n, p in model.named_parameters()}
    sd = O.lora_effective_sd(leaf, lora_scale) if lora_scale is not None else leaf
    loss = O.train_loss(sd, O.cfg_from_hf(model.config), batch)
    loss.backward()
    return float(loss.detach()), {n: t.grad for n, t in leaf.items() if t.grad is not None}


def global_rel(got, ref):
    num = sum(float((got[n].double() - ref[n].double()).pow(2).sum()) for n in ref)
    den = sum(float(ref[n].double().pow(2).sum()) for n in ref)
    return (num / den) ** 0.5
