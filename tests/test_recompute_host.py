"""Host logic of activation checkpointing (`model.gradient_checkpointing_enable()`) on CPU, over the mock kernel layer
(tests/mock_kernels.py): a checkpointed step must give exactly the loss and gradients of the default step (the mock
kernels are deterministic, like the real forward kernels), and its kernel-call trace must be the default trace plus, per
layer in backward, the recompute of that layer -- no attention forward, no down_proj.  The kernels themselves are checked
on the GPU (tests/test_gpu_recompute.py)."""
import pytest
import torch
import torch.nn.functional as F

import mock_kernels
from host_model import add_lora as _lora, grads as _grads, make_batch as _batch, tiny_model as _tiny_model


def _both(model, step):
    """step() with checkpointing off, then on: [(result, gradients, grad_ready calls)] for each."""
    out = []
    for on in (False, True):
        if on:
            model.gradient_checkpointing_enable()
        else:
            model.gradient_checkpointing_disable()
        for p in model.parameters():
            p.grad = None
        calls = []
        res = step(lambda lo, hi: calls.append((lo, hi)))
        out.append((res, _grads(model), calls))
    model.gradient_checkpointing_disable()
    return out


def _assert_same(out):
    (r0, g0, c0), (r1, g1, c1) = out
    assert torch.equal(r0, r1)
    assert g0.keys() == g1.keys() and g0
    for n in g0:
        assert torch.equal(g0[n], g1[n]), n
    assert c0 == c1


@pytest.mark.parametrize("case", ["full", "lora", "sample_idx", "int16"])
def test_checkpointed_step_is_exact(monkeypatch, case):
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    if case == "lora":
        _lora(model)
    batch = _batch(model, pad_tail=2)
    if case == "int16":
        batch = batch.to(torch.int16)
    idx = [-1, 3, 0, 5] if case == "sample_idx" else None
    _assert_same(_both(model, lambda gr: model.training_loss(batch, sample_idx=idx, grad_ready=gr)))


def test_checkpointed_accumulate_is_exact(monkeypatch):
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    a, b = _batch(model, seed=1), _batch(model, seed=2)

    def step(gr):
        model.training_loss(a, grad_ready=gr)
        return model.training_loss(b, accumulate=True, grad_ready=gr)
    _assert_same(_both(model, step))


@pytest.mark.parametrize("lora", [False, True])
def test_checkpointed_dropin_path_is_exact(monkeypatch, lora):
    """train.py:169-185 on the drop-in autograd path: forward -> forward_token -> F.cross_entropy -> backward."""
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    if lora:
        _lora(model)
    tok = model.tokenizer
    batch = _batch(model)

    def step(_gr):
        x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
        hidden = model.forward(x)
        hidden = hidden.reshape(-1, hidden.shape[-1])
        y = y.reshape(-1, y.shape[-1])
        logits = model.forward_token(hidden, y[:, :-1])
        loss = F.cross_entropy(logits.view(-1, tok.vocab_size), y.view(-1), reduction="mean", ignore_index=tok.pad_id)
        loss.backward()
        return loss.detach()
    _assert_same(_both(model, step))


def _split(names):
    """-> (the trace without the bracketed recompute calls, [the calls of each recompute, in order])."""
    rest, segs, cur = [], [], None
    for n in names:
        if n == "<recompute>":
            cur = []
        elif n == "</recompute>":
            segs.append(cur)
            cur = None
        elif cur is not None:
            cur.append(n)
        else:
            rest.append(n)
    return rest, segs


def _traced(monkeypatch, fn):
    """Kernel-call names of fn() with the recompute markers interleaved at the point where they happen."""
    from midi_b200 import engine
    names = []
    rec = engine.StackEngine._recompute

    def marked(self, *a, **k):
        names.append("<recompute>")
        r = rec(self, *a, **k)
        names.append("</recompute>")
        return r
    monkeypatch.setattr(engine.StackEngine, "_recompute", marked)
    return mock_kernels.trace(monkeypatch, fn, names)


# the recompute of one layer, per configuration: rmsnorm(x); QKV GEMM (+ q/k/v adapters: A GEMM, scale, B GEMM into qkv)
# and RoPE (the token-level forward rotates inside its attention kernel, the recompute with the stand-alone kernel);
# o_proj (+ adapter); add_rmsnorm; gate|up GEMM with SwiGLU fused, or GEMM + adapters + SwiGLU kernel
_ADAPTER = ["gemm", "scale", "gemm"]
_RECOMPUTE = {
    False: ["rmsnorm", "gemm", "rope_qk_", "gemm", "add_rmsnorm", "linear_swiglu"],
    True: (["rmsnorm", "gemm"] + _ADAPTER * 3 + ["rope_qk_", "gemm"] + _ADAPTER + ["add_rmsnorm", "gemm"] + _ADAPTER * 2
           + ["swiglu"]),
}


@pytest.mark.parametrize("lora", [False, True])
def test_checkpointed_trace_is_default_plus_recompute(monkeypatch, lora):
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    if lora:
        _lora(model)
    batch = _batch(model)
    n_outer, n_inner = model.config.net_config.num_hidden_layers, model.config.net_token_config.num_hidden_layers
    with monkeypatch.context() as m:
        base = _traced(m, lambda: model.training_loss(batch))
    assert "<recompute>" not in base
    model.gradient_checkpointing_enable()
    with monkeypatch.context() as m:
        ckpt = _traced(m, lambda: model.training_loss(batch))
    rest, segs = _split(ckpt)
    assert rest == base
    assert len(segs) == n_inner + n_outer
    for seg in segs:
        assert seg == _RECOMPUTE[lora]
        assert not any(n.startswith("attn_") for n in seg)
    # each recompute sits in backward, right before its layer's first gradient GEMM (down_proj's dgrad)
    first_bwd = ckpt.index("ce_bwd_")
    starts = [i for i, n in enumerate(ckpt) if n == "<recompute>"]
    assert all(i > first_bwd for i in starts)
    ends = [i for i, n in enumerate(ckpt) if n == "</recompute>"]
    assert all(ckpt[i + 1] == "gemm" for i in ends)
    model.gradient_checkpointing_disable()
    with monkeypatch.context() as m:
        again = _traced(m, lambda: model.training_loss(batch))
    assert again == base


def test_recompute_issues_no_down_proj_gemm(monkeypatch):
    """The GEMMs a recompute issues, by their (N, K): the QKV, o and gate|up projections, none with K = inner (down)."""
    from midi_b200 import engine, ops
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)
    model.gradient_checkpointing_enable()
    shapes, inside = [], [False]
    rec, gemm = engine.StackEngine._recompute, ops.gemm

    def marked(self, *a, **k):
        inside[0] = True
        try:
            return rec(self, *a, **k)
        finally:
            inside[0] = False

    def gemm_rec(A, B, M, N, K, **kw):
        if inside[0]:
            shapes.append((N, K))
        return gemm(A, B, M, N, K, **kw)
    monkeypatch.setattr(engine.StackEngine, "_recompute", marked)
    monkeypatch.setattr(ops, "gemm", gemm_rec)
    model.training_loss(batch)
    nc, tc = model.config.net_config, model.config.net_token_config
    want = ([(3 * tc.hidden_size, tc.hidden_size), (tc.hidden_size, tc.hidden_size)] * tc.num_hidden_layers
            + [(3 * nc.hidden_size, nc.hidden_size), (nc.hidden_size, nc.hidden_size)] * nc.num_hidden_layers)
    assert shapes == want                     # (gate|up runs in the fused SwiGLU GEMM, not through ops.gemm)


def test_is_gradient_checkpointing_follows_the_switch(monkeypatch):
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    assert model.supports_gradient_checkpointing and not model.is_gradient_checkpointing
    model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    assert model.is_gradient_checkpointing and model.net.gradient_checkpointing and model.net_token.gradient_checkpointing
    assert model._rt().checkpoint                      # a runtime built after the switch inherits it
    model.gradient_checkpointing_disable()
    assert not model.is_gradient_checkpointing and not model._rt().checkpoint
    model.gradient_checkpointing_enable()
    assert model._rt().checkpoint                      # and an existing runtime follows it
    model.__dict__["_b200_rt"] = None                  # (add_adapter / load_merge_lora rebuild the runtime)
    assert model._rt().checkpoint


def _dropin_forward(model, batch):
    tok = model.tokenizer
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
    hidden = model.forward(x)
    hidden = hidden.reshape(-1, hidden.shape[-1])
    y = y.reshape(-1, y.shape[-1])
    logits = model.forward_token(hidden, y[:, :-1])
    return F.cross_entropy(logits.view(-1, tok.vocab_size), y.view(-1), reduction="mean", ignore_index=tok.pad_id)


@pytest.mark.parametrize("which", ["net.layers.1.mlp.up_proj.weight", "net_token.layers.0.self_attn.q_proj.weight",
                                   "lm_head.weight", "fused_step"])
def test_dropin_guard_refuses_weights_changed_after_forward(monkeypatch, which):
    from midi_b200.lib import B200Error
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)
    model.gradient_checkpointing_enable()
    loss = _dropin_forward(model, batch)
    if which == "fused_step":
        model.training_loss(batch)                     # (the fused AdamW updates through a raw pointer)
        model.fused_optimizer_step(lr=1e-3, step=1)
    else:
        with torch.no_grad():
            dict(model.named_parameters())[which].mul_(1.5)
    with pytest.raises(B200Error, match="modified in place"):
        loss.backward()


def test_dropin_guard_is_silent_without_changes_and_off_by_default(monkeypatch):
    mock_kernels.install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)
    loss = _dropin_forward(model, batch)
    with torch.no_grad():
        model.lm_head.weight.mul_(1.5)                 # without checkpointing nothing is recomputed: no check
    loss.backward()
    model.gradient_checkpointing_enable()
    _dropin_forward(model, batch).backward()           # unchanged weights: no complaint
    assert all(p.grad is not None for p in model.parameters())
