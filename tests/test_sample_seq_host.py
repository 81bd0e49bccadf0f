"""Host logic of the fused trainer's train.py --sample-seq path (`training_loss(sample_idx=...)`) and of its validation
step (`validation_metrics`) on CPU, over the mock kernel layer (tests/mock_kernels.py), compared with the oracle's
autograd.  The kernels themselves are checked on the GPU (tests/test_gpu_sample_seq.py)."""
import pytest
import torch
import torch.nn.functional as F

from host_model import BF, add_lora, global_rel as _global_rel, grads as _grads, make_batch as _batch, \
    tiny_model as _tiny_model
from mock_kernels import install, trace as _trace


def _oracle_sampled(model, batch, idx, lora_scale=None):
    """train.py:169-185 with --sample-seq under the oracle's fp32 autograd: forward -> [:, idx] -> forward_token -> CE."""
    from oracle import midi_oracle as O
    leaf = {n: p.detach().float().requires_grad_(True) for n, p in model.named_parameters()}
    sd = O.lora_effective_sd(leaf, lora_scale) if lora_scale is not None else leaf
    cfg = O.cfg_from_hf(model.config)
    tok = model.tokenizer
    x, y = batch[:, :-1].long(), batch[:, 1:].long()
    h = O.forward(sd, cfg, x, inv_freq=model.net.rotary_emb.inv_freq)[:, idx]
    ys = y[:, idx].reshape(-1, y.shape[-1])
    logits = O.forward_token(sd, cfg, h.reshape(-1, h.shape[-1]), ys[:, :-1], inv_freq=model.net_token.rotary_emb.inv_freq)
    loss = F.cross_entropy(logits.reshape(-1, tok.vocab_size), ys.reshape(-1), reduction="mean", ignore_index=tok.pad_id)
    loss.backward()
    return float(loss.detach()), {n: t.grad for n, t in leaf.items() if t.grad is not None}


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("idx", [[-1, 3, 0, 5], [4], [4, -9, 7, 1, 2]])
def test_sample_idx_matches_oracle_autograd(monkeypatch, idx):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, pad_tail=2)
    ref_loss, ref = _oracle_sampled(model, batch, idx)
    loss = model.training_loss(batch, sample_idx=idx)
    assert abs(float(loss) - ref_loss) < 3e-2
    got = _grads(model)
    assert set(got) == {n for n, _ in model.named_parameters()}
    assert _global_rel(got, ref) < 3e-2
    # the event-level embedding gets gradient through the unselected rows' attention too, but no row outside the
    # selection feeds the token-level stack: its loss is that of the selected events only
    S = batch.shape[1] - 1
    full_loss = float(model.training_loss(batch, backward=False))
    assert (full_loss != float(loss)) or len(idx) == S


def test_sample_idx_int16_batch_and_tensor_index(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)
    idx = [-1, 2, 6, 0]
    l64 = model.training_loss(batch, sample_idx=idx)
    g64 = _grads(model)
    l16 = model.training_loss(batch.to(torch.int16), sample_idx=torch.tensor(idx, dtype=torch.int16))
    assert torch.equal(l16, l64)
    assert all(torch.equal(p.grad, g64[n]) for n, p in model.named_parameters())


def test_sample_idx_full_range_is_the_default_step(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, pad_tail=1)
    S = batch.shape[1] - 1
    l0 = model.training_loss(batch)
    g0 = _grads(model)
    l1 = model.training_loss(batch, sample_idx=range(S))
    assert torch.equal(l0, l1)
    assert all(torch.equal(p.grad, g0[n]) for n, p in model.named_parameters())


def test_sample_idx_accumulate_and_grad_ready(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    a, b = _batch(model, seed=1), _batch(model, seed=2)
    ia, ib = [-1, 0, 4], [5, 1, -2, 3]
    model.training_loss(a, sample_idx=ia)
    ga = _grads(model)
    model.training_loss(b, sample_idx=ib)
    gb = _grads(model)
    calls = []
    model.training_loss(a, sample_idx=ia)
    model.training_loss(b, sample_idx=ib, accumulate=True, grad_ready=lambda lo, hi: calls.append((lo, hi)))
    for n, p in model.named_parameters():
        assert torch.equal(p.grad, (ga[n].float() + gb[n].float()).to(BF)), n
    rt = model._rt()
    covered = sorted(calls)
    assert covered[0][0] == 0 and covered[-1][1] == rt.store.numel
    assert all(covered[i][1] == covered[i + 1][0] for i in range(len(covered) - 1))


def test_sample_idx_lora(monkeypatch):
    install(monkeypatch)
    model = add_lora(_tiny_model())
    batch = _batch(model)
    idx = [-1, 3, 0]
    ref_loss, ref = _oracle_sampled(model, batch, idx, lora_scale=2.0)
    loss = model.training_loss(batch, sample_idx=idx)
    assert abs(float(loss) - ref_loss) < 3e-2
    got = _grads(model)
    assert set(got) == {n for n in ref if ".lora_" in n}
    assert _global_rel(got, {n: ref[n] for n in got}) < 6e-2


def test_sample_idx_none_runs_the_default_calls(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)
    with monkeypatch.context() as m:
        base = _trace(m, lambda: model.training_loss(batch))
    with monkeypatch.context() as m:
        none = _trace(m, lambda: model.training_loss(batch, sample_idx=None))
    assert base == none
    assert "inner_input" in base and "b200_inner_input_bwd_hidden" in base
    assert not {"inner_input_rows", "inner_input_rows_bwd_hidden", "argmax_hits"} & set(base)
    with monkeypatch.context() as m:
        sampled = _trace(m, lambda: model.training_loss(batch, sample_idx=[-1, 2]))
    assert "inner_input_rows" in sampled and "inner_input_rows_bwd_hidden" in sampled
    assert "inner_input" not in sampled and "b200_inner_input_bwd_hidden" not in sampled


@pytest.mark.parametrize("bad", [
    [], (), torch.tensor([], dtype=torch.long), [9], [-10], [0, 0], [-1, 8], [[0, 1]], torch.tensor([[0, 1]]),
    torch.tensor([0.5]), [0.0], [True], torch.tensor([True]), "01", 3, {0, 1}, torch.tensor([1], device="meta"),
])
def test_sample_idx_rejects_invalid(monkeypatch, bad):
    from midi_b200.lib import B200Error
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model)                     # S = 9
    g0 = model._rt().store.gflat.clone()
    with pytest.raises(B200Error):
        model.training_loss(batch, sample_idx=bad)
    assert torch.equal(model._rt().store.gflat, g0)


def _compute_accuracy(logits, labels, pad_id):
    """train.py:153-166."""
    out = torch.argmax(logits, dim=-1).flatten()
    labels = labels.flatten()
    mask = labels != pad_id
    out, labels = out[mask], labels[mask]
    return torch.sum(out == labels).type(torch.float32) / len(labels)


def test_validation_metrics(monkeypatch):
    from oracle import midi_oracle as O
    install(monkeypatch)
    model = _tiny_model()
    tok = model.tokenizer
    batch = _batch(model, pad_tail=3)
    model.training_loss(batch)                                   # a gradient buffer with something in it
    g0 = model._rt().store.gflat.clone()
    loss, acc = model.validation_metrics(batch)
    assert loss.dim() == 0 and acc.dim() == 0 and loss.dtype == acc.dtype == torch.float32
    assert torch.equal(model._rt().store.gflat, g0)
    assert torch.equal(loss, model.training_loss(batch, backward=False))
    sd = {n: p.detach().float() for n, p in model.named_parameters()}
    with torch.no_grad():
        ref = O.train_loss(sd, O.cfg_from_hf(model.config), batch)
    assert abs(float(loss) - float(ref)) < 3e-2
    # the accuracy of train.py's validation_step on the drop-in path's logits (same kernels, same rounding)
    with torch.no_grad():
        y = batch[:, 1:].reshape(-1, batch.shape[-1])
        hidden = model.forward(batch[:, :-1].contiguous())
        logits = model.forward_token(hidden.reshape(-1, hidden.shape[-1]), y[:, :-1])
    assert torch.equal(acc, _compute_accuracy(logits, y, tok.pad_id))
    # no non-pad target: NaN, as mean CE and num_right / len(labels) give
    empty = torch.full_like(batch, tok.pad_id)
    l_e, a_e = model.validation_metrics(empty)
    assert torch.isnan(l_e) and torch.isnan(a_e)
