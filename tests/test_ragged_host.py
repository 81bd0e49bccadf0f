"""Host logic of the fused trainer's ragged batches (`training_loss(batch, lengths=...)`, `validation_metrics(batch,
lengths)`) on CPU, over the mock kernel layer (tests/mock_kernels.py) plus stand-ins for the entry points they add,
compared with the oracle's autograd of the padded step.  The kernels themselves are checked on the GPU
(tests/test_gpu_ragged.py)."""
import pytest
import torch

import mock_kernels

BF = torch.bfloat16
TARGETS = ["q_proj", "o_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "down_proj"]      # train.py:443


# ------------------------------------------------------------------ stand-ins for the new wrappers (midi_b200.ops)
def batch_to_xy_packed(batch, src, pad_id):
    B, S1, T = batch.shape
    flat = batch.to(torch.long).reshape(B * S1, T)
    idx = src.long()
    x = torch.full((idx.numel(), T), pad_id, dtype=torch.long)
    y = x.clone()
    live = idx >= 0
    x[live], y[live] = flat[idx[live]], flat[idx[live] + 1]
    return x, y


def _segments(tiles):
    """[(row0, rows)] of the segments a {first, last} tile table describes."""
    firsts = sorted(set(tiles[:, 0].tolist()))
    return [(64 * f, 64 * (int(tiles[f, 1]) + 1 - f)) for f in firsts]


def rope_qk_seg_(qkv, cos, sin, tiles, H, D, backward=False):
    for r0, n in _segments(tiles):
        blk = qkv[r0:r0 + n]
        mock_kernels.rope_qk_(blk, cos, sin, n, H, D, backward=backward)


def linear_rope_seg(x, w_qkv, cos, sin, tiles, D):
    qkv = mock_kernels.gemm(x, w_qkv, x.shape[0], w_qkv.shape[0], x.shape[1], lda=x.stride(0), ldb=w_qkv.stride(0))
    rope_qk_seg_(qkv, cos, sin, tiles, w_qkv.shape[0] // 3, D)
    return qkv


def attn_causal_fwd_seg(qkv, tiles, order, n_heads, D, want_lse, impl=None):
    outs, lses = [], []
    for r0, n in _segments(tiles):
        o, lse = mock_kernels.attn_causal_fwd(qkv[r0:r0 + n], 1, n, n_heads, D, True)
        outs.append(o)
        lses.append(lse[0])
    return torch.cat(outs), (torch.cat(lses, 1) if want_lse else None)


def attn_causal_bwd_seg(qkv, out, dout, lse, tiles, order, n_heads, D, rope=None, impl=None):
    return torch.cat([mock_kernels.attn_causal_bwd(qkv[r0:r0 + n], out[r0:r0 + n], dout[r0:r0 + n], None, 1, n, n_heads, D,
                                                   rope=rope) for r0, n in _segments(tiles)])


def argmax_hits(logits, targets, V, ignore_index):
    am = logits[:, :V].float().argmax(-1)
    live = (targets != ignore_index) & (targets >= 0) & (targets < V)
    return torch.stack([(live & (am == targets)).sum(), live.sum()]).float()


NEW = ("batch_to_xy_packed", "rope_qk_seg_", "linear_rope_seg", "attn_causal_fwd_seg", "attn_causal_bwd_seg", "argmax_hits")


def install(monkeypatch):
    from midi_b200 import ops
    mock_kernels.install(monkeypatch)
    for name in NEW:
        monkeypatch.setattr(ops, name, globals()[name])


# ------------------------------------------------------------------ helpers
def _tiny_model(seed=0):
    import midi_model as mm
    torch.manual_seed(seed)
    cfg = mm.MIDIModelConfig.get_config("v2", True, n_layer=4, n_head=4, n_embd=256, n_inner=512)
    return mm.MIDIModel(cfg).to(BF).train()


def _batch(model, lengths, S1, seed=1):
    """A right-padded batch (train.py:86-90 collate_fn): sample b holds lengths[b] events, then pad_id."""
    from midi_b200.synth import synth_batch
    b = synth_batch(model.tokenizer, len(lengths), S1, seed=seed)
    for i, L in enumerate(lengths):
        b[i, L:] = model.tokenizer.pad_id
    return b


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _oracle_padded(model, batch, lora_scale=None):
    """train.py:169-185 on the padded batch under the oracle's fp32 autograd."""
    from oracle import midi_oracle as O
    leaf = {n: p.detach().float().requires_grad_(True) for n, p in model.named_parameters()}
    sd = O.lora_effective_sd(leaf, lora_scale) if lora_scale is not None else leaf
    loss = O.train_loss(sd, O.cfg_from_hf(model.config), batch)
    loss.backward()
    return float(loss.detach()), {n: t.grad for n, t in leaf.items() if t.grad is not None}


def _global_rel(got, ref):
    num = sum(float((got[n].double() - ref[n].double()).pow(2).sum()) for n in ref)
    den = sum(float(ref[n].double().pow(2).sum()) for n in ref)
    return (num / den) ** 0.5


LENGTHS = [70, 66, 10, 1]          # 69, 65, 9 and 0 trained rows -> segments of 128, 128 and 64 rows


def _trace(monkeypatch, fn):
    """Names of the kernel-layer calls `fn` issues (ops wrappers and raw C-ABI calls), in order."""
    from midi_b200 import lib, ops
    names = []
    for name in ("embed_sum", "inner_input", "batch_to_xy", "embed_bwd", "rmsnorm", "add_rmsnorm", "rmsnorm_bwd",
                 "rope_table", "rope_qk_", "swiglu", "swiglu_bwd", "scale", "gemm", "linear_swiglu", "linear_rope",
                 "attn_causal_fwd", "attn_causal_bwd", "attn_tiny_fwd", "attn_tiny_bwd", "ce_fwd", "ce_bwd_") + NEW:
        f = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _f=f, _n=name, **k: (names.append(_n), _f(*a, **k))[1])
    call = lib.call
    monkeypatch.setattr(lib, "call", lambda n, *a: (names.append(n), call(n, *a))[1])
    fn()
    monkeypatch.setattr(lib, "call", call)
    return names


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("mode", ["full", "checkpoint", "int16"])
def test_ragged_step_matches_oracle_padded_step(monkeypatch, mode):
    install(monkeypatch)
    model = _tiny_model()
    if mode == "checkpoint":
        model.gradient_checkpointing_enable()
    batch = _batch(model, LENGTHS, 70)
    ref_loss, ref = _oracle_padded(model, batch)
    loss = model.training_loss(batch.to(torch.int16) if mode == "int16" else batch, lengths=LENGTHS)
    assert abs(float(loss) - ref_loss) < 3e-2
    got = _grads(model)
    assert set(got) == {n for n, _ in model.named_parameters()}
    assert _global_rel(got, ref) < 3e-2


@pytest.mark.parametrize("fuse", ["fwd", "unfused"])
def test_ragged_step_rope_settings(monkeypatch, fuse):
    """The GEMM-epilogue RoPE (B200_FUSE_ROPE_FWD=1) and the stand-alone RoPE backward (B200_FUSE_ROPE=0) give the step
    of the default settings on the mock layer, where every variant rounds the same way."""
    from midi_b200 import engine
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    l0 = model.training_loss(batch, lengths=LENGTHS)
    g0 = _grads(model)
    monkeypatch.setattr(engine, "FUSE_ROPE_FWD" if fuse == "fwd" else "FUSE_ROPE", fuse == "fwd")
    with monkeypatch.context() as m:
        names = _trace(m, lambda: model.training_loss(batch, lengths=LENGTHS))
    assert ("linear_rope_seg" in names) == (fuse == "fwd")
    assert ("rope_qk_seg_" in names) == (fuse != "fwd")
    assert torch.equal(model.training_loss(batch, lengths=LENGTHS), l0)
    assert all(torch.equal(p.grad, g0[n]) for n, p in model.named_parameters())


def test_ragged_step_lora(monkeypatch):
    from midi_b200 import lora
    install(monkeypatch)
    model = _tiny_model()
    model.requires_grad_(False)
    model.add_adapter(lora.LoraAdapterConfig(r=8, lora_alpha=16, target_modules=TARGETS, lora_dropout=0, bias="none",
                                             task_type="CAUSAL_LM"))
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(BF))
    batch = _batch(model, LENGTHS, 70)
    ref_loss, ref = _oracle_padded(model, batch, lora_scale=2.0)
    loss = model.training_loss(batch, lengths=LENGTHS)
    assert abs(float(loss) - ref_loss) < 3e-2
    got = _grads(model)
    assert set(got) == {n for n in ref if ".lora_" in n}
    assert _global_rel(got, {n: ref[n] for n in got}) < 6e-2


def test_ragged_accumulate_and_grad_ready(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    la, lb = LENGTHS, [3, 70, 41, 0]
    a, b = _batch(model, la, 70, seed=1), _batch(model, lb, 70, seed=2)
    model.training_loss(a, lengths=la)
    ga = _grads(model)
    model.training_loss(b, lengths=lb)
    gb = _grads(model)
    calls = []
    model.training_loss(a, lengths=la)
    model.training_loss(b, lengths=torch.tensor(lb), accumulate=True, grad_ready=lambda lo, hi: calls.append((lo, hi)))
    for n, p in model.named_parameters():
        assert torch.equal(p.grad, (ga[n].float() + gb[n].float()).to(BF)), n
    rt = model._rt()
    covered = sorted(calls)
    assert covered[0][0] == 0 and covered[-1][1] == rt.store.numel
    assert all(covered[i][1] == covered[i + 1][0] for i in range(len(covered) - 1))
    # the same hand-over as the padded step's
    pad_calls = []
    model.training_loss(a, grad_ready=lambda lo, hi: pad_calls.append((lo, hi)))
    assert pad_calls == calls


@pytest.mark.parametrize("dtype", [torch.int64, torch.int16])
def test_events_past_the_length_are_not_read(monkeypatch, dtype):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    l0 = model.training_loss(batch.to(dtype), lengths=LENGTHS)
    g0 = _grads(model)
    junk = _batch(model, [70] * 4, 70, seed=9)
    dirty = batch.clone()
    for i, L in enumerate(LENGTHS):
        dirty[i, L:] = junk[i, L:]
    assert (dirty != batch).any()
    assert torch.equal(model.training_loss(dirty.to(dtype), lengths=LENGTHS), l0)
    assert all(torch.equal(p.grad, g0[n]) for n, p in model.named_parameters())
    v0 = model.validation_metrics(batch.to(dtype), LENGTHS)
    v1 = model.validation_metrics(dirty.to(dtype), LENGTHS)
    assert torch.equal(v0[0], v1[0]) and torch.equal(v0[1], v1[1])


def test_full_lengths_issue_the_default_calls(monkeypatch):
    """Every sample full and S % 64 == 0: the packed layout is the padded one, so the step issues the default step's calls
    -- the pack call and the segment variants in place of theirs -- and gets its loss and gradients exactly."""
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, [65, 65], 65).to(torch.int16)
    with monkeypatch.context() as m:
        base = _trace(m, lambda: model.training_loss(batch))
    g0 = _grads(model)
    l0 = model.training_loss(batch)
    with monkeypatch.context() as m:
        rag = _trace(m, lambda: model.training_loss(batch, lengths=[65, 65]))
    swap = {"batch_to_xy": "batch_to_xy_packed", "rope_qk_": "rope_qk_seg_", "attn_causal_fwd": "attn_causal_fwd_seg",
            "attn_causal_bwd": "attn_causal_bwd_seg"}
    assert rag == [swap.get(n, n) for n in base]
    assert torch.equal(model.training_loss(batch, lengths=[65, 65]), l0)
    assert all(torch.equal(p.grad, g0[n]) for n, p in model.named_parameters())


def test_lengths_none_runs_the_default_calls(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    with monkeypatch.context() as m:
        base = _trace(m, lambda: model.training_loss(batch))
    with monkeypatch.context() as m:
        none = _trace(m, lambda: model.training_loss(batch, lengths=None))
    assert base == none
    with monkeypatch.context() as m:
        vbase = _trace(m, lambda: model.validation_metrics(batch))
    with monkeypatch.context() as m:
        vnone = _trace(m, lambda: model.validation_metrics(batch, None))
    assert vbase == vnone
    assert not set(NEW[:-1]) & set(base + vbase)


def test_validation_metrics_lengths(monkeypatch):
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    model.training_loss(batch, lengths=LENGTHS)
    g0 = model._rt().store.gflat.clone()
    loss, acc = model.validation_metrics(batch, LENGTHS)
    assert torch.equal(model._rt().store.gflat, g0)
    assert torch.equal(loss, model.training_loss(batch, lengths=LENGTHS, backward=False))
    # the padded batch's metrics: the same targets, each row's logits from the same causal context
    lp, ap = model.validation_metrics(batch)
    assert abs(float(loss) - float(lp)) < 1e-2 and abs(float(acc) - float(ap)) < 5e-2


@pytest.mark.parametrize("bad", [
    [70, 66, 10], [70, 66, 10, 1, 1], [71, 1, 1, 1], [-1, 70, 70, 70], [70, 66.0, 10, 1], [70, True, 10, 1],
    torch.tensor([70.0, 66.0, 10.0, 1.0]), torch.tensor([[70, 66, 10, 1]]), torch.tensor([70, 66, 10, 1], device="meta"),
    "abcd", 70, [1, 1, 0, 1], [0, 0, 0, 0],
])
def test_lengths_rejects_invalid(monkeypatch, bad):
    from midi_b200.lib import B200Error
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    g0 = model._rt().store.gflat.clone()
    with pytest.raises(B200Error):
        model.training_loss(batch, lengths=bad)
    with pytest.raises(B200Error):
        model.validation_metrics(batch, bad)
    assert torch.equal(model._rt().store.gflat, g0)


def test_lengths_with_sample_idx_is_rejected(monkeypatch):
    from midi_b200.lib import B200Error
    install(monkeypatch)
    model = _tiny_model()
    batch = _batch(model, LENGTHS, 70)
    with pytest.raises(B200Error, match="sample_idx"):
        model.training_loss(batch, lengths=LENGTHS, sample_idx=[-1, 3])


def test_segment_attention_needs_the_wgmma_kernels(monkeypatch):
    """The mma.sync attention has no segment mode: a ragged call raises instead of running something else."""
    from midi_b200 import lib, ops
    from midi_b200.lib import B200Error
    monkeypatch.setattr(lib, "call", lambda *a: pytest.fail("no kernel may be called"))
    qkv = torch.zeros(128, 3 * 64, dtype=BF)
    tiles = torch.tensor([[0, 1], [0, 1]], dtype=torch.int32)
    order = torch.tensor([[1, 0], [0, 1]], dtype=torch.int32)
    monkeypatch.setattr(ops, "ATTN_IMPL", "mma")
    with pytest.raises(B200Error, match="segment"):
        ops.attn_causal_fwd_seg(qkv, tiles, order, 1, 64, want_lse=True)
    with pytest.raises(B200Error, match="segment"):
        ops.attn_causal_bwd_seg(qkv, qkv[:, :64], qkv[:, :64], None, tiles, order, 1, 64)


def test_ragged_layout_tables():
    """Tile table, source rows and longest-first orders of the packed layout."""
    import midi_model as mm
    src, seg = mm._ragged_layout([69, 0, 64, 1], 70, torch.device("cpu"))
    assert seg.rows == 128 + 64 + 64 and seg.max_len == 128 and src.shape == (256,)
    assert seg.tiles.tolist() == [[0, 1], [0, 1], [2, 2], [3, 3]]
    assert src[:69].tolist() == list(range(69)) and (src[69:128] == -1).all()
    assert src[128:192].tolist() == list(range(140, 204))
    assert src[192].item() == 210 and (src[193:] == -1).all()
    assert seg.order[0].tolist()[0] == 1 and sorted(seg.order[0].tolist()) == [0, 1, 2, 3]
    assert seg.order[1].tolist()[0] == 0 and sorted(seg.order[1].tolist()) == [0, 1, 2, 3]
