"""Host logic of the fused trainer's ragged batches (`training_loss(batch, lengths=...)`, `validation_metrics(batch,
lengths)`) on CPU, over the mock kernel layer (tests/mock_kernels.py), compared with the oracle's autograd of the padded
step.  The kernels themselves are checked on the GPU (tests/test_gpu_ragged.py)."""
import pytest
import torch

from host_model import BF, add_lora, global_rel as _global_rel, grads as _grads, make_batch, \
    oracle_padded as _oracle_padded, tiny_model as _tiny_model
from mock_kernels import install, trace as _trace


def _batch(model, lengths, S1, seed=1):
    return make_batch(model, S1=S1, seed=seed, lengths=lengths)


LENGTHS = [70, 66, 10, 1]          # 69, 65, 9 and 0 trained rows -> segments of 128, 128 and 64 rows


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
    install(monkeypatch)
    model = add_lora(_tiny_model())
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
    assert not {"batch_to_xy_packed", "rope_qk_seg_", "linear_rope_seg", "attn_causal_fwd_seg",
                "attn_causal_bwd_seg"} & set(base + vbase)


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
