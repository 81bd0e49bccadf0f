"""GPU tests (`pytest -m gpu`) of ragged batches in the fused trainer (`training_loss(batch, lengths=...)`): the segment
kernels against the unsegmented kernels run on each segment alone, and the ragged step against the padded step.

Kernels: in segment mode the attention kernels run the same tiles in the same order on the same operands as the
unsegmented kernels on one segment, so their outputs must be bit-identical segment by segment; each case is also scored
per row against fp64 inside NaN-sentinel buffers.  The segment RoPE entry points and the packing kernel are exact too.

Model: with every sample full and S % 64 == 0 the packed layout is the padded one, so the loss and every GEMM-produced
gradient must be bit-identical; RMSNorm-weight and embedding gradients are summed with fp32 atomics in a run-dependent
order and get the 1e-3 global relative bound of the other trainer tests.  With varied lengths the ragged step is scored
against the oracle's fp32 autograd of the padded batch, and against the native padded step, whose GEMMs run plans
chosen for a different M."""
import pytest

import gpu_checks as G
import gpu_model as GM
from host_model import TARGETS, global_rel as _rel, make_batch
from parity_metrics import assert_within

# metric-name prefix -> upper bound.  Every metric a test reports must match one.  Measured on an NVIDIA H100 80GB HBM3 at
# a 700 W power limit: every exact comparison 0; attention worst row 3.4e-3 (o), 4.5e-3 / 4.6e-3 / 4.3e-3 (dq / dk / dv,
# with or without the fused RoPE backward), LSE 1.2e-6; atomic gradients <= 1.7e-6; varied lengths vs the oracle 1.0e-4
# (loss) and 3.0e-3 (gradients); vs the native padded step 9.5e-7 (loss) and 1.1e-4 (gradients), bounded at about 2x.
BOUNDS = [
    ("seg_mismatch", 0.0),                # segment kernels vs the unsegmented kernel on each segment alone
    ("sentinels_changed", 0.0),
    ("nan_in_range", 0.0),
    ("lse_abs", G.AE_LSE_ABS),            # vs fp64: the attention conformance bounds of gpu_checks.py (ae_)
    ("row", G.AE_ROW),
    ("pack_mismatch", 0.0),
    ("loss_mismatch", 0.0),               # ragged vs padded loss, bitwise (full lengths, garbage tail, validation)
    ("gemm_grad_mismatch", 0.0),          # differing elements of GEMM-produced gradients
    ("atomic_grad_rel", 1e-3),            # norm weights + embedding tables: global relative difference
    ("oracle_loss_abs", G.SAMPLE_SEQ_LOSS_ABS),      # vs the oracle's fp32 autograd of the padded batch
    ("oracle_grad_rel", G.SAMPLE_SEQ_GRAD_REL),
    ("native_loss_abs", 2e-6),            # vs the native padded step (GEMM plans for another M)
    ("native_grad_rel", 2.5e-4),
    ("accum_grad_rel", 1e-3),             # two accumulated micro-batches vs bf16(sum of the separate gradients)
    ("grad_ready_cover_error", 0.0),
    ("val_grad_changed", 0.0),
]
D = 64


def _tables(seg_rows):
    """The `Segments` (tile table, orders) of segments of the given row counts (multiples of 64), on the GPU."""
    import torch
    import midi_model as mm
    return mm._ragged_layout(list(seg_rows), 1, torch.device("cuda"))[1]


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.gpu
@pytest.mark.parametrize("segs", [[64], [64, 192, 64, 1216, 128], [2048]], ids=["one_tile", "mixed", "s2048"])
@pytest.mark.parametrize("nh", [1, 16])
def test_segment_attention_kernels(segs, nh):
    tag = f"{'-'.join(map(str, segs))}_h{nh}"
    assert_within({f"{k}_{tag}": v for k, v in G.seg_attention_case(segs, nh).items()}, BOUNDS)


@pytest.mark.gpu
def test_segment_rope_kernels():
    """b200_gemm_bf16_rope_seg and b200_rope_qk_seg (forward and backward) per segment against the r % S entries."""
    import torch
    from oracle import midi_oracle as O
    from midi_b200 import ops
    segs = [64, 192, 64, 1216, 128]
    N, H, K = sum(segs), 1024, 1024
    seg = _tables(segs)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (torch.randn(N, K, generator=g, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(3 * H, K, generator=g, device="cuda") * 0.03).to(torch.bfloat16)
    cos, sin = ops.rope_table(O.default_inv_freq(D).to(torch.bfloat16).cuda(), max(segs))
    fused = ops.linear_rope_seg(x, w, cos, sin, seg.tiles, D)
    plain = ops.linear(x, w)
    rot = {bw: plain.clone() for bw in (False, True)}
    for bw in (False, True):
        ops.rope_qk_seg_(rot[bw], cos, sin, seg.tiles, H, D, backward=bw)
    m = {"seg_mismatch_gemm_rope": 0.0, "seg_mismatch_rope_fwd": 0.0, "seg_mismatch_rope_bwd": 0.0}
    r0 = 0
    for R in segs:
        ref = ops.linear_rope(x[r0:r0 + R], w, cos, sin, R, D)
        m["seg_mismatch_gemm_rope"] += float((ref != fused[r0:r0 + R]).sum())
        for bw in (False, True):
            one = plain[r0:r0 + R].clone()
            ops.rope_qk_(one, cos, sin, R, H, D, backward=bw)
            m[f"seg_mismatch_rope_{'bwd' if bw else 'fwd'}"] += float((one != rot[bw][r0:r0 + R]).sum())
        r0 += R
    # the fused epilogue rotates exactly as the stand-alone kernel does (as in the unsegmented entries)
    m["seg_mismatch_gemm_vs_rope_kernel"] = float((fused != rot[False]).sum())
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_pack_kernel_matches_torch_gather():
    import torch
    from midi_b200 import ops
    B, S1, T, pad = 3, 300, 8, 0
    g = torch.Generator(device="cuda").manual_seed(1)
    batch = torch.randint(-32768, 32768, (B, S1, T), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    batch[0, 0, :2] = torch.tensor([-32768, 32767], dtype=torch.int16)
    batch[2, S1 - 1, -2:] = torch.tensor([32767, -32768], dtype=torch.int16)
    src = torch.tensor([0, 1, -1, 5, S1 - 2, -1, S1, 2 * S1 + S1 - 2, 2 * S1 + 7, -1] * 37, dtype=torch.int32, device="cuda")
    x, y = ops.batch_to_xy_packed(batch, src, pad)
    flat = batch.reshape(B * S1, T).long()
    idx = src.long().clamp(min=0)
    gap = (src < 0)[:, None]
    m = {"pack_mismatch_x": float((x != flat[idx].masked_fill(gap, pad)).sum()),
         "pack_mismatch_y": float((y != flat[idx + 1].masked_fill(gap, pad)).sum()),
         "pack_mismatch_shape": float(x.shape != (src.numel(), T) or x.dtype != torch.long)}
    assert_within(m, BOUNDS)


# ------------------------------------------------------------------------------------------ model
@pytest.fixture(scope="module")
def model():
    return GM.cuda_model()


def _batch(model, lengths, S1, seed):
    return make_batch(model, S1=S1, seed=seed, lengths=lengths).to("cuda")


def _exact(a, b, tag):
    """GM.exact, and whether the two steps made the same grad_ready calls."""
    m = GM.exact(a, b, tag)
    if a[2] or b[2]:
        m[f"grad_ready_cover_error_{tag}_calls"] = float(a[2] != b[2])
    return m


@pytest.mark.gpu
def test_full_lengths_are_the_padded_step(model):
    import torch
    from midi_b200 import engine
    m = {}
    for S1, B in ((2049, 2), (129, 3)):
        batch = _batch(model, [S1] * B, S1, seed=3)
        for dt in (torch.int64, torch.int16):
            b = batch.to(dt)
            pad = GM.step(model, lambda gr: model.training_loss(b, grad_ready=gr))
            rag = GM.step(model, lambda gr: model.training_loss(b, grad_ready=gr, lengths=[S1] * B))
            m.update(_exact(pad, rag, f"S{S1 - 1}_{str(dt)[6:]}"))
            m.update(GM.cover(model, rag[2], f"S{S1 - 1}_{str(dt)[6:]}"))
    # the other RoPE settings: QKV GEMM epilogue in the forward, stand-alone RoPE kernel in the backward
    batch = _batch(model, [129] * 3, 129, seed=4)
    for flag, val in (("FUSE_ROPE_FWD", True), ("FUSE_ROPE", False)):
        old = getattr(engine, flag)
        setattr(engine, flag, val)
        try:
            pad = GM.step(model, lambda gr: model.training_loss(batch))
            rag = GM.step(model, lambda gr: model.training_loss(batch, lengths=[129] * 3))
        finally:
            setattr(engine, flag, old)
        m.update(_exact(pad, rag, f"S128_{flag}_{int(val)}"))
    # activation checkpointing: the checkpointed ragged step against the padded one
    model.gradient_checkpointing_enable()
    try:
        pad = GM.step(model, lambda gr: model.training_loss(batch))
        rag = GM.step(model, lambda gr: model.training_loss(batch, lengths=[129] * 3))
    finally:
        model.gradient_checkpointing_disable()
    m.update(_exact(pad, rag, "S128_checkpoint"))
    assert_within(m, BOUNDS)


VARIED = [2049, 1300, 700, 65]


@pytest.mark.gpu
def test_varied_lengths_against_oracle_and_padded_step(model):
    import torch
    import torch.nn.functional as F
    from oracle import midi_oracle as O
    batch = _batch(model, VARIED, 2049, seed=5)
    rag = GM.step(model, lambda gr: model.training_loss(batch, lengths=VARIED, grad_ready=gr))
    pad = GM.step(model, lambda gr: model.training_loss(batch))
    names = list(rag[1])
    m = {"native_loss_abs": float((rag[0] - pad[0]).abs()), "native_grad_rel": _rel(rag[1], pad[1])}
    m.update(GM.cover(model, rag[2], "varied"))
    # events past each length are never read: garbage there changes nothing
    junk = _batch(model, [2049] * 4, 2049, seed=9)
    dirty = batch.clone()
    for i, L in enumerate(VARIED):
        dirty[i, L:] = junk[i, L:]
    for dt in (torch.int64, torch.int16):
        b = dirty.to(dt)
        m.update(_exact(rag, GM.step(model, lambda gr: model.training_loss(b, lengths=VARIED, grad_ready=gr)),
                        f"garbage_{str(dt)[6:]}"))
    # the oracle's fp32 autograd of the padded batch (train.py:169-185)
    ocfg = O.cfg_from_hf(model.config)
    sd = {k: v.detach().float().requires_grad_(True) for k, v in model.state_dict().items()}
    lo = O.train_loss(sd, ocfg, batch)
    lo.backward()
    m["oracle_loss_abs"] = float((rag[0] - lo.detach()).abs())
    m["oracle_grad_rel"] = _rel(rag[1], {n: sd[n].grad for n in names})
    print("ragged loss", float(rag[0]), "padded", float(pad[0]), "oracle", float(lo))
    del sd, lo
    torch.cuda.empty_cache()
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_varied_lengths_checkpoint_accumulate_validation(model):
    import torch
    m = {}
    batch = _batch(model, VARIED, 2049, seed=5)
    plain = GM.step(model, lambda gr: model.training_loss(batch, lengths=VARIED))
    model.gradient_checkpointing_enable()
    try:
        ck = GM.step(model, lambda gr: model.training_loss(batch, lengths=VARIED))
    finally:
        model.gradient_checkpointing_disable()
    m.update(_exact(plain, ck, "checkpoint"))
    # two accumulated micro-batches
    la, lb = [130, 2, 77, 129], [64, 130, 0, 100]
    a, b = _batch(model, la, 130, seed=21), _batch(model, lb, 130, seed=22)
    _, ga, _ = GM.step(model, lambda gr: model.training_loss(a, lengths=la))
    _, gb, _ = GM.step(model, lambda gr: model.training_loss(b, lengths=lb))
    calls = []
    model.training_loss(a, lengths=la)
    model.training_loss(b, lengths=torch.tensor(lb), accumulate=True, grad_ready=lambda lo, hi: calls.append((lo, hi)))
    got = {n: p.grad.clone() for n, p in model.named_parameters()}
    gsum = {n: (ga[n].float() + gb[n].float()).to(torch.bfloat16) for n in ga}
    m["accum_grad_rel"] = _rel(got, gsum)
    m.update(GM.cover(model, calls, "accum"))
    # validation: the loss training_loss(backward=False) returns, gradient buffer untouched
    gflat = model._rt().store.gflat
    g0 = gflat.clone()
    loss, acc = model.validation_metrics(batch, VARIED)
    m["val_grad_changed"] = float((gflat != g0).sum())
    m["loss_mismatch_val"] = float(not torch.equal(loss, model.training_loss(batch, lengths=VARIED, backward=False)))
    print("val loss", float(loss), "acc", float(acc))
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_lora_ragged_step():
    import torch
    from midi_b200 import lora
    lm = GM.cuda_model()
    lm.requires_grad_(False)
    lm.add_adapter(lora.LoraAdapterConfig(r=16, lora_alpha=32, target_modules=TARGETS, lora_dropout=0, bias="none",
                                          task_type="CAUSAL_LM"))
    g = torch.Generator(device="cuda").manual_seed(5)
    with torch.no_grad():
        for n, p in lm.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(torch.bfloat16))
    m = {}
    batch = _batch(lm, [129] * 3, 129, seed=6)
    pad = GM.step(lm, lambda gr: lm.training_loss(batch, grad_ready=gr))
    rag = GM.step(lm, lambda gr: lm.training_loss(batch, lengths=[129] * 3, grad_ready=gr))
    m.update(_exact(pad, rag, "lora_full"))
    m.update(GM.cover(lm, rag[2], "lora"))
    vb = _batch(lm, VARIED, 2049, seed=7)
    lm.gradient_checkpointing_enable()
    ck = GM.step(lm, lambda gr: lm.training_loss(vb, lengths=VARIED))
    lm.gradient_checkpointing_disable()
    plain = GM.step(lm, lambda gr: lm.training_loss(vb, lengths=VARIED))
    m.update(_exact(plain, ck, "lora_checkpoint"))
    del lm
    torch.cuda.empty_cache()
    assert_within(m, BOUNDS)
