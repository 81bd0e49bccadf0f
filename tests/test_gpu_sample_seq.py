"""GPU tests (`pytest -m gpu`) of the fused trainer's train.py --sample-seq path (`training_loss(sample_idx=...)`), its
validation step (`validation_metrics`) and the argmax-hits kernel behind the accuracy, through the sm_90a kernels.

The reference for the sampled step is the drop-in autograd path running train.py's own expression
(`forward(x)[:, rand_idx]` -> `forward_token` -> `F.cross_entropy`) on the same weights, batch and indices; it runs the
same kernels, so the loss must agree bit for bit (the drop-in loss is bf16, the dtype of the logits: the fused fp32 loss
rounded to bf16 must equal it) and the gradients within the spread of the backward's non-deterministic fp32 reductions.
The oracle's fp32 autograd bounds the error itself."""
import pytest

import gpu_checks as G
import gpu_model as GM
from host_model import BF, global_rel as _rel, grads as _grads, make_batch
from parity_metrics import assert_within

# metric-name prefix -> upper bound.  Every metric a test reports must match one.
BOUNDS = [
    ("dropin_loss_mismatch", 0.0),        # fused loss (rounded to bf16) vs the drop-in --sample-seq loss
    ("dropin_grad_rel", G.INT16_PATH_GRAD_REL),      # global relative gradient error
    ("oracle_loss_abs", G.SAMPLE_SEQ_LOSS_ABS),      # vs the oracle's fp32 autograd
    ("oracle_grad_rel", G.SAMPLE_SEQ_GRAD_REL),
    ("full_range_loss_mismatch", 0.0),    # sample_idx = range(S) vs training_loss(batch)
    ("full_range_grad_rel", 1e-3),
    ("accum_grad_rel", 1e-3),             # two accumulated micro-batches vs bf16(sum of the separate gradients)
    ("grad_ready_cover_error", 0.0),
    ("argmax_mismatch", 0.0),             # hits / counts vs torch.argmax
    ("val_loss_mismatch", 0.0),
    ("val_acc_mismatch", 0.0),
    ("val_grad_changed", 0.0),
    ("val_empty_not_nan", 0.0),
]


@pytest.fixture(scope="module")
def model():
    return GM.cuda_model()


def _batch(model, S1, seed, pad_tail=0):
    return make_batch(model, 2, S1, seed=seed, pad_tail=pad_tail).to("cuda")


def _fused(model, batch, idx, **kw):
    loss = model.training_loss(batch, sample_idx=idx, **kw)
    return loss.detach().clone(), _grads(model)


def _dropin(model, batch, idx):
    """train.py:169-185 with --sample-seq on the drop-in autograd path."""
    import torch.nn.functional as F
    tok = model.tokenizer
    for p in model.parameters():
        p.grad = None
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
    hidden = model.forward(x)[:, idx]
    ys = y[:, idx].reshape(-1, y.shape[-1])
    logits = model.forward_token(hidden.reshape(-1, hidden.shape[-1]), ys[:, :-1])
    loss = F.cross_entropy(logits.view(-1, tok.vocab_size), ys.reshape(-1), reduction="mean", ignore_index=tok.pad_id)
    loss.backward()
    return loss.detach().clone(), _grads(model)


def _vs_dropin(model, batch, idx, tag):
    import torch
    lf, gf = _fused(model, batch, idx)
    ld, gd = _dropin(model, batch, idx)
    assert ld.dtype == torch.bfloat16
    return {f"dropin_loss_mismatch_{tag}": float(lf.to(torch.bfloat16) != ld),
            f"dropin_grad_rel_{tag}": _rel(gf, gd)}


@pytest.mark.gpu
def test_sampled_step_matches_the_dropin_expression(model):
    m = {}
    for S1 in (130, 2049):
        m.update(_vs_dropin(model, _batch(model, S1, seed=5), GM.rand_idx(S1 - 1), f"S{S1 - 1}"))
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_sampled_step_matches_oracle_autograd(model):
    import torch
    import torch.nn.functional as F
    from oracle import midi_oracle as O
    tok = model.tokenizer
    batch = _batch(model, 130, seed=5)
    idx = GM.rand_idx(129)
    lf, gf = _fused(model, batch, idx)
    ocfg = O.cfg_from_hf(model.config)
    sd = {k: v.detach().float().requires_grad_(True) for k, v in model.state_dict().items()}
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
    h = O.forward(sd, ocfg, x, inv_freq=model.net.rotary_emb.inv_freq)[:, idx]
    ys = y[:, idx].reshape(-1, 8)
    lg = O.forward_token(sd, ocfg, h.reshape(-1, h.shape[-1]), ys[:, :-1], inv_freq=model.net_token.rotary_emb.inv_freq)
    lo = F.cross_entropy(lg.view(-1, tok.vocab_size), ys.reshape(-1), reduction="mean", ignore_index=tok.pad_id)
    lo.backward()
    assert_within({"oracle_loss_abs": float((lf - lo.detach()).abs()),
                   "oracle_grad_rel": _rel(gf, {n: sd[n].grad for n in gf})}, BOUNDS)
    del sd, lg, h
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_full_range_is_the_default_step(model):
    batch = _batch(model, 130, seed=11)
    l0 = model.training_loss(batch).detach().clone()
    g0 = _grads(model)
    l1, g1 = _fused(model, batch, range(129))
    assert_within({"full_range_loss_mismatch": float(l0 != l1), "full_range_grad_rel": _rel(g1, g0)}, BOUNDS)


@pytest.mark.gpu
def test_sampled_step_edge_cases(model):
    import torch
    m = {}
    # unsorted and negative positions; a batch whose last 20 events are padding (-1 selects a pad event); S = 3 (K = 1)
    m.update(_vs_dropin(model, _batch(model, 130, seed=7), [5, -1, 0, -7, 3, 100, -128], "unsorted"))
    m.update(_vs_dropin(model, _batch(model, 130, seed=8, pad_tail=20), GM.rand_idx(129, seed=3), "padtail"))
    m.update(_vs_dropin(model, _batch(model, 4, seed=9), GM.rand_idx(3), "S3"))
    # two accumulated micro-batches with different indices == the sum of their separate gradients
    a, b = _batch(model, 130, seed=21), _batch(model, 130, seed=22)
    ia, ib = GM.rand_idx(129, seed=1), GM.rand_idx(129, seed=2)
    _, ga = _fused(model, a, ia)
    _, gb = _fused(model, b, ib)
    calls = []
    model.training_loss(a, sample_idx=ia)
    model.training_loss(b, sample_idx=ib, accumulate=True, grad_ready=lambda lo, hi: calls.append((lo, hi)))
    gsum = {n: (ga[n].float() + gb[n].float()).to(BF) for n in ga}
    m["accum_grad_rel"] = _rel(_grads(model), gsum)
    # grad_ready hands over [0, numel) exactly once
    cover = torch.zeros(model._rt().store.numel, dtype=torch.int32)
    for lo, hi in calls:
        cover[lo:hi] += 1
    m["grad_ready_cover_error"] = float((cover != 1).sum())
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_argmax_hits_kernel_matches_torch_argmax():
    import torch
    from midi_b200 import ops
    V, ld, R = 3406, 3408, 1000
    g = torch.Generator(device="cuda").manual_seed(0)
    L = torch.full((R, ld), float("nan"), dtype=torch.bfloat16, device="cuda")       # NaN in the pad columns
    L[:, :V] = torch.randn(R, V, generator=g, device="cuda").to(torch.bfloat16)
    cols = torch.randint(0, V, (100, 3), generator=g, device="cuda")
    for r in range(100):                                                              # exact ties of 2-3 columns
        L[r, cols[r, : 2 + r % 2]] = 8.0
    L[100, :V] = 0.0                                                                  # all equal -> 0
    L[101, :V] = -1.0
    L[101, 7] = -0.0
    L[101, 3] = 0.0                                                                   # -0 == +0: lowest index
    L[102, 50] = float("nan")
    L[102, 20] = float("nan")                                                         # NaN is the maximum, first one
    L[103, V - 1] = float("nan")
    L[104, :V] = float("-inf")
    L[105, V - 1] = 100.0                                                             # last column
    L[106, 3403] = 50.0                                                               # the scalar-loaded tail
    L[107, 3399] = 50.0                                                               # last full vector
    ref = torch.argmax(L[:, :V], dim=-1)
    pad = 0
    r = torch.arange(R, device="cuda")
    rnd = torch.randint(0, V, (R,), generator=g, device="cuda")
    tie_other = torch.where(r < 100, cols[:, 1].repeat(10)[:R], rnd)                   # the second tied column: a miss
    variants = {"exact": ref, "shifted": (ref + 1) % V, "tie_other": tie_other,
                "mixed": torch.where(r % 3 == 0, ref, torch.where(r % 3 == 1, torch.full_like(ref, pad), rnd))}
    m = {}
    for tag, t in variants.items():
        for n in (1, 3, 5, 131, 517, R):                                             # ragged row counts
            tt = t[:n].contiguous()
            live = (tt != pad) & (tt >= 0) & (tt < V)
            want = torch.stack([(live & (ref[:n] == tt)).sum(), live.sum()]).float()
            got = ops.argmax_hits(L[:n], tt, V, pad)
            m[f"argmax_mismatch_{tag}_{n}"] = float((got != want).sum())
    m["argmax_mismatch_empty"] = float((ops.argmax_hits(L[:0], ref[:0], V, pad) != 0).sum())
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_validation_metrics(model):
    import torch
    tok = model.tokenizer
    batch = _batch(model, 130, seed=13, pad_tail=9)
    model.training_loss(batch)
    gflat = model._rt().store.gflat
    g0 = gflat.clone()
    loss, acc = model.validation_metrics(batch)
    m = {"val_grad_changed": float((gflat != g0).sum())}
    m["val_loss_mismatch"] = float(loss != model.training_loss(batch, backward=False))
    with torch.no_grad():                                         # train.py:190-204 on the drop-in path
        y = batch[:, 1:].reshape(-1, 8)
        hidden = model.forward(batch[:, :-1].contiguous())
        logits = model.forward_token(hidden.reshape(-1, hidden.shape[-1]), y[:, :-1])
        out = torch.argmax(logits, dim=-1).flatten()              # train.py:153-166 compute_accuracy
        labels = y.flatten()
        mask = labels != tok.pad_id
        ref_acc = torch.sum(out[mask] == labels[mask]).type(torch.float32) / len(labels[mask])
    m["val_acc_mismatch"] = float(acc != ref_acc)
    m["val_acc_mismatch_int16"] = float(model.validation_metrics(batch.to(torch.int16))[1] != ref_acc)
    l_e, a_e = model.validation_metrics(torch.full_like(batch, tok.pad_id))
    m["val_empty_not_nan"] = float(not (torch.isnan(l_e) and torch.isnan(a_e)))
    print("val loss", float(loss), "acc", float(acc))
    assert_within(m, BOUNDS)
