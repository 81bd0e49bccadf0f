"""The conformance metrics of tests/parity_metrics.py, judged by the bounds the GPU groups use (the tables of
gpu_checks.GROUPS), on the CPU: each corruption a kernel could plausibly make fails, while the same references
recomputed in fp32 with another summation order (and rounded to bf16 as a kernel would) pass.  Also the bound check
itself, and the bound tables of every GPU test."""
import importlib
import math

import pytest
import torch

import gpu_checks as G
import parity_metrics as P

BF = torch.bfloat16


def _fails(group, metrics):
    res = P.check_bounds(metrics, G.GROUPS[group].bounds)
    assert all(b is not None for _, _, b, _ in res), res
    return any(not ok for *_, ok in res)


# ------------------------------------------------------------------------------------------ the bound check
def _oks(metrics, bounds, info=()):
    return {k: ok for k, _, _, ok in P.check_bounds(metrics, bounds, info)}


def test_check_bounds_rules():
    bounds = [("a_long", 1.0), ("a", 2.0), ("min:c", 3.0)]
    res = P.check_bounds({"a_long_x": 1.5, "a_x": 1.5, "c": 3.0, "c_low": 2.9, "nan": math.nan, "t": 9.0},
                         bounds, info=("t",))
    assert res == [("a_long_x", 1.5, 1.0, False),      # the longer prefix, placed first, wins
                   ("a_x", 1.5, 2.0, True),
                   ("c", 3.0, 3.0, True),              # min: a lower bound
                   ("c_low", 2.9, 3.0, False),
                   ("nan", math.nan, None, False),     # matches no bound and is not informational
                   ("t", 9.0, None, True)]             # informational: reported with bound None
    assert _oks({"a": math.nan, "a_inf": math.inf}, bounds) == {"a": False, "a_inf": False}
    assert _oks({"a": 2.0, "c": math.inf}, bounds) == {"a": True, "c": True}


def test_renamed_metric_of_a_group_fails():
    """A metric whose name matches no bound of its group fails instead of dropping out of the check."""
    g = G.GROUPS["model_train"]
    good = {"loss_abs": 1e-3, "loss_ref": 8.0, "grad_global_rel": 1e-2, "grad_worst_rel": 3e-2}
    assert all(_oks(good, g.bounds, g.info).values())
    renamed = {("los_abs" if k == "loss_abs" else k): v for k, v in good.items()}
    assert _oks(renamed, g.bounds, g.info) == {"los_abs": False, "loss_ref": True, "grad_global_rel": True,
                                                "grad_worst_rel": True}


def _bound_tables():
    for name, g in G.GROUPS.items():
        yield name, g.bounds, g.info
    for mod in ("test_gpu_ragged", "test_gpu_recompute", "test_gpu_sample_seq", "test_gpu_backward"):
        yield mod, importlib.import_module(mod).BOUNDS, ()


def test_bound_tables_have_no_dead_or_doubled_entries():
    """No entry sits behind an earlier prefix of itself (it could never match), and no informational metric also has
    a bound."""
    problems = []
    for name, bounds, info in _bound_tables():
        prefixes = [p.removeprefix("min:") for p, _ in bounds]
        problems += [(name, "shadowed", b, a) for i, b in enumerate(prefixes) for a in prefixes[:i] if b.startswith(a)]
        problems += [(name, "bounded and informational", n) for n in info if any(n.startswith(p) for p in prefixes)]
    assert not problems, problems


# ------------------------------------------------------------------------------------------ attention rows


def _randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _attn32_reordered(q, k, v):
    """fp32 causal attention with the keys summed in reverse order."""
    q, k, v = q.float(), k.float(), v.float()
    S = q.shape[-2]
    s = (q @ k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool), 1), float("-inf"))
    p = torch.softmax(s, -1)
    return p.flip(-1) @ v.flip(-2)


@pytest.fixture(scope="module")
def attn_ref():
    # eight heads at S = 2047: the last 64-row tile is ragged (63 rows)
    q, k, v, do = (_randn(1, 8, 2047, 64, seed=i) for i in range(4))
    o64, _, dq64, _, _ = P.attn_ref64(q, k, v, do, 0, 0.125)
    return q, k, v, o64, dq64


def test_attention_rows_pass_when_only_rounding_differs(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    o32 = _attn32_reordered(q, k, v)
    assert not _fails("attn_edges", {"ae_wg_o_row": P.row_worst(o32, o64),
                                     "ae_wg_dq_row": P.row_worst(dq64.float(), dq64)})
    # bf16 outputs, as the kernels store them
    assert not _fails("attn_edges", {"ae_wg_o_row": P.row_worst(o32.to(BF), o64),
                                     "ae_wg_dq_row": P.row_worst(dq64.to(BF), dq64)})


def test_attention_zeroed_last_row_of_ragged_tile_fails(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    y = _attn32_reordered(q, k, v).to(BF)
    y[0, 1, 2046] = 0          # the last row of the ragged tile, one head
    # a global relative norm barely moves ...
    glob = float((y.double() - o64).norm() / o64.norm())
    assert glob < 6e-3
    # ... the per-row score does not
    assert _fails("attn_edges", {"ae_wg_o_row": P.row_worst(y, o64)})
    g = dq64.to(BF)
    g[0, 0, 2046] = 0
    assert _fails("attn_edges", {"ae_wg_dq_row": P.row_worst(g, dq64)})


def test_attention_nan_fails(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    y = o64.to(BF)
    y[0, 0, 1000, 7] = float("nan")
    assert P.row_worst(y, o64) == math.inf
    assert _fails("attn_edges", {"ae_wg_o_row": P.row_worst(y, o64)})


def test_zero_reference_rows_use_the_input_scale_floor():
    ref = torch.zeros(2, 4, 64, dtype=torch.float64)
    noise = torch.full_like(ref, 1e-7)
    assert P.row_worst(noise, ref, atol=8e-3) < 1e-4
    assert P.row_worst(noise + 1.0, ref, atol=8e-3) > 1.0


@pytest.fixture(scope="module")
def gemm_ref():
    a = _randn(257, 300, seed=10).to(BF)
    b = (_randn(520, 300, seed=11) * 0.05).to(BF)
    return a, b, a.double() @ b.double().T


def _gm(y, ref, family="store", **kw):
    return {f"gm_{family}_{k}": v for k, v in P.exact_metrics(y, ref, **kw).items()}


def test_gemm_reordered_fp32_passes(gemm_ref):
    a, b, ref = gemm_ref
    y = (a.float().flip(1) @ b.float().flip(1).T).to(BF)
    m = _gm(y, ref)
    assert m["gm_store_maxulp"] <= 1 and not _fails("gemm_matrix", m)


def test_gemm_group_moved_by_4_ulp_fails(gemm_ref):
    a, b, ref = gemm_ref
    y = (a.float() @ b.float().T).to(BF)
    # an 8-column group whose references are all well above the noise floor
    rms = float(ref.pow(2).mean().sqrt())
    big = (ref.abs() > 0.5 * rms).view(257, -1, 8).all(-1)
    r, g = (int(i) for i in torch.nonzero(big)[0])
    bits = y.view(torch.int16)
    bits[r, 8 * g:8 * g + 8] += 4          # 4 ulp away from zero (sign-magnitude bits)
    m = _gm(y, ref)
    assert m["gm_store_maxulp"] >= 4
    assert _fails("gemm_matrix", m)


def test_chained_epilogue_flip_passes_but_3_ulp_fails(gemm_ref):
    a, b, ref = gemm_ref
    r = (_randn(257, 520, seed=12)).to(BF)
    acc = P.round_bf16(ref)
    want = (acc + r.double()).float().to(BF)
    y = ((a.float().flip(1) @ b.float().flip(1).T).to(BF).float() + r.float()).to(BF)
    m = _gm(y, acc + r.double(), "residual", want=want, inter=ref)
    assert not _fails("gemm_matrix", m)
    y.view(torch.int16)[5, 16:24] += 3
    assert _fails("gemm_matrix", _gm(y, acc + r.double(), "residual", want=want, inter=ref))


def test_gemm_nan_fails(gemm_ref):
    a, b, ref = gemm_ref
    y = ref.to(BF)
    y[100, 200] = float("nan")
    assert _fails("gemm_matrix", _gm(y, ref))


def test_sentinels():
    M, N, ldc = 5, 13, 32
    buf = P.nan_buffer((M + 3, ldc))
    buf[:M, :N] = 1.0
    buf[:M, N:16] = 0.0
    inside, pad = (slice(0, M), slice(0, N)), (slice(0, M), slice(N, 16))
    rep = P.sentinel_report(buf, inside, pad)
    assert rep == {"sentinels_changed": 0.0, "nan_in_range": 0.0, "padcols_nonzero": 0.0}
    assert not _fails("gemm_matrix", {f"gm_{k}": v for k, v in rep.items()})
    # one sentinel overwritten (a store past the row, or into the next row's pitch)
    bad = buf.clone()
    bad[M, 0] = 0.0
    assert P.sentinel_report(bad, inside, pad)["sentinels_changed"] == 1
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})
    # one output never written
    bad = buf.clone()
    bad[M - 1, N - 1] = float("nan")
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})
    # a padding column not zeroed
    bad = buf.clone()
    bad[0, 15] = float("nan")
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})


def test_poisoned_operand_keeps_values_and_pads_with_nan():
    v = _randn(3, 5, seed=1).to(BF)
    t = P.poisoned(v, 4, 8)
    assert torch.equal(t[:3, :5], v)
    assert bool(torch.isnan(t[:3, 5:].float()).all()) and bool(torch.isnan(t[3].float()).all())


# ------------------------------------------------------------------------------------------ train-step references
def _ex(prefix, family, y, ref, **kw):
    return {f"{prefix}_{family}_{k}": v for k, v in P.exact_metrics(y, ref, **kw).items()}


def test_rmsnorm_bwd64_is_fp64_autograd():
    x, dy, dres = _randn(7, 40, seed=20), _randn(7, 40, seed=21), _randn(7, 40, seed=22)
    w = 1 + 0.1 * _randn(40, seed=23)
    xa, wa = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    (wa * xa * torch.rsqrt(xa.pow(2).mean(-1, keepdim=True) + 1e-6)).backward(dy)
    dx, dw = P.rmsnorm_bwd64(dy, x, w, dres=dres)
    assert torch.allclose(dx, xa.grad + dres, rtol=1e-12, atol=1e-12)
    assert torch.allclose(dw, wa.grad, rtol=1e-12, atol=1e-12)
    # the rstd the backward is handed replaces the exact one
    r = torch.rsqrt(x.pow(2).mean(-1) + 1e-6)
    assert torch.allclose(P.rmsnorm_bwd64(dy, x, w, r, dres)[0], dx, rtol=1e-12, atol=1e-12)


def test_rmsnorm_dw_from_one_cta_partial_fails():
    """dw is the column sum over every row; one CTA's partial (the rows of a grid-stride loop over 528 CTAs) fails."""
    M, H = 5000, 768
    dy, x = _randn(M, H, seed=24).to(BF), _randn(M, H, seed=25).to(BF)
    w = (1 + 0.1 * _randn(H, seed=26)).to(BF)
    dx64, dw64 = P.rmsnorm_bwd64(dy, x, w)
    r = torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-6)
    contrib = dy.float() * (x.float() * r)
    full = contrib.flip(0).sum(0).to(BF)                 # fp32 in another order, one rounding
    assert not _fails("rmsnorm_exact", _ex("rn", "dw", full, dw64))
    part = contrib[0::528].sum(0).to(BF)
    assert _fails("rmsnorm_exact", _ex("rn", "dw", part, dw64))
    assert not _fails("rmsnorm_exact", _ex("rn", "dx", dx64.float().to(BF), dx64))


def test_ce64_is_fp64_cross_entropy():
    V, ign = 37, 5
    z = _randn(11, V, seed=30) * 3
    t = torch.randint(0, V, (11,), generator=torch.Generator().manual_seed(31))
    t[::4] = ign
    za = z.clone().requires_grad_(True)
    loss = torch.nn.functional.cross_entropy(za, t, ignore_index=ign)
    (loss * 0.5).backward()
    lse, row_loss, mean, count, d = P.ce64(z, t, V, ign, grad_scale=0.5)
    assert count == int((t != ign).sum()) and abs(mean - float(loss.detach())) < 1e-12
    assert torch.allclose(lse, torch.logsumexp(z, -1), rtol=1e-13)
    assert torch.allclose(d, za.grad, rtol=1e-12, atol=1e-14)
    # targets -1 and V count as ignored: zero loss and gradient on their rows
    t2 = t.clone()
    t2[1], t2[2] = -1, V
    _, rl2, _, c2, d2 = P.ce64(z, t2, V, ign)
    assert c2 == count - 2 + int(t[1] == ign) + int(t[2] == ign)
    assert float(rl2[1:3].abs().max()) == 0 and float(d2[1:3].abs().max()) == 0


def test_ce_zeroed_last_vector_fails():
    V, R = 3406, 200
    z = (_randn(R, V, seed=32) * 3).to(BF)
    t = torch.randint(0, V, (R,), generator=torch.Generator().manual_seed(33))
    d64 = P.ce64(z, t, V, 0)[4]
    y = ((torch.exp(z.float() - torch.logsumexp(z.float(), -1, keepdim=True))
          - torch.nn.functional.one_hot(t, V).float()) / R).to(BF)         # fp32, another evaluation order
    assert not _fails("loss_optim_exact", _ex("lo", "ce_bwd", y, d64))
    y[:, 3400:] = 0                                                          # the masked last vector, 3400..3405
    assert _fails("loss_optim_exact", _ex("lo", "ce_bwd", y, d64))


def test_adamw64_is_torch_adamw_in_fp64():
    n = 4 * 256
    p0, g = _randn(n, seed=40) * 0.05, _randn(n, seed=41) * 0.5
    nodecay = torch.tensor([0, 0, 1, 1], dtype=torch.uint8)
    pa, pb = torch.nn.Parameter(p0[:512].clone()), torch.nn.Parameter(p0[512:].clone())
    opt = torch.optim.AdamW([dict(params=[pa], weight_decay=5.0), dict(params=[pb], weight_decay=0.0)], lr=1e-2,
                            betas=(0.9, 0.99), eps=1e-8)
    p, m, v = p0, torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step in (1, 2, 3):
        pa.grad, pb.grad = g[:512] * 0.3, g[512:] * 0.3
        opt.step()
        p, m, v = P.adamw64(p, g, m, v, nodecay, 1e-2, 0.9, 0.99, 1e-8, 5.0, step, coef=0.3)
        assert torch.allclose(p, torch.cat([pa, pb]).detach(), rtol=1e-12, atol=1e-15)
        assert torch.allclose(m, torch.cat([opt.state[pa]["exp_avg"], opt.state[pb]["exp_avg"]]), rtol=1e-12)


def test_adamw_decay_on_a_nodecay_block_fails():
    n = 64 * 256
    p0 = (_randn(n, seed=42) * 0.05).to(BF)
    g = (_randn(n, seed=43) * 0.5).to(BF)
    g[256:512] = 0                                        # decay alone moves this block
    nodecay = torch.zeros(n // 256, dtype=torch.uint8)
    nodecay[1::2] = 1
    m, v = torch.zeros(n), torch.zeros(n)
    args = (0.9, 0.99, 1e-8, 5.0, 1)
    p64 = P.adamw64(p0, g, m, v, nodecay, 1e-2, *args)[0]
    assert not _fails("loss_optim_exact", _ex("lo", "adamw_p", p64.float().to(BF), p64))
    wrong = P.adamw64(p0, g, m, v, torch.zeros_like(nodecay), 1e-2, *args)[0]
    assert _fails("loss_optim_exact", _ex("lo", "adamw_p", wrong.float().to(BF), p64))
    inverted = P.adamw64(p0, g, m, v, 1 - nodecay, 1e-2, *args)[0]
    assert _fails("loss_optim_exact", _ex("lo", "adamw_p", inverted.float().to(BF), p64))


@pytest.mark.parametrize("layout", ["outer", "inner"])
def test_embed_bwd64_is_fp64_embedding_backward(layout):
    V, H, pad = 50, 16, 17
    g = torch.Generator().manual_seed(50)
    per_row = 8 if layout == "outer" else 7
    ids = torch.randint(0, V, (30, per_row), generator=g)
    ids[3, 2] = pad
    table = _randn(V, H, seed=51).requires_grad_(True)
    if layout == "outer":
        dout = _randn(30, H, seed=52)
        torch.nn.functional.embedding(ids, table, padding_idx=pad).sum(-2).backward(dout)
        ref = P.embed_bwd64(ids, dout, V, 8, 1, 0, 0, pad)
    else:
        dout = _randn(30 * 8, H, seed=52)
        torch.nn.functional.embedding(ids, table, padding_idx=pad).backward(dout.view(30, 8, H)[:, 1:])
        dout[0::8] = float("nan")                           # rows e*8 are never read
        ref = P.embed_bwd64(ids, dout, V, 7, 8, 1, 1, pad)
    assert torch.allclose(ref, table.grad, rtol=1e-12, atol=1e-12)
    # ids outside [0, V) contribute nothing
    ids2 = ids.clone()
    ids2[0, 0], ids2[1, 1] = -1, V
    assert bool(torch.isfinite(P.embed_bwd64(ids2, dout, V, per_row, *((1, 0, 0) if layout == "outer" else (8, 1, 1)),
                                             pad)).all())


def test_swiglu_bwd64_is_fp64_autograd():
    gu, d = _randn(9, 48, seed=60) * 6, _randn(9, 24, seed=61)
    a = gu.clone().requires_grad_(True)
    (torch.nn.functional.silu(a[:, :24]) * a[:, 24:]).backward(d)
    assert torch.allclose(P.swiglu_bwd64(gu, d), a.grad, rtol=1e-12, atol=1e-14)


def _rope_tables(D, S):
    half = D // 2
    ang = torch.arange(S, dtype=torch.float64)[:, None] * (10000.0 ** (-torch.arange(half, dtype=torch.float64) / half))
    return ang.cos(), ang.sin()


@pytest.mark.parametrize("D", [64, 256])
def test_rope_bwd64_is_the_transpose_of_the_rotation(D):
    S, half = 9, D // 2
    cos, sin = _rope_tables(D, S)
    x = _randn(2, 3, S, D, seed=70).requires_grad_(True)
    gy = _randn(2, 3, S, D, seed=71)
    c, s = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)
    (x * c + torch.cat([-x[..., half:], x[..., :half]], -1) * s).backward(gy)
    assert torch.allclose(P.rope_bwd64(gy, cos, sin, torch.arange(S)), x.grad, rtol=1e-12, atol=1e-12)


def test_rope_swapped_pair_fails():
    """The forward is an exact claim against the three-rounding chain; one rotated pair stored swapped fails, as it
    does in the backward's per-element score."""
    D, S, nh = 64, 37, 4
    cos, sin = (t.to(BF) for t in _rope_tables(D, S))
    x = _randn(S, nh, D, seed=72).to(BF)
    pos = torch.arange(S).view(S, 1)
    want = G._rope_chain64(x, cos, sin, pos)[0].float().to(BF)
    bad = want.clone()
    bad[5, 2, 3], bad[5, 2, 3 + D // 2] = want[5, 2, 3 + D // 2], want[5, 2, 3]
    assert not _fails("rope_exact", {"ro_fwd_mismatch": G._ne(want, want)})
    assert _fails("rope_exact", {"ro_fwd_mismatch": G._ne(bad, want)})
    g64 = P.rope_bwd64(x, cos, sin, pos)
    y = g64.float().to(BF)
    assert not _fails("rope_exact", _ex("ro", "bwd", y, g64))
    y[5, 2, 3], y[5, 2, 3 + D // 2] = g64[5, 2, 3 + D // 2].float().to(BF), g64[5, 2, 3].float().to(BF)
    assert _fails("rope_exact", _ex("ro", "bwd", y, g64))
