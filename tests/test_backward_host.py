"""On the CPU: the fp64 stack the backward conformance tests score against (parity_metrics.stack64), and what the per-tensor
gradient metrics of tests/test_gpu_backward.py catch that the global gradient norm does not.

stack64 is checked against the oracle's stack under fp32 autograd, by torch.autograd.gradcheck, and on packed
sequences.  Then wiring defects are planted in the mock kernel layer (tests/mock_kernels.py) -- never in the product --
and the fused step of the host test model runs through them.  Each defect must fail the per-tensor / per-head bounds of
test_gpu_backward.BOUNDS; the table printed at the end also says whether the global relative gradient norm against the
oracle (bounded at 6e-2 by the model-level checks) would have let it through."""
import torch

import host_model
import mock_kernels
import parity_metrics as P
import test_gpu_backward as TB
from host_model import BF

GLOBAL_BOUND = 6e-2                     # grad_global_rel / lora_grad_global_rel of the model-level checks


def _sd(cfg, seed, dtype=torch.float64, scale=0.1):
    """Random weights of one stack (norm weights around 1)."""
    g = torch.Generator().manual_seed(seed)
    H, I, p = cfg.hidden, cfg.inner, cfg.prefix
    sd = {f"{p}.norm.weight": 1 + 0.1 * torch.randn(H, generator=g)}
    for l in range(cfg.n_layer):
        pre = f"{p}.layers.{l}."
        for n, shape in (("self_attn.q_proj", (H, H)), ("self_attn.k_proj", (H, H)), ("self_attn.v_proj", (H, H)),
                         ("self_attn.o_proj", (H, H)), ("mlp.gate_proj", (I, H)), ("mlp.up_proj", (I, H)),
                         ("mlp.down_proj", (H, I))):
            sd[pre + n + ".weight"] = scale * torch.randn(shape, generator=g)
        for n in ("input_layernorm", "post_attention_layernorm"):
            sd[pre + n + ".weight"] = 1 + 0.1 * torch.randn(H, generator=g)
    return {k: v.to(dtype) for k, v in sd.items()}


def _tables(inv, S):
    fr = torch.arange(S, dtype=torch.float32)[:, None] * inv.float()[None]
    return fr.cos(), fr.sin()


def test_stack64_matches_oracle_stack_in_fp32():
    from oracle import midi_oracle as O
    cfg = O.StackCfg("net", 2, 4, 64, 128)
    inv = O.default_inv_freq(cfg.head_dim)
    sd32 = {k: v.requires_grad_(True) for k, v in _sd(cfg, 0, torch.float32).items()}
    sd64 = {k: v.detach().double().requires_grad_(True) for k, v in sd32.items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 12, 64, generator=g)
    dy = torch.randn(2, 12, 64, generator=g)
    x32, x64 = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    y32 = O.llama_stack(sd32, cfg, x32, inv)
    y64 = P.stack64(sd64, cfg, x64, *_tables(inv, 12))
    y32.backward(dy)
    y64.backward(dy.double())
    assert P._rel(y32.detach().double(), y64.detach()) < 1e-5
    assert P._rel(x32.grad.double(), x64.grad) < 1e-5
    for k in sd32:
        assert P._rel(sd32[k].grad.double(), sd64[k].grad) < 1e-5, k


def test_stack64_gradcheck():
    from oracle import midi_oracle as O
    cfg = O.StackCfg("net", 2, 2, 16, 24)
    sd = {k: v.requires_grad_(True) for k, v in _sd(cfg, 2, scale=0.3).items()}
    cos, sin = _tables(O.default_inv_freq(cfg.head_dim), 5)
    x = torch.randn(1, 5, 16, generator=torch.Generator().manual_seed(3), dtype=torch.float64, requires_grad=True)
    names = list(sd)

    def f(x, *ws):
        return P.stack64(dict(zip(names, ws)), cfg, x, cos, sin)
    assert torch.autograd.gradcheck(f, (x, *sd.values()))


def test_stack64_segments_run_alone():
    """lengths: each packed sequence runs alone from position 0, so the gradients are the per-sequence sums."""
    from oracle import midi_oracle as O
    cfg = O.StackCfg("net", 2, 4, 64, 128)
    sd = {k: v.requires_grad_(True) for k, v in _sd(cfg, 4).items()}
    cos, sin = _tables(O.default_inv_freq(cfg.head_dim), 21)
    g = torch.Generator().manual_seed(5)
    x, dy = torch.randn(1, 21, 64, generator=g, dtype=torch.float64), torch.randn(1, 21, 64, generator=g, dtype=torch.float64)
    lengths = [5, 16]
    ws = list(sd.values())
    packed = torch.autograd.grad(P.stack64(sd, cfg, x, cos, sin, lengths), ws, dy)
    alone = [torch.autograd.grad(P.stack64(sd, cfg, xs, cos, sin), ws, d)
             for xs, d in zip(x.split(lengths, 1), dy.split(lengths, 1))]
    for n, gp, a, b in zip(sd, packed, *alone):
        assert P._rel(gp, a + b) < 1e-12, n
    whole = torch.autograd.grad(P.stack64(sd, cfg, x, cos, sin), ws, dy)
    assert P._rel(whole[0], packed[0]) > 1e-3            # the segments really are separate


# ------------------------------------------------------------------------------------------ planted defects
def _plant(monkeypatch, model, defect):
    """Patch the mock kernel layer's own entries (midi_b200.ops as installed by mock_kernels) with one wiring defect."""
    from midi_b200 import ops
    rt = model._rt()
    eng = rt.outer
    D, H = eng.cfg.head_dim, eng.cfg.hidden
    if defect == "dq_one_head_x1.02":
        orig = ops.attn_causal_bwd

        def attn_bwd(qkv, out, dout, lse, B, S, nh, D_, rope=None, impl=None):
            d = orig(qkv, out, dout, lse, B, S, nh, D_, rope=rope)
            d[:, D:2 * D] = (d[:, D:2 * D].float() * 1.02).to(BF)          # head 1 of q
            return d
        monkeypatch.setattr(ops, "attn_causal_bwd", attn_bwd)
    elif defect in ("ln2_ignores_accumulate", "dres_dropped_layer0_ln2"):
        orig = ops.rmsnorm_bwd
        ln2 = {w.ln2.data_ptr() for w in eng.layers}
        first_ln2 = eng.layers[0].ln2.data_ptr()

        def rmsnorm_bwd(dy, x, w, rstd, dres, dw, accumulate_dw):
            if defect == "ln2_ignores_accumulate" and w.data_ptr() in ln2:
                accumulate_dw = False
            if defect == "dres_dropped_layer0_ln2" and w.data_ptr() == first_ln2:
                dres = None
            return orig(dy, x, w, rstd, dres, dw, accumulate_dw)
        monkeypatch.setattr(ops, "rmsnorm_bwd", rmsnorm_bwd)
    elif defect == "lora_v_dt_unscaled_layer1":
        orig = ops.gemm
        lw = eng.layers[1].lora["v"]
        vb = lw.B.data_ptr()

        def gemm(A, B, M, N, K, **kw):
            out = orig(A, B, M, N, K, **kw)
            if B.data_ptr() == vb and kw.get("b_mn") and kw.get("out") is None:    # dts = dy B, then scaled
                out = (out.float() / lw.scale).to(BF)
            return out
        monkeypatch.setattr(ops, "gemm", gemm)
    elif defect == "rope_pair_sign_layer1":
        orig = ops.attn_causal_bwd
        calls = []

        def attn_bwd(qkv, out, dout, lse, B, S, nh, D_, rope=None, impl=None):
            calls.append(1)
            if len(calls) != 3 or rope is None:                          # backward runs layer 3, 2, 1, 0
                return orig(qkv, out, dout, lse, B, S, nh, D_, rope=rope)
            d = orig(qkv, out, dout, lse, B, S, nh, D_, rope=None)
            good, bad = d.clone(), d.clone()
            mock_kernels.rope_qk_(good, rope[0], rope[1], S, H, D_, backward=True)
            mock_kernels.rope_qk_(bad, rope[0], rope[1], S, H, D_, backward=False)
            for c in (1, 1 + D_ // 2):                                   # pair 1 of head 0 of q: sin term's sign flipped
                good[:, c] = bad[:, c]
            return good
        monkeypatch.setattr(ops, "attn_causal_bwd", attn_bwd)
    else:
        raise ValueError(defect)


def _scenario(model, batches, lora_scale=None):
    """fp64 / bf16-floor / fp32-oracle gradients of the (accumulated) steps over `batches`."""
    ref, fl, orc = {}, {}, {}
    for b in batches:
        _, r, f = TB._step_reference(model, b, lora_scale=lora_scale)
        _, o = host_model.oracle_padded(model, b, lora_scale)
        for acc, new in ((ref, r), (fl, f), (orc, o)):
            for n, t in new.items():
                if t is not None:
                    acc[n] = acc.get(n, 0) + t.double()
    return ref, fl, orc


def _step(model, batches, ref, fl, orc):
    """The fused step(s), the second and later accumulating -> (bounds the per-tensor metrics fail, global rel)."""
    for p in model.parameters():
        p.grad = None
    for i, b in enumerate(batches):
        model.training_loss(b, accumulate=i > 0)
    got = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    m = P.grad_report(got, ref, "step", TB._heads(model), fl, show=False)
    failed = [k for k, v, bound, ok in P.check_bounds(m, TB.BOUNDS) if not ok]
    return failed, host_model.global_rel(got, {n: orc[n] for n in got}), m


DEFECTS = [("dq_one_head_x1.02", "plain"), ("ln2_ignores_accumulate", "accumulate"),
           ("dres_dropped_layer0_ln2", "plain"), ("lora_v_dt_unscaled_layer1", "lora"),
           ("rope_pair_sign_layer1", "plain")]


def test_planted_defects_fail_per_tensor_metrics(monkeypatch):
    mock_kernels.install(monkeypatch)
    models = {"plain": host_model.tiny_model(0), "lora": host_model.add_lora(host_model.tiny_model(0))}
    models["accumulate"] = models["plain"]
    b1 = host_model.make_batch(models["plain"], 2, 17, seed=1)
    b2 = host_model.make_batch(models["plain"], 2, 17, seed=2)
    setups = {"plain": ([b1], None), "accumulate": ([b1, b2], None), "lora": ([b1], 2.0)}
    refs = {k: _scenario(models[k], batches, scale) for k, (batches, scale) in setups.items()}
    rows = []
    for name in setups:                                   # without a defect every bound holds
        failed, glob, m = _step(models[name], setups[name][0], *refs[name])
        assert not failed, (name, failed, m)
        rows.append((f"none ({name})", glob, []))
    for defect, name in DEFECTS:
        with monkeypatch.context() as mp:
            _plant(mp, models[name], defect)
            failed, glob, m = _step(models[name], setups[name][0], *refs[name])
        rows.append((defect, glob, failed))
    print(f"\n{'planted defect':28s} {'global rel':>10s}  global bound {GLOBAL_BOUND:g}   per-tensor bounds failed")
    for defect, glob, failed in rows:
        verdict = "-" if defect.startswith("none") else "lets it through" if glob <= GLOBAL_BOUND else "catches it"
        print(f"{defect:28s} {glob:10.3e}  {verdict:15s}  "
              f"{', '.join(failed) or '-'}")
    missed = [d for d, _, failed in rows[len(setups):] if not failed]
    assert not missed, f"planted defects the per-tensor metrics let through: {missed}"
