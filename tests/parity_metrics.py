"""Metrics that compare a bf16 kernel result with a high-precision reference element by element or row by row, the
NaN sentinel / poisoned-input buffers the conformance groups of gpu_checks.py build their operands in, the fp64
attention references they are scored against, and the one check that judges every GPU test's metrics by its bounds.

Global norms hide localized errors: a wrong 8-column group in one row of a 1000 x 1024 GEMM, or a zeroed last row of
one attention head, moves a relative Frobenius norm by less than its usual bound.  These helpers score the worst
element or the worst row instead; grad_report does the same for every gradient of a backward pass, against the fp64
stack (stack64, train_loss64) and as a ratio to the bf16 eager oracle's error.  Pure PyTorch on any device, so tests/test_parity_metrics.py can show on the CPU that
each metric fails on the corruptions it is meant to catch."""
from __future__ import annotations

import math

import torch

BF = torch.bfloat16
NAN = float("nan")


# ------------------------------------------------------------------------------------------ bounds
def check_bounds(metrics: dict, bounds, info=()) -> list:
    """(name, value, bound, ok) for every metric.

    bounds: (prefix, bound) pairs; the first prefix a name starts with gives its bound.  A "min:" prefix is a lower
            bound (ok when value >= bound), any other an upper bound (ok when value <= bound and value is not NaN).
    info  : the names reported without a bound (timings, lengths, distances kept for the record).  Any other metric
            that matches no prefix fails, so a renamed or misspelt metric cannot drop out of the check unnoticed."""
    rows = []
    for k, v in metrics.items():
        hit = next(((p, b) for p, b in bounds if k.startswith(p.removeprefix("min:"))), None)
        if hit is None:
            rows.append((k, v, None, k in info))
        elif hit[0].startswith("min:"):
            rows.append((k, v, hit[1], v >= hit[1]))
        else:
            rows.append((k, v, hit[1], v <= hit[1] and not math.isnan(v)))
    return rows


def assert_within(metrics: dict, bounds, info=()):
    """check_bounds as a test assertion; prints the metrics."""
    print(metrics)
    bad = [(k, v, b) for k, v, b, ok in check_bounds(metrics, bounds, info) if not ok]
    assert not bad, f"out of bounds or without one: {bad}"


# ------------------------------------------------------------------------------------------ per-element exactness
def ordered_bf16(t: torch.Tensor) -> torch.Tensor:
    """bf16 bit patterns mapped to integers that are monotonic in the value (for ulp distances)."""
    i = t.contiguous().view(torch.int16).int()
    return torch.where(i >= 0, i, -(i & 0x7FFF))


def round_bf16(x: torch.Tensor) -> torch.Tensor:
    """x (fp64) rounded to bf16 and returned as fp64: one rounding point of a kernel's epilogue, restated."""
    return x.to(torch.float32).to(BF).double()


def exact_metrics(y: torch.Tensor, ref64: torch.Tensor, want: torch.Tensor | None = None,
                  inter: torch.Tensor | None = None) -> dict:
    """y (bf16) against an fp64 reference of the same bf16 operands.

    want : the correctly rounded result the kernel should return (default bf16(ref64)); epilogues with several
           rounding points pass the fp64 chain rounded at the same points.
    inter: magnitude of the value rounded at an earlier rounding point (the bf16 accumulator before a residual add or
           a rotation).  fp32 summation order may flip that rounding by one ulp, which moves a result that cancels
           by many of its own ulps; such elements are left out of the ulp count and get that ulp in their tolerance.
           Where they do not cancel, a flip can still cost two ulps of the result: an fp32 accumulator exactly on a
           bf16 midpoint rounds to even, one ulp away from the fp64 one, and the sum with the residual then lands on
           the next midpoint and rounds away from the reference.

    Returns frac (elements != want), maxulp (largest ulp distance to want among elements that are not tiny) and
    err_over_tol (worst |y - ref| / (2^-7 |ref| [+ 2^-7 inter] + 1e-3 rms)).  A non-finite y makes maxulp and
    err_over_tol infinite."""
    y = y.contiguous()
    ref64 = ref64.double()
    if want is None:
        want = ref64.to(torch.float32).to(BF)
    want = want.to(BF).contiguous()
    finite = bool(torch.isfinite(y).all())
    rms = float(ref64.pow(2).mean().sqrt()) if ref64.numel() else 0.0
    big = ref64.abs() > 0.05 * rms
    tol = ref64.abs() * 2.0 ** -7 + 1e-3 * rms + 1e-30
    if inter is not None:
        inter = inter.double().abs()
        big &= ref64.abs() >= inter
        tol = tol + inter * 2.0 ** -7
    ulp = (ordered_bf16(y) - ordered_bf16(want)).abs()
    maxulp = float(ulp[big].max()) if bool(big.any()) else 0.0
    err = float(((y.double() - ref64).abs() / tol).max()) if y.numel() else 0.0
    if not finite:
        maxulp, err = float("inf"), float("inf")
    return {"frac": float((y != want).float().mean()) if y.numel() else 0.0, "maxulp": maxulp, "err_over_tol": err}


# ------------------------------------------------------------------------------------------ per-row error
def row_rel(y: torch.Tensor, ref: torch.Tensor, floor_frac: float = 0.05, atol: float = 0.0) -> torch.Tensor:
    """Relative L2 error of every row (last dimension) of y against ref, as a tensor of the leading shape.

    The denominator is the row norm of ref, floored at floor_frac x the median row norm so that near-zero rows do not
    divide by zero, and at `atol`, a row norm on the scale of the inputs, for references that are zero as a whole (the
    dq of a one-key attention is exactly 0; its kernel value is fp32 rounding noise).  A row of y with a non-finite
    value scores +inf."""
    y64, r64 = y.double(), ref.double()
    err = (y64 - r64).norm(dim=-1)
    nrm = r64.norm(dim=-1)
    floor = floor_frac * float(nrm.flatten().median()) if nrm.numel() else 0.0
    score = err / nrm.clamp_min(max(floor, atol, 1e-30))
    return torch.where(torch.isfinite(y64).all(-1), score, torch.full_like(score, float("inf")))


def row_worst(y: torch.Tensor, ref: torch.Tensor, floor_frac: float = 0.05, atol: float = 0.0) -> float:
    """Worst per-row relative error (see row_rel): one score per (batch, head, row) of an attention tensor."""
    r = row_rel(y, ref, floor_frac, atol)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------ sentinels / poison
def nan_buffer(shape, dtype=BF, device="cpu") -> torch.Tensor:
    return torch.full(shape, NAN, dtype=dtype, device=device)


def poisoned(values: torch.Tensor, rows: int, ld: int) -> torch.Tensor:
    """A [rows, ld] buffer filled with NaN whose top-left corner holds `values` (2-D).  Kernels get its data pointer
    and ld: an operand read past its logical extent turns the result into NaN instead of passing silently."""
    buf = nan_buffer((rows, ld), values.dtype, values.device)
    buf[:values.shape[0], :values.shape[1]] = values
    return buf


def sentinel_report(buf: torch.Tensor, inside, zero=None) -> dict:
    """buf was NaN-filled before the kernel wrote the region `inside` (an index expression, e.g. (slice(0, M),
    slice(0, N))).  Returns the number of sentinels outside `inside` and `zero` that changed, the number of elements of
    `inside` still NaN (not written) and, for the padding region `zero` that must be written as exact zeros, the number
    of elements that are not 0."""
    mask_in = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    mask_in[inside] = True
    mask_zero = torch.zeros_like(mask_in)
    if zero is not None:
        mask_zero[zero] = True
    isnan = torch.isnan(buf.float())
    out = {"sentinels_changed": float((~isnan & ~mask_in & ~mask_zero).sum()),
           "nan_in_range": float((isnan & mask_in).sum())}
    if zero is not None:
        out["padcols_nonzero"] = float(((buf.float() != 0) & mask_zero).sum())
    return out


# ------------------------------------------------------------------------------------------ fp64 references
def attn_ref64(q, k, v, do, off, scale=0.125, o_in=None):
    """fp64 causal attention (query q sees keys <= q + off) and its gradients; tensors (B, h, S, D).

    The backward is written out (dS = P (dP - delta), delta = rowsum(dO o)) because the kernels take o as an input: with
    o_in (the bf16 o handed to the backward) delta is formed from it, so the reference is the exact gradient of the
    inputs the kernel gets.  Without o_in (o exact) this is fp64 autograd.  It matters where softmax saturates: there
    dS cancels almost completely and the rounding of o alone moves dq, dk far more than any kernel error."""
    q, k, v, do = (t.detach().double() for t in (q, k, v, do))
    s = (q @ k.transpose(-1, -2)) * scale
    Sq, Sk = q.shape[-2], k.shape[-2]
    m = torch.arange(Sk, device=q.device)[None] > (torch.arange(Sq, device=q.device)[:, None] + off)
    s = s.masked_fill(m, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.softmax(s, -1)
    o = p @ v
    delta = (do * (o if o_in is None else o_in.double())).sum(-1, keepdim=True)
    ds = p * (do @ v.transpose(-1, -2) - delta)
    return o, lse, ds @ k * scale, ds.transpose(-1, -2) @ q * scale, p.transpose(-1, -2) @ do


def rope_bwd64(g, cos, sin, pos):
    """gradient w.r.t. the pre-rotation projection: the transpose of x' = x c + rotate_half(x) s, in fp64 at `pos`
    (g (..., D), tables [positions, D/2])."""
    half = g.shape[-1] // 2
    c, s = cos.double()[pos], sin.double()[pos]
    g1, g2 = g[..., :half].double(), g[..., half:].double()
    return torch.cat([g1 * c + g2 * s, g2 * c - g1 * s], -1)


def rmsnorm_bwd64(dy, x, w, rstd=None, dres=None, eps=1e-6):
    """RMSNorm y = w * x * rstd backward in fp64 over rows of (M, H): (dx, dw) with dx = [dres +] rstd (dn - n mean(dn n)),
    dn = dy w, n = x rstd, and dw = sum over rows of dy n.  rstd: the per-row value the backward is handed (the forward
    kernel's fp32 rstd); None = exact 1 / sqrt(mean(x^2) + eps), which makes this fp64 autograd."""
    dy, x, w = dy.double(), x.double(), w.double()
    r = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + eps) if rstd is None else rstd.double().view(-1, 1)
    n, dn = x * r, dy * w
    dx = r * (dn - n * (dn * n).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.double()
    return dx, (dy * n).sum(0)


def ce64(logits, targets, V, ignore_index, grad_scale=1.0):
    """Mean cross-entropy over rows of logits[:, :V] in fp64, rows whose target is ignore_index or outside [0, V)
    ignored: (lse [R], row_loss [R] (0 on ignored rows), mean loss, count, dlogits [R, V] = (softmax - onehot) *
    grad_scale / max(count, 1) on live rows, 0 on ignored ones)."""
    z = logits[:, :V].double()
    t = targets.long()
    live = (t != ignore_index) & (t >= 0) & (t < V)
    lse = torch.logsumexp(z, -1)
    tc = torch.where(live, t, torch.zeros_like(t))
    row_loss = torch.where(live, lse - z.gather(1, tc[:, None])[:, 0], torch.zeros_like(lse))
    count = int(live.sum())
    mean = float(row_loss.sum()) / count if count else 0.0
    d = torch.exp(z - lse[:, None])
    d[torch.arange(len(t), device=z.device)[live], t[live]] -= 1.0
    d = torch.where(live[:, None], d * (grad_scale / max(count, 1)), torch.zeros_like(d))
    return lse, row_loss, mean, count, d


def adamw64(p, g, m, v, nodecay, lr, b1, b2, eps, wd, step, coef=1.0):
    """One torch.optim.AdamW step (decoupled decay, bias correction) in fp64 over a flat buffer, with the gradient
    multiplied by the clip coefficient first and the decay skipped on the 256-element blocks nodecay marks: (p, m, v)
    unrounded.  The kernel stores p in bf16 (one rounding) and m, v in fp32."""
    p, g, m, v = p.double(), g.double() * float(coef), m.double(), v.double()
    decay = torch.where(nodecay.bool().repeat_interleave(256), torch.ones_like(p), torch.full_like(p, 1.0 - lr * wd))
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    denom = v.sqrt() / math.sqrt(1 - b2 ** step) + eps
    return p * decay - lr / (1 - b1 ** step) * (m / denom), m, v


def embed_bwd64(ids, dout, V, per_row, row_stride, row_inner, row_off, pad_id):
    """Embedding backward in fp64: row v of the [V, H] result sums the gradient rows of every id i == v, where id i (flat
    index) reads row (i // per_row) * row_stride + (i % per_row) * row_inner + row_off of dout; ids outside [0, V) and
    pad_id contribute nothing (the pad row is 0).  Rows no valid id reads are never touched, so they may hold NaN."""
    ids = ids.reshape(-1).long()
    i = torch.arange(ids.numel(), device=ids.device)
    keep = (ids >= 0) & (ids < V) & (ids != pad_id)
    rows = (i // per_row) * row_stride + (i % per_row) * row_inner + row_off
    out = torch.zeros(V, dout.shape[1], dtype=torch.float64, device=dout.device)
    return out.index_add_(0, ids[keep], dout[rows[keep]].double())


def swiglu_bwd64(gu, dact):
    """act = silu(g) u on packed [rows, 2I] = [g | u]: (dg | du) in fp64 = (dact u silu'(g) | dact silu(g))."""
    I = gu.shape[1] // 2
    g, u, d = gu[:, :I].double(), gu[:, I:].double(), dact.double()
    sg = torch.sigmoid(g)
    return torch.cat([d * u * sg * (1 + g * (1 - sg)), d * g * sg], 1)


# ------------------------------------------------------------------------------------------ fp64 stack, gradient report
def stack64(sd, cfg, x, cos, sin, lengths=None):
    """One Llama stack (hf modeling_llama.py:303-332, :421) entirely in float64 and differentiable by torch autograd:
    RMSNorm, q/k/v, RoPE from the given tables, causal softmax over 1/sqrt(D) scores, o_proj with residual, SwiGLU MLP
    with residual, final norm.  Unlike oracle.midi_oracle.llama_stack nothing is cast to fp32 on the way.

    sd     : {parameter name: tensor} under cfg.prefix (layers 0 .. cfg.n_layer - 1 and the final norm), upcast here;
             LoRA runs pass oracle.midi_oracle.lora_effective_sd over fp64 leaves
    x      : (B, S, H) inputs_embeds
    cos/sin: RoPE tables [>= S, D/2] indexed by position (the engine's ops.rope_table, upcast)
    lengths: x is (1, sum(lengths), H) holding consecutive sequences, each run alone from position 0 (packed rows)."""
    if lengths is not None:
        parts = torch.split(x, [int(n) for n in lengths], dim=1)
        return torch.cat([stack64(sd, cfg, t, cos, sin) for t in parts], 1)
    B, S, H = x.shape
    nh = cfg.n_head
    D = H // nh
    c, s = cos[:S].double(), sin[:S].double()
    mask = torch.ones(S, S, dtype=torch.bool, device=x.device).triu(1)
    p = cfg.prefix

    def w(name):
        return sd[name].double()

    def norm(t, g):
        return g * (t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + cfg.eps))

    def rope(t):
        t1, t2 = t[..., :D // 2], t[..., D // 2:]
        return torch.cat((t1 * c - t2 * s, t2 * c + t1 * s), -1)

    x = x.double()
    for l in range(cfg.n_layer):
        pre = f"{p}.layers.{l}."
        n1 = norm(x, w(pre + "input_layernorm.weight"))
        q, k, v = (torch.nn.functional.linear(n1, w(pre + f"self_attn.{t}_proj.weight")).view(B, S, nh, D).transpose(1, 2)
                   for t in "qkv")
        sc = (rope(q) @ rope(k).transpose(-1, -2)) * (1.0 / math.sqrt(D))
        a = torch.softmax(sc.masked_fill(mask, float("-inf")), -1) @ v
        x = x + torch.nn.functional.linear(a.transpose(1, 2).reshape(B, S, H), w(pre + "self_attn.o_proj.weight"))
        n2 = norm(x, w(pre + "post_attention_layernorm.weight"))
        act = torch.nn.functional.silu(torch.nn.functional.linear(n2, w(pre + "mlp.gate_proj.weight")))
        x = x + torch.nn.functional.linear(act * torch.nn.functional.linear(n2, w(pre + "mlp.up_proj.weight")),
                                           w(pre + "mlp.down_proj.weight"))
    return norm(x, w(f"{p}.norm.weight"))


def train_loss64(sd, cfg, batch, rope_net, rope_tok, sample_idx=None):
    """train.py:168-185 in float64 over stack64: the embedding sum (pad rows contribute nothing), the event-level stack,
    the token-level input [hidden, embed(y[:, :-1])], the token-level stack, lm_head and the mean cross-entropy over
    non-pad targets.  cfg: oracle.midi_oracle.ModelCfg; rope_net / rope_tok: (cos, sin) of each stack;
    sample_idx: train.py --sample-seq's event positions (negative ones count from the end)."""
    F = torch.nn.functional
    x, y = batch[:, :-1].long(), batch[:, 1:].long()
    B, S, T = x.shape
    e = F.embedding(x, sd["net.embed_tokens.weight"].double(), padding_idx=cfg.pad_id).sum(-2)
    hidden = stack64(sd, cfg.net, e, *rope_net)
    if sample_idx is not None:
        hidden, y = hidden[:, list(sample_idx)], y[:, list(sample_idx)]
    hidden, y = hidden.reshape(-1, hidden.shape[-1]), y.reshape(-1, T)
    xe = F.embedding(y[:, :-1], sd["net_token.embed_tokens.weight"].double(), padding_idx=cfg.pad_id)
    h = stack64(sd, cfg.net_token, torch.cat([hidden[:, None], xe], 1), *rope_tok)
    logits = F.linear(h, sd["lm_head.weight"].double())
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), y.reshape(-1), ignore_index=cfg.pad_id)


def grad_kind(name: str, t: torch.Tensor) -> str:
    """Which per-block metrics a gradient gets: "dx" (input gradient, per token row), "table" (embedding / lm_head:
    relative norm only), "lora" (A / B), "qkv" (row blocks are heads), "o" (column blocks are heads), "mlp", "norm"."""
    if name.startswith("dx"):
        return "dx"
    if "embed_tokens" in name or name.startswith("lm_head"):
        return "table"
    if ".lora_" in name:
        return "lora"
    if any(f".{t}_proj." in name for t in "qkv"):
        return "qkv"
    if ".o_proj." in name:
        return "o"
    if ".mlp." in name:
        return "mlp"
    if t.dim() == 1:
        return "norm"
    raise ValueError(f"no gradient kind for {name}")


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def grad_errors(got: torch.Tensor, ref: torch.Tensor, kind: str, n_head: int) -> dict:
    """Errors of one gradient against its fp64 reference.

    fro : relative Frobenius error of the whole tensor (every kind)
    row  : worst relative error of an output row (matrices except tables)
    dxrow: worst relative error of a token row of dx, with its floor at 1e-3 x the median row norm, as the decode groups
           score hidden rows
    head : worst relative error of one head's block -- D rows of dWq / dWk / dWv, D columns of dWo
    elem : worst |error| of one element of a norm weight's gradient over that vector's norm"""
    y, r = got.double(), ref.double()
    out = {"fro": _rel(y, r)}
    if not torch.isfinite(y).all():
        out["fro"] = float("inf")
    if kind == "dx":
        out["dxrow"] = row_worst(y, r, floor_frac=1e-3)
    elif kind in ("qkv", "o", "mlp", "lora"):
        out["row"] = row_worst(y, r)
    if kind in ("qkv", "o"):
        blocks = zip(y.chunk(n_head, 0), r.chunk(n_head, 0)) if kind == "qkv" else zip(y.chunk(n_head, 1), r.chunk(n_head, 1))
        out["head"] = max(_rel(a, b) for a, b in blocks)
    if kind == "norm":
        out["elem"] = float((y - r).abs().max() / r.norm().clamp_min(1e-30))
    return out


def grad_report(got: dict, ref: dict, tag: str, n_head=None, floor: dict = None, show=True) -> dict:
    """Every gradient of `got` ({name: tensor}; "dx..." for input gradients) scored against `ref` (fp64) by
    grad_errors -> the worst value of each metric over the tensors, as "<metric>_<tag>", and with `floor` (the same
    gradients from the bf16 eager oracle) the worst ratio of a tensor's error to that tensor's floor error, as
    "floor_ratio_<metric>_<tag>".  n_head: {name: heads} or one count for every tensor.  Also "min:" counters
    n_tensors_<tag> and, where heads were scored, n_heads_<tag>.  show: print the worst tensor of every metric."""
    worst, where = {}, {}
    n_heads = 0
    for name, g in got.items():
        kind = grad_kind(name, g)
        nh = n_head.get(name) if isinstance(n_head, dict) else n_head
        e = grad_errors(g, ref[name], kind, nh)
        vals = dict(e)
        if floor is not None:
            f = grad_errors(floor[name], ref[name], kind, nh)
            vals.update({f"floor_ratio_{k}": v / max(f[k], 1e-30) for k, v in e.items()})
        n_heads += nh if kind in ("qkv", "o") else 0
        for k, v in vals.items():
            if k not in worst or not v <= worst[k]:
                worst[k], where[k] = v, name
    if show:
        for k in worst:
            print(f"  {tag}: worst {k} = {worst[k]:.3e} at {where[k]}")
    out = {f"{k}_{tag}": v for k, v in worst.items()}
    out[f"n_tensors_{tag}"] = float(len(got))
    if n_heads:
        out[f"n_heads_{tag}"] = float(n_heads)
    return out
