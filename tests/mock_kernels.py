"""TEST INFRASTRUCTURE: a CPU stand-in for the kernel layer (`midi_b200.ops` / the C-ABI calls the host code issues),
so that the HOST LOGIC of the engine -- the per-layer forward / backward schedule, which gradients are computed and where
they land in the flat buffers, the LoRA composition, the optimizer span, the autograd Functions -- runs in the CPU test
suite and is compared with the oracle's autograd.  It is installed by monkeypatching inside a test and nowhere else; the
product has no such switch (test_no_cpu_fallback).  It says nothing about the CUDA kernels themselves: those are compared
with the oracle on the GPU (tests/gpu_checks.py).  The stand-ins of the generate path's C-ABI entries are in
tests/mock_decode.py; `install` is the one entry point of the whole layer, for the trainer's tests and the generate tests
alike.

Semantics follow the kernels' contracts in include/midi_b200.h: bf16 storage, fp32 arithmetic, one rounding per stored
value; packed layouts, row pitches and in-place behaviour as the engine relies on them.
"""
import ctypes
import math

import torch
import torch.nn.functional as F

BF = torch.bfloat16


def _f(t):
    return t.to(torch.float32)


def _mat(t, rows, cols, ld):
    """[rows, cols] view with row pitch `ld` starting at t's first element (what the kernels get as pointer + ld)."""
    return torch.as_strided(t, (rows, cols), (ld, 1), t.storage_offset())


def _from_ptr(ptr, numel, dtype):
    nbytes = numel * torch.tensor([], dtype=dtype).element_size()
    buf = (ctypes.c_char * nbytes).from_address(ptr)
    return torch.frombuffer(buf, dtype=dtype, count=numel)


# ------------------------------------------------------------------ embeddings
def embed_sum(ids, table):
    return _f(table)[ids].sum(-2).to(BF)


def inner_input(hidden, ids, table):
    parts = []
    if hidden is not None:
        parts.append(hidden[:, None])
    if ids is not None and ids.shape[1] > 0:
        parts.append(table[ids])
    x = torch.cat(parts, 1)
    return x.reshape(-1, table.shape[1]).contiguous()


def inner_input_rows(hidden, y, rows, table):
    y_sel = y[rows.long()]
    return inner_input(hidden[rows.long()], y_sel[:, :-1], table), y_sel.clone()


def inner_input_rows_bwd_hidden(dx, inv, n_events, Tin):
    H = dx.shape[1]
    out = torch.zeros((inv.shape[0], H), dtype=BF)
    sel = inv >= 0
    out[sel] = dx.view(n_events, Tin, H)[:, 0][inv[sel].long()]
    return out


def batch_to_xy(batch):
    b = batch.to(torch.long)
    B, S1, T = b.shape
    return b[:, :-1].reshape(B * (S1 - 1), T).contiguous(), b[:, 1:].reshape(B * (S1 - 1), T).contiguous()


def batch_to_xy_packed(batch, src, pad_id):
    B, S1, T = batch.shape
    flat = batch.to(torch.long).reshape(B * S1, T)
    idx = src.long()
    x = torch.full((idx.numel(), T), pad_id, dtype=torch.long)
    y = x.clone()
    live = idx >= 0
    x[live], y[live] = flat[idx[live]], flat[idx[live] + 1]
    return x, y


def embed_bwd(ids, dout, dtable, per_row, row_stride, row_inner, row_off, pad_id, accumulate):
    j = torch.arange(ids.numel())
    rows = (j // per_row) * row_stride + row_off + (j % per_row) * row_inner
    acc = torch.zeros(dtable.shape, dtype=torch.float32)
    keep = ids != pad_id
    acc.index_add_(0, ids[keep], _f(dout)[rows[keep]])
    if accumulate:
        acc = acc.to(BF).float() + _f(dtable)
    dtable.copy_(acc.to(BF))


# ------------------------------------------------------------------ norm / rope / swiglu
def rmsnorm(x, w, eps, want_rstd=False):
    xf = _f(x)
    rstd = torch.rsqrt(xf.pow(2).mean(-1) + eps)
    y = (w.float() * (xf * rstd[:, None]).to(BF).float()).to(BF)
    return (y, rstd) if want_rstd else y


def add_rmsnorm(x, res, w, eps):
    h = (_f(x) + _f(res)).to(BF)
    y, rstd = rmsnorm(h, w, eps, want_rstd=True)
    return h, y, rstd


def rmsnorm_bwd(dy, x, w, rstd, dres, dw, accumulate_dw):
    xf, dyf = _f(x), _f(dy)
    nn = xf * rstd[:, None]
    dn = dyf * w.float()
    dot = (dn * nn).mean(-1, keepdim=True)
    dx = rstd[:, None] * (dn - nn * dot)
    if dres is not None:
        dx = dx + _f(dres)
    if dw is not None:
        g = (dyf * nn).sum(0)
        if accumulate_dw:
            g = g.to(BF).float() + _f(dw)
        dw.copy_(g.to(BF))
    return dx.to(BF)


def rope_table(inv_freq, n_pos, pos0=0):
    pos = torch.arange(pos0, pos0 + n_pos, dtype=torch.float32)
    fr = pos[:, None] * inv_freq.detach().float()[None, :]
    return fr.cos().to(BF), fr.sin().to(BF)


def _rot(x, cos, sin, backward):
    # x [..., D] fp32; cos/sin [..., D/2] fp32.  forward: x*cos + rotate_half(x)*sin; backward: its transpose
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    if not backward:
        return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), -1)
    return torch.cat((x1 * cos + x2 * sin, x2 * cos - x1 * sin), -1)


def rope_qk_(qkv, cos, sin, S, H, D, backward=False, pos0=0, pos0_dev=None, row_off=None):
    rows = qkv.shape[0]
    pos = pos0 + torch.arange(rows) % S
    if pos0_dev is not None:                                            # the device-side position base
        pos = pos + int(pos0_dev.reshape(-1)[0])
    if row_off is not None:                                             # ragged: row b's S rows at + row_off[b]
        pos = pos + row_off.long().repeat_interleave(S)
    c, s = cos.float()[pos][:, None], sin.float()[pos][:, None]          # [rows, 1, D/2]
    for col0 in (0, H):
        blk = _f(qkv[:, col0:col0 + H]).view(rows, H // D, D)
        qkv[:, col0:col0 + H] = _rot(blk, c, s, backward).reshape(rows, H).to(BF)


def rope_qk_ragged_(qkv, cos, sin, S, H, D, row_off, pos0=0, pos0_dev=None):
    rope_qk_(qkv, cos, sin, S, H, D, pos0=pos0, pos0_dev=pos0_dev, row_off=row_off)


def _segments(tiles):
    """[(row0, rows)] of the segments a {first, last} tile table describes."""
    firsts = sorted(set(tiles[:, 0].tolist()))
    return [(64 * f, 64 * (int(tiles[f, 1]) + 1 - f)) for f in firsts]


def rope_qk_seg_(qkv, cos, sin, tiles, H, D, backward=False):
    for r0, n in _segments(tiles):
        rope_qk_(qkv[r0:r0 + n], cos, sin, n, H, D, backward=backward)


def _silu(g):
    return g * torch.sigmoid(g)


def swiglu(gu):
    I = gu.shape[1] // 2
    return (_silu(_f(gu[:, :I])).to(BF).float() * _f(gu[:, I:])).to(BF)


def swiglu_bwd(gu, dact):
    I = gu.shape[1] // 2
    g, u, d = _f(gu[:, :I]), _f(gu[:, I:]), _f(dact)
    sg = torch.sigmoid(g)
    dg = d * u * (sg * (1 + g * (1 - sg)))
    du = d * (g * sg)
    return torch.cat((dg, du), 1).to(BF)


def scale(x, s):
    if s == 1.0:
        return x
    return (_f(x) * s).to(BF)


# ------------------------------------------------------------------ GEMM
def gemm(A, B, M, N, K, *, lda, ldb, a_mn=False, b_mn=False, out=None, ldc=None, residual=None, accumulate=False,
         allow_split=False):
    a = _mat(A, K, M, lda).t() if a_mn else _mat(A, M, K, lda)
    b = _mat(B, K, N, ldb).t() if b_mn else _mat(B, N, K, ldb)
    acc = _f(a) @ _f(b).t()
    if out is None:
        out = torch.empty((M, N), dtype=BF)
    if ldc is None:
        ldc = out.stride(0)
    N8 = (N + 7) // 8 * 8
    c = _mat(out, M, N8, ldc)
    if residual is not None:
        assert not accumulate
        r = _f(_mat(residual, M, N, residual.stride(0))).clone()
        c[:, :N] = (acc.to(BF).float() + r).to(BF)
    elif accumulate:
        assert ldc == N
        c[:, :N] = (acc.to(BF).float() + _f(c[:, :N])).to(BF)
    else:
        c[:, :N] = acc.to(BF)
        if N8 > N:
            c[:, N:] = 0
    return out


def linear_swiglu(x, w_gu):
    gu = gemm(x, w_gu, x.shape[0], w_gu.shape[0], x.shape[1], lda=x.stride(0), ldb=w_gu.stride(0))
    return gu, swiglu(gu)


def linear_rope(x, w_qkv, cos, sin, S, D):
    qkv = gemm(x, w_qkv, x.shape[0], w_qkv.shape[0], x.shape[1], lda=x.stride(0), ldb=w_qkv.stride(0))
    rope_qk_(qkv, cos, sin, S, w_qkv.shape[0] // 3, D)
    return qkv


def linear_rope_seg(x, w_qkv, cos, sin, tiles, D):
    qkv = gemm(x, w_qkv, x.shape[0], w_qkv.shape[0], x.shape[1], lda=x.stride(0), ldb=w_qkv.stride(0))
    rope_qk_seg_(qkv, cos, sin, tiles, w_qkv.shape[0] // 3, D)
    return qkv


# ------------------------------------------------------------------ attention
def _split(qkv, n_seq, S, nh, D):
    H = nh * D
    q, k, v = (_f(qkv[:, i * H:(i + 1) * H]).reshape(n_seq, S, nh, D).transpose(1, 2) for i in range(3))
    return q, k, v


def _attn(q, k, v):
    S, D = q.shape[-2], q.shape[-1]
    sc = q @ k.transpose(-1, -2) / math.sqrt(D)
    mask = torch.ones(S, S, dtype=torch.bool).tril()
    sc = sc.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(sc, -1)
    p = torch.softmax(sc, -1)
    return p.to(BF).float() @ v, lse


def attn_causal_fwd(qkv, B, S, n_heads, D, want_lse, impl=None):
    q, k, v = _split(qkv, B, S, n_heads, D)
    o, lse = _attn(q, k, v)
    out = o.transpose(1, 2).reshape(B * S, n_heads * D).to(BF)
    return out, (lse.contiguous() if want_lse else None)


def _attn_bwd(qkv, dout, n_seq, S, nh, D, cos_sin):
    H = nh * D
    with torch.enable_grad():                      # (called from inside autograd.Function.backward in the drop-in path)
        qkv32 = _f(qkv).detach().clone().requires_grad_(True)
        q, k, v = (qkv32[:, i * H:(i + 1) * H].reshape(n_seq, S, nh, D).transpose(1, 2) for i in range(3))
        sc = q @ k.transpose(-1, -2) / math.sqrt(D)
        sc = sc.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
        o = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(n_seq * S, H)
        o.backward(_f(dout).detach())
    dqkv = qkv32.grad.to(BF)
    if cos_sin is not None:
        rope_qk_(dqkv, cos_sin[0], cos_sin[1], S, H, D, backward=True)
    return dqkv


def attn_causal_bwd(qkv, out, dout, lse, B, S, n_heads, D, rope=None, impl=None):
    return _attn_bwd(qkv, dout, B, S, n_heads, D, rope)


def attn_causal_fwd_seg(qkv, tiles, order, n_heads, D, want_lse, impl=None):
    outs, lses = [], []
    for r0, n in _segments(tiles):
        o, lse = attn_causal_fwd(qkv[r0:r0 + n], 1, n, n_heads, D, True)
        outs.append(o)
        lses.append(lse[0])
    return torch.cat(outs), (torch.cat(lses, 1) if want_lse else None)


def attn_causal_bwd_seg(qkv, out, dout, lse, tiles, order, n_heads, D, rope=None, impl=None):
    return torch.cat([attn_causal_bwd(qkv[r0:r0 + n], out[r0:r0 + n], dout[r0:r0 + n], None, 1, n, n_heads, D, rope=rope)
                      for r0, n in _segments(tiles)])


def attn_tiny_fwd(qkv, n_events, L, n_heads, D, rope=None):
    if rope is not None:
        rope_qk_(qkv, rope[0], rope[1], L, n_heads * D, D)          # the kernel rotates q, k in place
    q, k, v = _split(qkv, n_events, L, n_heads, D)
    o, _ = _attn(q, k, v)
    return o.transpose(1, 2).reshape(n_events * L, n_heads * D).to(BF)


def attn_tiny_bwd(qkv, dout, n_events, L, n_heads, D, rope=None):
    return _attn_bwd(qkv, dout, n_events, L, n_heads, D, rope)


# ------------------------------------------------------------------ loss
def ce_fwd(logits, targets, V, ignore_index):
    lg = _f(logits[:, :V])
    lse = torch.logsumexp(lg, -1)
    keep = targets != ignore_index
    row = lse - lg.gather(1, targets.clamp(0, V - 1)[:, None])[:, 0]
    cnt = keep.sum().float()
    loss = (row * keep).sum() / cnt
    return torch.stack([loss, cnt]).float(), lse


def argmax_hits(logits, targets, V, ignore_index):
    am = logits[:, :V].float().argmax(-1)
    live = (targets != ignore_index) & (targets >= 0) & (targets < V)
    return torch.stack([(live & (am == targets)).sum(), live.sum()]).float()


def ce_bwd_(logits, targets, lse, lac, V, ignore_index, grad_scale=1.0, grad_scale_dev=None):
    lg = _f(logits[:, :V])
    p = torch.exp(lg - lse[:, None])
    p[torch.arange(p.shape[0]), targets.clamp(0, V - 1)] -= 1.0
    keep = (targets != ignore_index).float()[:, None]
    s = grad_scale / float(lac[1])
    if grad_scale_dev is not None:
        s = s * float(grad_scale_dev)
    logits[:, :V] = (p * keep * s).to(BF)
    if logits.shape[1] > V:
        logits[:, V:] = 0



# ------------------------------------------------------------------ raw C-ABI calls the host code issues itself
def _inner_input_bwd_hidden(dx_ptr, dh_ptr, n_events, Tin, H, _s):
    dx = _from_ptr(dx_ptr, n_events * Tin * H, BF).view(n_events, Tin, H)
    _from_ptr(dh_ptr, n_events * H, BF).view(n_events, H).copy_(dx[:, 0])


def _grad_clip_coef(gptr, n, max_norm, nc_ptr, _a, _b, _s):
    g = _from_ptr(gptr, n, BF).float()
    norm = float(g.pow(2).sum().sqrt())
    nc = _from_ptr(nc_ptr, 2, torch.float32)
    nc[0] = norm
    nc[1] = min(1.0, max_norm / (norm + 1e-6))


def _adamw_step(pptr, gptr, mptr, vptr, fptr, n, lr, b1, b2, eps, wd, step, nc_ptr, _s):
    p, g = _from_ptr(pptr, n, BF), _from_ptr(gptr, n, BF).float()
    m, v = _from_ptr(mptr, n, torch.float32), _from_ptr(vptr, n, torch.float32)
    flags = _from_ptr(fptr, (n + 255) // 256, torch.uint8)
    g = g * float(_from_ptr(nc_ptr, 2, torch.float32)[1])
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    decay = torch.where(flags.repeat_interleave(256)[:n] != 0, torch.ones(()), torch.tensor(1.0 - lr * wd))
    upd = (m / (1 - b1 ** step)) / ((v / (1 - b2 ** step)).sqrt() + eps)
    p.copy_((p.float() * decay - lr * upd).to(BF))


CALLS = {"b200_inner_input_bwd_hidden": _inner_input_bwd_hidden, "b200_grad_clip_coef": _grad_clip_coef,
         "b200_adamw_step": _adamw_step}


def _query(name, *args):
    if name == "b200_gradnorm_parts":
        return 1
    if name == "b200_attn_decode_workspace_bytes":
        return 256
    raise AssertionError(f"mock kernel layer: unexpected C-ABI query {name}")


class _NoStream:
    """torch.cuda.Stream stand-in for the CPU run of the device-resident loops (stream plumbing only)."""

    def __init__(self, *a, **k):
        self.cuda_stream = 0

    def wait_stream(self, other):
        pass


class _Event:
    """torch.cuda.Event stand-in: the mock kernels have finished when their call returns."""

    def __init__(self, *a, **k):
        pass

    def record(self, stream=None):
        pass

    def query(self):
        return True


# the `midi_b200.ops` wrappers the host code calls, each replaced by the stand-in of the same name above
OPS = ("embed_sum", "inner_input", "inner_input_rows", "inner_input_rows_bwd_hidden", "batch_to_xy", "batch_to_xy_packed",
       "embed_bwd", "rmsnorm", "add_rmsnorm", "rmsnorm_bwd", "rope_table", "rope_qk_", "rope_qk_seg_", "rope_qk_ragged_",
       "swiglu", "swiglu_bwd", "scale", "gemm", "linear_swiglu", "linear_rope", "linear_rope_seg", "attn_causal_fwd",
       "attn_causal_bwd", "attn_causal_fwd_seg", "attn_causal_bwd_seg", "attn_tiny_fwd", "attn_tiny_bwd", "ce_fwd",
       "argmax_hits", "ce_bwd_")


def install(monkeypatch, persist=False):
    """Route the host code's kernel calls to the CPU stand-ins above and those of tests/mock_decode.py for the duration
    of one test.  `persist`: let the generate loops take the persistent kernel's path (mock_decode.decode_events) for the
    tiny test model, whose shapes the kernel is not built for."""
    import contextlib

    import mock_decode
    from midi_b200 import decode, engine, lib, ops, serve
    g = globals()
    for name in OPS:
        monkeypatch.setattr(ops, name, g[name])
    monkeypatch.setattr(ops, "_ws", lambda key, nbytes, device, zero=False: torch.zeros(max(nbytes, 256), dtype=torch.uint8))
    monkeypatch.setattr(ops, "GEMM_PROFILE", None)
    calls = {**CALLS, **mock_decode.CALLS}

    def call(name, *args):
        if name not in calls:
            raise AssertionError(f"mock kernel layer: unexpected C-ABI call {name}")
        return calls[name](*args)

    monkeypatch.setattr(lib, "call", call)
    monkeypatch.setattr(lib, "query", _query)
    monkeypatch.setattr(lib, "load", lambda: mock_decode.LIB if persist else None)
    if persist:
        monkeypatch.setattr(decode.GraphGenerator, "persistent_ok", lambda self: True)
    monkeypatch.setattr(lib, "stream", lambda: None)
    monkeypatch.setattr(lib, "require_cuda", lambda t, what="tensor": None)
    def require_bf16(n, p, dev):                 # the dtype half of the product's check stays; only `is_cuda` is waived
        if p.dtype != BF:
            raise lib.B200Error(f"parameter {n} is {p.dtype}")

    monkeypatch.setattr(engine, "_require_device", require_bf16)
    monkeypatch.setattr(engine, "WGRAD_STREAM", False)
    monkeypatch.setattr(serve, "_pinned", lambda shape, dtype: torch.zeros(shape, dtype=dtype))
    monkeypatch.setattr(torch.cuda, "Stream", _NoStream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _NoStream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    for record in (mock_decode.DRAWS, mock_decode.LAUNCHES, mock_decode.ON_EVENT, mock_decode._KEYS):
        record.clear()


def trace(monkeypatch, fn, names=None):
    """fn() with every wrapper of OPS and every raw C-ABI call recorded by name, in call order, into `names` (a new list
    by default), which is returned.  Use inside a `monkeypatch.context()`: the recording stays patched in until it ends."""
    from midi_b200 import lib, ops
    names = [] if names is None else names
    for name in OPS:
        f = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _f=f, _n=name, **k: (names.append(_n), _f(*a, **k))[1])
    call = lib.call
    monkeypatch.setattr(lib, "call", lambda n, *a: (names.append(n), call(n, *a))[1])
    fn()
    return names
