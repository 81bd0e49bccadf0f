"""TEST INFRASTRUCTURE: a CPU stand-in for the kernel layer (`midi_b200.ops` / the C-ABI calls the host code issues),
so that the HOST LOGIC of the engine -- the per-layer forward / backward schedule, which gradients are computed and where
they land in the flat buffers, the LoRA composition, the optimizer span, the autograd Functions -- runs in the CPU test
suite and is compared with the oracle's autograd.  It is installed by monkeypatching inside a test and nowhere else; the
product has no such switch (test_no_cpu_fallback).  It says nothing about the CUDA kernels themselves: those are compared
with the oracle on the GPU (tests/gpu_checks.py).

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


def rope_qk_(qkv, cos, sin, S, H, D, backward=False, pos0=0, pos0_dev=None):
    rows = qkv.shape[0]
    pos = pos0 + torch.arange(rows) % S
    c, s = cos.float()[pos][:, None], sin.float()[pos][:, None]          # [rows, 1, D/2]
    for col0 in (0, H):
        blk = _f(qkv[:, col0:col0 + H]).view(rows, H // D, D)
        qkv[:, col0:col0 + H] = _rot(blk, c, s, backward).reshape(rows, H).to(BF)


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



# ------------------------------------------------------------------ decode-step entry points (pointer level)
def _bfmat(ptr, rows, cols, ld):
    t = _from_ptr(ptr, (rows - 1) * ld + cols, BF)
    return torch.as_strided(t, (rows, cols), (ld, 1))


def _pool(ptr, batch, max_pages, nh, page, D):
    return _from_ptr(ptr, batch * max_pages * nh * page * D, BF).view(batch * max_pages, nh, page, D)


def _gemv_bf16(x, W, res, y, B, N, K, ldx, ldw, ldr, ldy, _s):
    acc = _f(_bfmat(x, B, K, ldx)) @ _f(_bfmat(W, N, K, ldw)).t()
    if res:
        acc = acc.to(BF).float() + _f(_bfmat(res, B, N, ldr))
    out = _bfmat(y, B, ldy if ldy >= N else N, ldy)
    out[:, :N] = acc.to(BF)
    out[:, N:] = 0


def _gemv_fused(x, ids, ids_stride, table, V, norm_w, eps, W, res, y, B, N_out, K, ldx, ldw, ldr, ldy, swiglu_, _s):
    assert not ids, "mock kernel layer: the ids/table input of b200_gemv_fused is used by the graph loop only"
    h = _bfmat(x, B, K, ldx).clone()
    if norm_w:
        h = rmsnorm(h, _from_ptr(norm_w, K, BF), eps)
    rows_w = 2 * N_out if swiglu_ else N_out
    z = (_f(h) @ _f(_bfmat(W, rows_w, K, ldw)).t())
    if swiglu_:
        z = _f(swiglu(z.to(BF)))
    if res:
        z = z.to(BF).float() + _f(_bfmat(res, B, N_out, ldr))
    _bfmat(y, B, N_out, ldy).copy_(z.to(BF))


def _dev_int(ptr):
    return int(_from_ptr(ptr, 1, torch.int32)[0]) if ptr else 0


def _kv_append(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, s_new, pos0, pos0_dev, ld, _s):
    pos0 = pos0 + _dev_int(pos0_dev)
    H = nh * D
    q = _bfmat(qkv, batch * s_new, 3 * H, ld)
    kp, vp = _pool(k_pool, batch, max_pages, nh, page, D), _pool(v_pool, batch, max_pages, nh, page, D)
    table = _from_ptr(bt, batch * max_pages, torch.int32).view(batch, max_pages)
    for b in range(batch):
        for i in range(s_new):
            pos = pos0 + i
            pg = int(table[b, pos // page])
            row = q[b * s_new + i]
            kp[pg, :, pos % page] = row[H:2 * H].view(nh, D)
            vp[pg, :, pos % page] = row[2 * H:].view(nh, D)


def _gather_kv(pool, table, b, n_pos, page):
    pages = [pool[int(table[b, j])] for j in range((n_pos + page - 1) // page)]          # each [nh, page, D]
    return torch.cat(pages, 1)[:, :n_pos]                                               # [nh, n_pos, D]


def _attend(q, k, v, scale):
    # q [nh, D], k/v [nh, T, D] (fp32) -> [nh, D], probabilities rounded to bf16 before P.V like the kernels
    p = torch.softmax((k @ q[:, :, None])[:, :, 0] * scale, -1)
    return (p.to(BF).float()[:, None, :] @ v)[:, 0]


def _attn_decode(q, k_pool, v_pool, bt, max_pages, page, out, batch, s_q, nh, D, past, past_dev, max_T, ldq, ldo, scale,
                 n_split, _ws, _wsb, _s):
    past = past + _dev_int(past_dev)
    H = nh * D
    qm, om = _bfmat(q, batch * s_q, H, ldq), _bfmat(out, batch * s_q, H, ldo)
    kp, vp = _pool(k_pool, batch, max_pages, nh, page, D), _pool(v_pool, batch, max_pages, nh, page, D)
    table = _from_ptr(bt, batch * max_pages, torch.int32).view(batch, max_pages)
    for b in range(batch):
        for i in range(s_q):
            n_pos = past + i + 1
            k, v = _f(_gather_kv(kp, table, b, n_pos, page)), _f(_gather_kv(vp, table, b, n_pos, page))
            om[b * s_q + i] = _attend(_f(qm[b * s_q + i]).view(nh, D), k, v, scale).reshape(H).to(BF)


def _attn_decode_fused(qkv, k_pool, v_pool, bt, max_pages, page, cos_t, sin_t, out, batch, nh, D, pos0, pos_dev, max_T, ldq,
                       ldo, scale, n_split, _ws, _wsb, _s):
    pos0 = pos0 + _dev_int(pos_dev)
    H, half = nh * D, D // 2
    q = _bfmat(qkv, batch, 3 * H, ldq)
    c = _from_ptr(cos_t + pos0 * half * 2, half, BF).float()[None, None]
    s_ = _from_ptr(sin_t + pos0 * half * 2, half, BF).float()[None, None]
    for col0 in (0, H):
        q[:, col0:col0 + H] = _rot(_f(q[:, col0:col0 + H]).view(batch, nh, D), c, s_, False).reshape(batch, H).to(BF)
    _kv_append(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, 1, pos0, None, ldq, None)
    _attn_decode(qkv, k_pool, v_pool, bt, max_pages, page, out, batch, 1, nh, D, pos0, None, max_T, ldq, ldo, scale, n_split,
                 None, 0, None)


def _sample_from_logits(logits, rows, V, ld, temp, top_p, top_k, step, event_tok, lut, n_event_types, eos_id, pad_id,
                        dense_mask, uniforms, out, out_stride, _s):
    assert top_k == 1, "mock kernel layer: greedy sampling only"
    lg = _f(_bfmat(logits, rows, V, ld)).clone()
    if dense_mask:                                    # app.py:73-87 options: [rows, V] uint8, ANDed with the grammar range
        lg[_from_ptr(dense_mask, rows * V, torch.uint8).view(rows, V) == 0] = float("-inf")
    table = _from_ptr(lut, n_event_types * 8 * 2, torch.int32).view(n_event_types, 8, 2)
    ev = _from_ptr(event_tok, rows, torch.int64)
    o = _from_ptr(out, (rows - 1) * out_stride + 1, torch.int64)
    for r in range(rows):
        if step == 0:
            lo, hi = eos_id, eos_id + 1 + n_event_types
        else:
            e = int(ev[r]) - (eos_id + 1)
            if int(ev[r]) == eos_id or e < 0 or e >= n_event_types:
                lo, hi = pad_id, pad_id + 1
            else:
                lo, hi = int(table[e, step - 1, 0]), int(table[e, step - 1, 1])
                if hi <= lo:
                    lo, hi = pad_id, pad_id + 1
        o[r * out_stride] = lo + int(torch.argmax(lg[r, lo:hi]))


def _uniform_fill(u, n, seed, state, _s):
    _from_ptr(state, 2, torch.int64)[0] += 1          # greedy mock: the draws themselves are never used


def _event_commit(ev_t, seq, ev_next, pos_dev, B, T, max_len, _s):
    pos = _from_ptr(pos_dev, 1, torch.int32)
    p = int(pos[0])
    ev = _from_ptr(ev_t, T * B, torch.int64).view(T, B).t()                # [B, T]
    if p + 1 < max_len:
        _from_ptr(seq, B * max_len * T, torch.int64).view(B, max_len, T)[:, p + 1] = ev
    _from_ptr(ev_next, B * T, torch.int64).view(B, T).copy_(ev)
    pos[0] = p + 1


class _NoStream:
    """torch.cuda.Stream stand-in for the CPU run of the device-resident loops (stream plumbing only)."""

    def __init__(self, *a, **k):
        self.cuda_stream = 0

    def wait_stream(self, other):
        pass


_DECODE_CALLS = {"b200_uniform_fill": _uniform_fill, "b200_event_commit": _event_commit, "b200_gemv_bf16": _gemv_bf16, "b200_gemv_fused": _gemv_fused, "b200_kv_append": _kv_append,
                 "b200_attn_decode": _attn_decode, "b200_attn_decode_fused": _attn_decode_fused,
                 "b200_sample_from_logits": _sample_from_logits}


# ------------------------------------------------------------------ raw C-ABI calls the host code issues itself
def _call(name, *args):
    if name in _DECODE_CALLS:
        return _DECODE_CALLS[name](*args)
    if name == "b200_inner_input_bwd_hidden":
        dx_ptr, dh_ptr, n_events, Tin, H, _ = args
        dx = _from_ptr(dx_ptr, n_events * Tin * H, BF).view(n_events, Tin, H)
        _from_ptr(dh_ptr, n_events * H, BF).view(n_events, H).copy_(dx[:, 0])
        return
    if name == "b200_grad_clip_coef":
        gptr, n, max_norm, nc_ptr, _, _, _ = args
        g = _from_ptr(gptr, n, BF).float()
        norm = float(g.pow(2).sum().sqrt())
        nc = _from_ptr(nc_ptr, 2, torch.float32)
        nc[0] = norm
        nc[1] = min(1.0, max_norm / (norm + 1e-6))
        return
    if name == "b200_adamw_step":
        pptr, gptr, mptr, vptr, fptr, n, lr, b1, b2, eps, wd, step, nc_ptr, _ = args
        p, g = _from_ptr(pptr, n, BF), _from_ptr(gptr, n, BF).float()
        m, v = _from_ptr(mptr, n, torch.float32), _from_ptr(vptr, n, torch.float32)
        flags = _from_ptr(fptr, (n + 255) // 256, torch.uint8)
        g = g * float(_from_ptr(nc_ptr, 2, torch.float32)[1])
        m.mul_(b1).add_(g, alpha=1 - b1)
        v.mul_(b2).addcmul_(g, g, value=1 - b2)
        decay = torch.where(flags.repeat_interleave(256)[:n] != 0, torch.ones(()), torch.tensor(1.0 - lr * wd))
        upd = (m / (1 - b1 ** step)) / ((v / (1 - b2 ** step)).sqrt() + eps)
        p.copy_((p.float() * decay - lr * upd).to(BF))
        return
    raise AssertionError(f"mock kernel layer: unexpected C-ABI call {name}")


def _query(name, *args):
    if name == "b200_gradnorm_parts":
        return 1
    if name == "b200_attn_decode_workspace_bytes":
        return 256
    raise AssertionError(f"mock kernel layer: unexpected C-ABI query {name}")


# the `midi_b200.ops` wrappers the host code calls, each replaced by the stand-in of the same name above
OPS = ("embed_sum", "inner_input", "inner_input_rows", "inner_input_rows_bwd_hidden", "batch_to_xy", "batch_to_xy_packed",
       "embed_bwd", "rmsnorm", "add_rmsnorm", "rmsnorm_bwd", "rope_table", "rope_qk_", "rope_qk_seg_", "swiglu", "swiglu_bwd",
       "scale", "gemm", "linear_swiglu", "linear_rope", "linear_rope_seg", "attn_causal_fwd", "attn_causal_bwd",
       "attn_causal_fwd_seg", "attn_causal_bwd_seg", "attn_tiny_fwd", "attn_tiny_bwd", "ce_fwd", "argmax_hits", "ce_bwd_")


def install(monkeypatch):
    """Route the host code's kernel calls to the CPU stand-ins above for the duration of one test."""
    from midi_b200 import engine, lib, ops
    g = globals()
    for name in OPS:
        monkeypatch.setattr(ops, name, g[name])
    monkeypatch.setattr(ops, "_ws", lambda key, nbytes, device, zero=False: torch.zeros(max(nbytes, 256), dtype=torch.uint8))
    monkeypatch.setattr(ops, "GEMM_PROFILE", None)
    monkeypatch.setattr(lib, "load", lambda: None)
    monkeypatch.setattr(lib, "call", _call)
    monkeypatch.setattr(lib, "query", _query)
    monkeypatch.setattr(lib, "stream", lambda: None)
    monkeypatch.setattr(lib, "require_cuda", lambda t, what="tensor": None)
    def require_bf16(n, p, dev):                 # the dtype half of the product's check stays; only `is_cuda` is waived
        if p.dtype != BF:
            raise lib.B200Error(f"parameter {n} is {p.dtype}")

    monkeypatch.setattr(engine, "_require_device", require_bf16)
    monkeypatch.setattr(engine, "WGRAD_STREAM", False)
    import contextlib
    monkeypatch.setattr(torch.cuda, "Stream", _NoStream)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _NoStream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())


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
