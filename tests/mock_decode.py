"""TEST INFRASTRUCTURE: CPU stand-ins for the generate path's C-ABI entries (include/midi_b200.h), installed with the rest of
the mock kernel layer by tests/mock_kernels.py.  One stand-in per kernel, each compile-time flag an argument (None: off):
`row_off` (ragged rows at the shared position + row_off[b]), `row_end` / `row_last` (the request queue's per-row stop),
`rows` (per-request settings and seeds) and `stream` (the serving queue's host buffers).  CALLS maps each C-ABI name to one.

Grammar ranges, the step count of an event and the counter-based uniforms are tests/decode_reference.py's.  The sampler
takes softmax(logits / temp) in the grammar range and mask, top-k then top-p on the sorted probabilities, and the uniform
pick from the renormalised mass; top_k = 1 is the argmax of the allowed logits, lowest id on ties.  Each draw is appended
to DRAWS (row, u, temp, top_p, top_k, denied ids, step, and -- where the caller keys it -- seed and event j).

The persistent stand-in runs whole events in the order the host-issued loop issues them, with the same entries, so a
request gives the same events on both loops; a row that is not live appends, attends, draws and commits nothing.  With
`stream`, after each event it writes the live rows' events to `out_events`, then `committed[b]`, calls every hook in
ON_EVENT with the number of events run so far, and ends the launch if `ctl` is nonzero.  LAUNCHES records (n_events,
exit_on_done, events run, ended by ctl) per streaming launch.
"""
import math
from types import SimpleNamespace

import numpy as np
import torch

from decode_reference import PD_T, counter_uniform, event_n_steps, grammar_range
from mock_kernels import BF, _f, _from_ptr, _rot, rmsnorm, swiglu

DRAWS = []
ON_EVENT = []
LAUNCHES = []
_KEYS = {}                  # u pointer -> [(seed, j)] of the last b200_uniform_fill_rows into it

# what the persistent loop asks of the loaded library besides calls: its workspace size
LIB = SimpleNamespace(b200_decode_events_workspace_bytes=lambda _desc: 256)


def _bfmat(ptr, rows, cols, ld):
    t = _from_ptr(ptr, (rows - 1) * ld + cols, BF)
    return torch.as_strided(t, (rows, cols), (ld, 1))


def _vals(ptr, n, dtype=torch.int32):
    """n values of a device array as a list."""
    return _from_ptr(ptr, n, dtype).tolist()


def _dev_int(ptr):
    return int(_from_ptr(ptr, 1, torch.int32)[0]) if ptr else 0


def _rows(batch, row_off, live):
    """(b, row_off[b]) of the rows an entry runs: every row, or only the live ones; offset 0 without row_off."""
    offs = _vals(row_off, batch) if row_off else [0] * batch
    return [(b, offs[b]) for b in range(batch) if live is None or live[b]]


def _table(bt, batch, max_pages):
    return _from_ptr(bt, batch * max_pages, torch.int32).view(batch, max_pages)


def _pool(ptr, table, nh, page, D):
    """A KV pool as [n_pages, nh, page, D]: every page the block table names (a batch-1 table may name any page of the
    pool), and at least batch * max_pages."""
    n = max(int(table.max()) + 1, table.numel())
    return _from_ptr(ptr, n * nh * page * D, BF).view(n, nh, page, D)


# ------------------------------------------------------------------ projections
def gemv_bf16(x, W, res, y, B, N, K, ldx, ldw, ldr, ldy):
    acc = _f(_bfmat(x, B, K, ldx)) @ _f(_bfmat(W, N, K, ldw)).t()
    if res:
        acc = acc.to(BF).float() + _f(_bfmat(res, B, N, ldr))
    out = _bfmat(y, B, ldy if ldy >= N else N, ldy)
    out[:, :N] = acc.to(BF)
    out[:, N:] = 0


def gemv_fused(x, ids, ids_stride, table, V, norm_w, eps, W, res, y, B, N_out, K, ldx, ldw, ldr, ldy, swiglu_):
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


# ------------------------------------------------------------------ paged KV: append and attention
def kv_append(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, s_new, pos0, pos0_dev, ld, row_off=None, live=None):
    pos0 = pos0 + _dev_int(pos0_dev)
    H = nh * D
    q = _bfmat(qkv, batch * s_new, 3 * H, ld)
    table = _table(bt, batch, max_pages)
    kp, vp = _pool(k_pool, table, nh, page, D), _pool(v_pool, table, nh, page, D)
    for b, off in _rows(batch, row_off, live):
        for i in range(s_new):
            pos, row = pos0 + off + i, q[b * s_new + i]
            pg = int(table[b, pos // page])
            kp[pg, :, pos % page] = row[H:2 * H].view(nh, D)
            vp[pg, :, pos % page] = row[2 * H:].view(nh, D)


def _gather_kv(pool, table, b, n_pos, page):
    pages = [pool[int(table[b, j])] for j in range((n_pos + page - 1) // page)]          # each [nh, page, D]
    return torch.cat(pages, 1)[:, :n_pos]                                               # [nh, n_pos, D]


def _attend(q, k, v, scale):
    # q [nh, D], k/v [nh, T, D] (fp32) -> [nh, D], probabilities rounded to bf16 before P.V like the kernels
    p = torch.softmax((k @ q[:, :, None])[:, :, 0] * scale, -1)
    return (p.to(BF).float()[:, None, :] @ v)[:, 0]


def attn_decode(q, k_pool, v_pool, bt, max_pages, page, out, batch, s_q, nh, D, past, past_dev, max_T, ldq, ldo, scale,
                n_split, _ws, _wsb, row_off=None, live=None):
    past = past + _dev_int(past_dev)
    H = nh * D
    qm, om = _bfmat(q, batch * s_q, H, ldq), _bfmat(out, batch * s_q, H, ldo)
    table = _table(bt, batch, max_pages)
    kp, vp = _pool(k_pool, table, nh, page, D), _pool(v_pool, table, nh, page, D)
    for b, off in _rows(batch, row_off, live):
        for i in range(s_q):
            n_pos = past + off + i + 1
            k, v = _f(_gather_kv(kp, table, b, n_pos, page)), _f(_gather_kv(vp, table, b, n_pos, page))
            om[b * s_q + i] = _attend(_f(qm[b * s_q + i]).view(nh, D), k, v, scale).reshape(H).to(BF)


def attn_decode_fused(qkv, k_pool, v_pool, bt, max_pages, page, cos_t, sin_t, out, batch, nh, D, pos0, pos_dev, max_T,
                      ldq, ldo, scale, n_split, _ws, _wsb, row_off=None, live=None):
    """RoPE of each row's q and k at its position, then kv_append and attn_decode."""
    pos0 = pos0 + _dev_int(pos_dev)
    H, half = nh * D, D // 2
    q = _bfmat(qkv, batch, 3 * H, ldq)
    for b, off in _rows(batch, row_off, live):
        c, s = (_from_ptr(t + (pos0 + off) * half * 2, half, BF).float()[None] for t in (cos_t, sin_t))
        for col0 in (0, H):
            q[b, col0:col0 + H] = _rot(_f(q[b, col0:col0 + H]).view(nh, D), c, s, False).reshape(H).to(BF)
    kv_append(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, 1, pos0, 0, ldq, row_off, live)
    attn_decode(qkv, k_pool, v_pool, bt, max_pages, page, out, batch, 1, nh, D, pos0, 0, max_T, ldq, ldo, scale, n_split,
                0, 0, row_off, live)


# ------------------------------------------------------------------ sampler and uniforms
def _draw(lg, lo, hi, allowed, temp, top_p, top_k, u):
    """One row: lg float [V] logits, allowed bool [V]."""
    if top_k == 1:
        return lo + int(torch.argmax(lg[lo:hi].masked_fill(~allowed[lo:hi], float("-inf"))))
    p = torch.softmax(lg.double() / temp, 0)
    p[~allowed] = 0
    cand = torch.nonzero(p > 0).flatten()
    ids = cand[torch.sort(-p[cand], stable=True).indices[:top_k]].tolist()      # by p descending, ties to the lowest id
    if not ids:
        return lo
    keep, cum = [], 0.0
    for i, pi in zip(ids, p[ids].tolist()):
        if cum > top_p:
            break
        keep.append((i, pi))
        cum += pi
    total = sum(pi for _, pi in keep)
    run = 0.0
    for i, pi in keep:
        run += pi
        if run > u * total:
            return i
    return keep[-1][0]


def _sample(lg, rows, step, ev0, lut, n_event_types, eos_id, pad_id, mask, temps, top_ps, top_ks, us, keys=None):
    """The ids rows `rows` of lg (fp32 [B, V]) draw at token step `step`: {row: id}, each draw appended to DRAWS."""
    got = {}
    for r in rows:
        lo, hi = grammar_range(step, ev0[r], lut, eos_id, pad_id, n_event_types)
        allowed = torch.zeros(lg.shape[1], dtype=torch.bool)
        allowed[lo:hi] = True
        if mask is not None:
            allowed &= mask[r] != 0
        temp, top_p, top_k, u = float(temps[r]), float(top_ps[r]), max(1, int(top_ks[r])), float(us[r])
        got[r] = _draw(lg[r], lo, hi, allowed, temp, top_p, top_k, u)
        rec = dict(row=r, u=u, temp=temp, top_p=top_p, top_k=top_k, step=step,
                   deny=torch.nonzero(mask[r] == 0).flatten().tolist() if mask is not None else [])
        if keys is not None:
            rec["seed"], rec["j"] = keys[r]
        DRAWS.append(rec)
    return got


def sample_from_logits(logits, rows, V, ld, temp, top_p, top_k, step, event_tok, lut, n_event_types, eos_id, pad_id,
                       dense_mask, uniforms, out, out_stride, keys=None):
    """temp / top_p / top_k: one value per row, or one value for every row."""
    per_row = [x if isinstance(x, list) else [x] * rows for x in (temp, top_p, top_k)]
    mask = _from_ptr(dense_mask, rows * V, torch.uint8).view(rows, V) if dense_mask else None
    table = _from_ptr(lut, n_event_types * 8 * 2, torch.int32).view(n_event_types, 8, 2).numpy()
    o = _from_ptr(out, (rows - 1) * out_stride + 1, torch.int64)
    got = _sample(_f(_bfmat(logits, rows, V, ld)), range(rows), step, _vals(event_tok, rows, torch.int64), table,
                  n_event_types, eos_id, pad_id, mask, *per_row, _vals(uniforms, rows, torch.float32), keys)
    for r, t in got.items():
        o[r * out_stride] = t


def _sample_from_logits_rows(logits, rows, V, ld, row_temp, row_top_p, row_top_k, *rest):
    """b200_sample_from_logits_rows: each row's settings from the device arrays, its draws keyed as the uniforms were."""
    sample_from_logits(logits, rows, V, ld, _vals(row_temp, rows, torch.float32), _vals(row_top_p, rows, torch.float32),
                       _vals(row_top_k, rows), *rest, keys=_KEYS.get(rest[-3]))


def uniform_fill(u, n, seed, state):
    st = _from_ptr(state, 2, torch.int64)
    _from_ptr(u, n, torch.float32).copy_(torch.from_numpy(counter_uniform(seed ^ int(st[1]), int(st[0]), np.arange(n))))
    st[0] += 1


def _row_keys(B, pos, row_off, row_first, row_seed):
    """(seed, j) of every row: its request's seed and the new event j = pos + row_off[b] - row_first[b] it draws for."""
    p = _dev_int(pos)
    offs, first, seeds = _vals(row_off, B), _vals(row_first, B), _vals(row_seed, B, torch.int64)
    return [(seeds[b], p + offs[b] - first[b]) for b in range(B)]


def _row_uniforms(keys, step):
    """u of every row at token step `step` (or [n_steps, B] for a column of steps): the draw of its request alone."""
    seeds, js = zip(*keys)
    return counter_uniform(list(seeds), PD_T * np.array(js) + step, 0)


def uniform_fill_rows(u, B, pos_dev, row_off, row_first, row_seed, step):
    keys = _row_keys(B, pos_dev, row_off, row_first, row_seed)
    _from_ptr(u, B, torch.float32).copy_(torch.from_numpy(_row_uniforms(keys, step)))
    _KEYS[u] = keys


# ------------------------------------------------------------------ commit
def event_commit(ev_t, seq, ev_next, pos_dev, B, T, max_len, row_off=None, row_end=None, row_last=None, eos_id=None):
    """Row b's event ev_t[:, b] to seq[b, pos + row_off[b] + 1] (below max_len) and ev_next[b]; pos + 1.  With row_last
    only the rows whose row_last is -1 commit, and such a row's row_last becomes its seq index at EOS or at row_end."""
    pos = _from_ptr(pos_dev, 1, torch.int32)
    p = int(pos[0])
    ev = _from_ptr(ev_t, T * B, torch.int64).view(T, B).t()                # [B, T]
    out = _from_ptr(seq, B * max_len * T, torch.int64).view(B, max_len, T)
    nxt = _from_ptr(ev_next, B * T, torch.int64).view(B, T)
    last = _from_ptr(row_last, B, torch.int32) if row_last else None
    ends = _vals(row_end, B) if row_end else None
    for b, off in _rows(B, row_off, None):
        if last is not None and int(last[b]) != -1:
            continue
        q = p + off + 1
        if q < max_len:
            out[b, q] = ev[b]
        nxt[b] = ev[b]
        if last is not None and (int(ev[b, 0]) == eos_id or q >= ends[b]):
            last[b] = q
    pos[0] = p + 1


# ------------------------------------------------------------------ persistent kernel
def _proj(x, w, n_out, K, norm=0, eps=0.0, res=None, swiglu=False, ldy=None):
    """gemv_fused on tensors: y = [swiglu]([rmsnorm](x) @ W.T) [+ res]."""
    y = torch.empty((x.shape[0], ldy or n_out), dtype=BF)
    gemv_fused(x.data_ptr(), 0, 0, 0, 0, norm, eps, w, res.data_ptr() if res is not None else 0, y.data_ptr(),
               x.shape[0], n_out, K, x.stride(0), K, res.stride(0) if res is not None else 0, y.stride(0), int(swiglu))
    return y


def _layers(tab, n):
    return _from_ptr(tab, n * 6, torch.int64).view(n, 6).tolist()     # qkv, o, gu, down, ln1, ln2


def _event(d, live, row_off, p, settings, keys, us):
    """One event of the live rows from ev_in: the sampled tokens, int64 [T, B] (pad for rows that are not live and for
    the steps the event does not run).  settings: per-row (temps, top_ps, top_ks); us: u [T, B] of every step."""
    B, H, V = d.batch, d.H, d.V
    live_rows = [b for b in range(B) if live[b]]
    ev_in = _from_ptr(d.ev_in, B * PD_T, torch.int64).view(B, PD_T)
    emb_o = _from_ptr(d.emb_outer, V * H, BF).view(V, H)
    ok = (ev_in >= 0) & (ev_in < V)                                     # the kernel embeds an out-of-range id as zero
    x = (_f(emb_o)[ev_in.clamp(0, V - 1)] * ok[..., None]).sum(-2).to(BF)
    kv = _from_ptr(d.kv_outer, d.n_outer * 2, torch.int64).view(d.n_outer, 2).tolist()
    D = H // d.nh_outer
    for (wq, wo, wgu, wd, ln1, ln2), (k_pool, v_pool) in zip(_layers(d.outer_w, d.n_outer), kv):
        qkv = _proj(x, wq, 3 * H, H, norm=ln1, eps=d.eps)
        attn = torch.zeros((B, H), dtype=BF)
        attn_decode_fused(qkv.data_ptr(), k_pool, v_pool, d.block_table, d.max_pages, d.page, d.cos_outer, d.sin_outer,
                          attn.data_ptr(), B, d.nh_outer, D, p, 0, d.max_len, 3 * H, H, 1.0 / math.sqrt(D), 1, 0, 0,
                          row_off, live)
        h = _proj(attn, wo, H, H, res=x)
        act = _proj(h, wgu, d.I_outer, H, norm=ln2, eps=d.eps, swiglu=True)
        x = _proj(act, wd, H, d.I_outer, res=h)
    hidden = rmsnorm(x, _from_ptr(d.outer_norm, H, BF), d.eps)
    nh2 = d.nh_inner
    D2 = H // nh2
    inner = _layers(d.inner_w, d.n_inner)
    pools = [(torch.zeros((B, nh2, PD_T, D2), dtype=BF), torch.zeros((B, nh2, PD_T, D2), dtype=BF)) for _ in inner]
    bt = torch.arange(B, dtype=torch.int32).view(B, 1)
    emb_i = _from_ptr(d.emb_inner, V * H, BF).view(V, H)
    ev_t = torch.full((PD_T, B), d.pad_id, dtype=torch.int64)
    lut = _from_ptr(d.lut, d.n_event_types * 8 * 2, torch.int32).view(d.n_event_types, 8, 2).numpy()
    mask = _from_ptr(d.dense_mask, B * V, torch.uint8).view(B, V)
    n_steps = PD_T
    for i in range(PD_T):
        if i >= n_steps:
            break
        x2 = hidden if i == 0 else emb_i[ev_t[i - 1]].contiguous()
        for (wq, wo, wgu, wd, ln1, ln2), (kp, vp) in zip(inner, pools):
            qkv = _proj(x2, wq, 3 * H, H, norm=ln1, eps=d.eps)
            attn = torch.zeros((B, H), dtype=BF)
            attn_decode_fused(qkv.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), 1, PD_T, d.cos_inner,
                              d.sin_inner, attn.data_ptr(), B, nh2, D2, i, 0, PD_T, 3 * H, H, 1.0 / math.sqrt(D2), 1, 0, 0,
                              None, live)
            h = _proj(attn, wo, H, H, res=x2)
            act = _proj(h, wgu, d.I_inner, H, norm=ln2, eps=d.eps, swiglu=True)
            x2 = _proj(act, wd, H, d.I_inner, res=h)
        logits = _proj(x2, d.lm_head, V, H, norm=d.inner_norm, eps=d.eps, ldy=d.pitch)
        got = _sample(_f(logits[:, :V]), live_rows, i, ev_t[0].tolist(), lut, d.n_event_types, d.eos_id, d.pad_id, mask,
                      *settings, us[i], keys)
        for b, t in got.items():
            ev_t[i, b] = t
        if i == 0:
            n_steps = event_n_steps(ev_t[0].tolist(), live, lut, d.eos_id, d.n_event_types)
    return ev_t


def decode_events(desc, row_off, row_end, row_last, exit_on_done, n_events, rows=None, stream=None):
    """decode_events_kernel of the request queue: up to n_events events of the rows whose row_last is -1, ending early
    when no row is live, at max_len, or -- with exit_on_done -- after the event in which a row finished.  rows: the
    per-request (row_temp, row_top_p, row_top_k, row_seed, row_first); stream: (out_events, committed, ctl)."""
    d = desc._obj
    B = d.batch
    pos = _from_ptr(d.pos, 1, torch.int32)
    rng = _from_ptr(d.rng_state, 2, torch.int64)
    last = _from_ptr(row_last, B, torch.int32)
    if stream is not None:
        out = _from_ptr(stream[0], B * d.max_len * PD_T, torch.int64).view(B, d.max_len, PD_T)
        seq = _from_ptr(d.seq, B * d.max_len * PD_T, torch.int64).view(B, d.max_len, PD_T)
        done, ctl = _from_ptr(stream[1], B, torch.int32), _from_ptr(stream[2], 1, torch.int32)
    if rows is not None:
        row_temp, row_top_p, row_top_k, row_seed, row_first = rows
        settings = _vals(row_temp, B, torch.float32), _vals(row_top_p, B, torch.float32), _vals(row_top_k, B)
    else:
        settings = [d.temp] * B, [d.top_p] * B, [d.top_k] * B
    steps = np.arange(PD_T)[:, None]
    ran, by_ctl = 0, False
    for _ in range(n_events):
        p = int(pos[0])
        live = [int(v) == -1 for v in last]
        if not any(live) or p + 1 >= d.max_len:
            break
        if rows is not None:                          # row b draws what its request draws alone (uniform_fill_rows)
            keys = _row_keys(B, d.pos, row_off, row_first, row_seed)
            us = _row_uniforms(keys, steps)
        else:                                         # the counter advances by PD_T per event (uniform_fill per step)
            keys, us = None, counter_uniform(int(rng[1]), int(rng[0]) + steps, np.arange(B))
        ev_t = _event(d, live, row_off, p, settings, keys, us)
        event_commit(ev_t.data_ptr(), d.seq, d.ev_in, d.pos, B, PD_T, d.max_len, row_off, row_end, row_last, d.eos_id)
        rng[0] += PD_T
        ran += 1
        fin = any(lv and int(v) != -1 for lv, v in zip(live, last))
        if stream is not None:
            for b, off in _rows(B, row_off, live):
                q = p + off + 1
                out[b, q] = seq[b, q]
                done[b] = q
            for hook in ON_EVENT:
                hook(ran)
            if int(ctl[0]) != 0:
                by_ctl = True
                break
        if fin and exit_on_done:
            break
    if stream is not None:
        LAUNCHES.append((n_events, exit_on_done, ran, by_ctl))


def _abi(fn):
    """The C-ABI entry of stand-in fn: fn's arguments, then the stream, which the stand-ins do not use."""
    return lambda *args: fn(*args[:-1])


CALLS = {name: _abi(fn) for name, fn in (
    ("b200_gemv_bf16", gemv_bf16), ("b200_gemv_fused", gemv_fused),
    ("b200_kv_append", kv_append), ("b200_kv_append_ragged", kv_append),
    ("b200_attn_decode", attn_decode), ("b200_attn_decode_ragged", attn_decode),
    ("b200_attn_decode_fused", attn_decode_fused), ("b200_attn_decode_fused_ragged", attn_decode_fused),
    ("b200_event_commit", event_commit), ("b200_event_commit_ragged", event_commit),
    ("b200_event_commit_queue", event_commit),
    ("b200_sample_from_logits", sample_from_logits), ("b200_sample_from_logits_rows", _sample_from_logits_rows),
    ("b200_uniform_fill", uniform_fill), ("b200_uniform_fill_rows", uniform_fill_rows),
)}
CALLS["b200_decode_events_queue"] = lambda *a: decode_events(*a[:6])
CALLS["b200_decode_events_queue_rows"] = lambda *a: decode_events(*a[:6], rows=a[8:13])
CALLS["b200_decode_events_queue_stream"] = lambda *a: decode_events(*a[:6], rows=a[8:13], stream=a[13:16])
