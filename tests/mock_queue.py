"""TEST INFRASTRUCTURE: CPU stand-ins for the request-queue entries (`b200_event_commit_queue`, `b200_decode_events_queue`),
on top of tests/mock_kernels.py and tests/mock_ragged.py, so that the host scheduler of `generate_many` runs in the CPU
suite on the host-issued loop and on the persistent kernel's launch protocol.  Semantics follow include/midi_b200.h.

The persistent stand-in runs whole events from the descriptor with the mock layer's arithmetic, in the order the
host-issued loop issues it (norm+QKV, RoPE+append+attention, o_proj, gate/up, down; 8 token steps; greedy sampling), so a
greedy request gives the same events on both loops.  A row that is not live is skipped: it appends, attends, draws and
commits nothing.
"""
import math

import torch

import mock_kernels as MK
import mock_ragged
from mock_kernels import BF, _attend, _f, _from_ptr, _gather_kv, _pool, _rot

PD_T = 8


def _event_commit_queue(ev_t, seq, ev_next, pos_dev, B, T, max_len, row_off, row_end, row_last, eos_id, _s):
    pos = _from_ptr(pos_dev, 1, torch.int32)
    p = int(pos[0])
    ev = _from_ptr(ev_t, T * B, torch.int64).view(T, B).t()                # [B, T]
    out = _from_ptr(seq, B * max_len * T, torch.int64).view(B, max_len, T)
    nxt = _from_ptr(ev_next, B * T, torch.int64).view(B, T)
    offs, ends = _from_ptr(row_off, B, torch.int32).tolist(), _from_ptr(row_end, B, torch.int32).tolist()
    last = _from_ptr(row_last, B, torch.int32)
    for b in range(B):
        if int(last[b]) != -1:
            continue
        q = p + offs[b]
        if q + 1 < max_len:
            out[b, q + 1] = ev[b]
        nxt[b] = ev[b]
        if int(ev[b, 0]) == eos_id or q + 1 >= ends[b]:
            last[b] = q + 1
    pos[0] = p + 1


def _proj(x, w, n_out, K, norm=0, eps=0.0, res=None, swiglu=False, ldy=None):
    """b200_gemv_fused on the mock layer: y = [swiglu]([rmsnorm](x) @ W.T) [+ res]."""
    y = torch.empty((x.shape[0], ldy or n_out), dtype=BF)
    MK._gemv_fused(x.data_ptr(), 0, 0, 0, 0, norm, eps, w, res.data_ptr() if res is not None else 0, y.data_ptr(),
                   x.shape[0], n_out, K, x.stride(0), K, res.stride(0) if res is not None else 0, y.stride(0), int(swiglu),
                   None)
    return y


def _layers(tab, n):
    return _from_ptr(tab, n * 6, torch.int64).view(n, 6).tolist()     # qkv, o, gu, down, ln1, ln2


def _outer_attention(d, qkv, li, b, r):
    """RoPE, KV append and attention of row b at position r (b200_attn_decode_fused_ragged for one row)."""
    H, nh = d.H, d.nh_outer
    D = H // nh
    kv = _from_ptr(d.kv_outer, d.n_outer * 2, torch.int64).view(d.n_outer, 2).tolist()[li]
    B = d.batch
    kp, vp = _pool(kv[0], B, d.max_pages, nh, d.page, D), _pool(kv[1], B, d.max_pages, nh, d.page, D)
    table = _from_ptr(d.block_table, B * d.max_pages, torch.int32).view(B, d.max_pages)
    c = _from_ptr(d.cos_outer + r * D, D // 2, BF).float()[None]
    s = _from_ptr(d.sin_outer + r * D, D // 2, BF).float()[None]
    row = qkv[b]
    for col0 in (0, H):
        row[col0:col0 + H] = _rot(_f(row[col0:col0 + H]).view(nh, D), c, s, False).reshape(H).to(BF)
    pg = int(table[b, r // d.page])
    kp[pg, :, r % d.page] = row[H:2 * H].view(nh, D)
    vp[pg, :, r % d.page] = row[2 * H:].view(nh, D)
    k, v = _f(_gather_kv(kp, table, b, r + 1, d.page)), _f(_gather_kv(vp, table, b, r + 1, d.page))
    return _attend(_f(row[:H]).view(nh, D), k, v, 1.0 / math.sqrt(D)).reshape(H).to(BF)


def _event(d, live, offs, p):
    """One event of every row from ev_in: the sampled tokens, int64 [T, B] (pad for rows that are not live)."""
    B, H, V = d.batch, d.H, d.V
    ev_in = _from_ptr(d.ev_in, B * PD_T, torch.int64).view(B, PD_T)
    emb_o = _from_ptr(d.emb_outer, V * H, BF).view(V, H)
    ok = (ev_in >= 0) & (ev_in < V)                                     # the kernel embeds an out-of-range id as zero
    x = (_f(emb_o)[ev_in.clamp(0, V - 1)] * ok[..., None]).sum(-2).to(BF)
    for li, (wq, wo, wgu, wd, ln1, ln2) in enumerate(_layers(d.outer_w, d.n_outer)):
        qkv = _proj(x, wq, 3 * H, H, norm=ln1, eps=d.eps)
        attn = torch.zeros((B, H), dtype=BF)
        for b in range(B):
            if live[b]:
                attn[b] = _outer_attention(d, qkv, li, b, p + offs[b])
        h = _proj(attn, wo, H, H, res=x)
        act = _proj(h, wgu, d.I_outer, H, norm=ln2, eps=d.eps, swiglu=True)
        x = _proj(act, wd, H, d.I_outer, res=h)
    hidden = MK.rmsnorm(x, _from_ptr(d.outer_norm, H, BF), d.eps)
    nh2 = d.nh_inner
    D2 = H // nh2
    inner = _layers(d.inner_w, d.n_inner)
    pools = [(torch.zeros((B, nh2, PD_T, D2), dtype=BF), torch.zeros((B, nh2, PD_T, D2), dtype=BF)) for _ in inner]
    bt = torch.arange(B, dtype=torch.int32).view(B, 1)
    emb_i = _from_ptr(d.emb_inner, V * H, BF).view(V, H)
    ev_t = torch.full((PD_T, B), d.pad_id, dtype=torch.int64)
    mask = torch.tensor(live)
    lut = _from_ptr(d.lut, d.n_event_types * 8 * 2, torch.int32).view(d.n_event_types, 8, 2)
    n_steps = PD_T
    for i in range(PD_T):
        if i >= n_steps:
            break
        x2 = hidden if i == 0 else emb_i[ev_t[i - 1]].contiguous()
        for (wq, wo, wgu, wd, ln1, ln2), (kp, vp) in zip(inner, pools):
            qkv = _proj(x2, wq, 3 * H, H, norm=ln1, eps=d.eps)
            attn = torch.empty((B, H), dtype=BF)
            MK._attn_decode_fused(qkv.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), 1, PD_T, d.cos_inner,
                                  d.sin_inner, attn.data_ptr(), B, nh2, D2, i, 0, PD_T, 3 * H, H, 1.0 / math.sqrt(D2), 1,
                                  None, 0, None)
            h = _proj(attn, wo, H, H, res=x2)
            act = _proj(h, wgu, d.I_inner, H, norm=ln2, eps=d.eps, swiglu=True)
            x2 = _proj(act, wd, H, d.I_inner, res=h)
        logits = _proj(x2, d.lm_head, V, H, norm=d.inner_norm, eps=d.eps, ldy=d.pitch)
        MK._sample_from_logits(logits.data_ptr(), B, V, d.pitch, d.temp, d.top_p, d.top_k, i, ev_t.data_ptr(),
                               d.lut, d.n_event_types, d.eos_id, d.pad_id, d.dense_mask, 0, ev_t.data_ptr() + 8 * B * i, 1,
                               None)
        ev_t[i, ~mask] = d.pad_id                                      # a row that is not live draws nothing
        if i == 0:                                                     # token steps this event needs (live rows only)
            need = 2
            for b in range(B):
                et = int(ev_t[0, b]) - (d.eos_id + 1)
                if live[b] and int(ev_t[0, b]) != d.eos_id and 0 <= et < d.n_event_types:
                    n_par = max([s + 1 for s in range(PD_T - 1) if lut[et, s, 1] > lut[et, s, 0]], default=0)
                    need = max(need, n_par + 1)
            n_steps = min(PD_T, need)
    return ev_t


def _decode_events_queue(desc, row_off, row_end, row_last, exit_on_done, n_events, _ws, _wsb, _s):
    d = desc._obj
    B = d.batch
    pos = _from_ptr(d.pos, 1, torch.int32)
    seq = _from_ptr(d.seq, B * d.max_len * PD_T, torch.int64).view(B, d.max_len, PD_T)
    ev_in = _from_ptr(d.ev_in, B * PD_T, torch.int64).view(B, PD_T)
    rng = _from_ptr(d.rng_state, 2, torch.int64)
    offs, ends = _from_ptr(row_off, B, torch.int32).tolist(), _from_ptr(row_end, B, torch.int32).tolist()
    last = _from_ptr(row_last, B, torch.int32)
    live = [int(v) == -1 for v in last]
    for _ in range(n_events):
        p = int(pos[0])
        if p + 1 >= d.max_len:
            break
        ev = _event(d, live, offs, p).t()                                 # [B, T]
        fin = False
        for b in range(B):
            if not live[b]:
                continue
            q = p + offs[b] + 1
            seq[b, q] = ev[b]
            ev_in[b] = ev[b]
            if int(ev[b, 0]) == d.eos_id or q >= ends[b]:
                last[b], live[b], fin = q, False, True
        pos[0] = p + 1
        rng[0] += PD_T
        if not any(live) or (fin and exit_on_done):
            break


CALLS = {"b200_event_commit_queue": _event_commit_queue, "b200_decode_events_queue": _decode_events_queue}


class _Lib:
    """What the persistent loop asks of the loaded library besides calls: its workspace size."""

    @staticmethod
    def b200_decode_events_workspace_bytes(_desc):
        return 256


def _call(name, *args):
    if name in CALLS:
        return CALLS[name](*args)
    return mock_ragged._call(name, *args)


def install(monkeypatch, persist=False):
    """mock_ragged.install plus the queue entries, for the duration of one test.  `persist`: let the loop take the
    persistent kernel's path (the stand-in above) for the tiny test model, whose shapes the kernel is not built for."""
    from midi_b200 import decode, lib
    mock_ragged.install(monkeypatch)
    monkeypatch.setattr(lib, "call", _call)
    if persist:
        monkeypatch.setattr(lib, "load", lambda: _Lib())
        monkeypatch.setattr(decode.GraphGenerator, "persistent_ok", lambda self: True)
