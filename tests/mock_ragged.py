"""TEST INFRASTRUCTURE: CPU stand-ins for the ragged-generate kernel entries (`b200_*_ragged`, `ops.rope_qk_ragged_`), on
top of the mock kernel layer of tests/mock_kernels.py, so that the host logic of ragged generation runs in the CPU suite.
Semantics follow include/midi_b200.h: each entry is its counterpart with row b at the shared position + row_off[b].

`install` also replaces mock_kernels' `rope_qk_` with one that honours the device-side position base `pos0_dev`: the
graph loop's unfused (B > 16) step passes its position that way, and no earlier CPU test ran that step.
"""
import torch

import mock_kernels as MK
from mock_kernels import BF, _attend, _bfmat, _dev_int, _f, _from_ptr, _gather_kv, _pool, _rot


def rope_qk_(qkv, cos, sin, S, H, D, backward=False, pos0=0, pos0_dev=None):
    if pos0_dev is not None:
        pos0 = pos0 + int(pos0_dev.reshape(-1)[0])
    MK.rope_qk_(qkv, cos, sin, S, H, D, backward=backward, pos0=pos0)


def rope_qk_ragged_(qkv, cos, sin, S, H, D, row_off, pos0=0, pos0_dev=None):
    rows = qkv.shape[0]
    base = pos0 + (int(pos0_dev.reshape(-1)[0]) if pos0_dev is not None else 0)
    pos = base + row_off.long().repeat_interleave(S) + torch.arange(rows) % S
    c, s = cos.float()[pos][:, None], sin.float()[pos][:, None]
    for col0 in (0, H):
        blk = _f(qkv[:, col0:col0 + H]).view(rows, H // D, D)
        qkv[:, col0:col0 + H] = _rot(blk, c, s, False).reshape(rows, H).to(BF)


def _offsets(row_off, batch):
    return _from_ptr(row_off, batch, torch.int32).tolist()


def _table(bt, batch, max_pages):
    return _from_ptr(bt, batch * max_pages, torch.int32).view(batch, max_pages)


def _kv_append_ragged(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, s_new, pos0, pos0_dev, ld, row_off, _s):
    pos0 = pos0 + _dev_int(pos0_dev)
    offs = _offsets(row_off, batch)
    H = nh * D
    q = _bfmat(qkv, batch * s_new, 3 * H, ld)
    kp, vp = _pool(k_pool, batch, max_pages, nh, page, D), _pool(v_pool, batch, max_pages, nh, page, D)
    table = _table(bt, batch, max_pages)
    for b in range(batch):
        for i in range(s_new):
            pos = pos0 + offs[b] + i
            pg = int(table[b, pos // page])
            row = q[b * s_new + i]
            kp[pg, :, pos % page] = row[H:2 * H].view(nh, D)
            vp[pg, :, pos % page] = row[2 * H:].view(nh, D)


def _attn_decode_ragged(q, k_pool, v_pool, bt, max_pages, page, out, batch, s_q, nh, D, past, past_dev, max_T, ldq, ldo,
                        scale, n_split, _ws, _wsb, row_off, _s):
    past = past + _dev_int(past_dev)
    offs = _offsets(row_off, batch)
    H = nh * D
    qm, om = _bfmat(q, batch * s_q, H, ldq), _bfmat(out, batch * s_q, H, ldo)
    kp, vp = _pool(k_pool, batch, max_pages, nh, page, D), _pool(v_pool, batch, max_pages, nh, page, D)
    table = _table(bt, batch, max_pages)
    for b in range(batch):
        for i in range(s_q):
            n_pos = past + offs[b] + i + 1
            k, v = _f(_gather_kv(kp, table, b, n_pos, page)), _f(_gather_kv(vp, table, b, n_pos, page))
            om[b * s_q + i] = _attend(_f(qm[b * s_q + i]).view(nh, D), k, v, scale).reshape(H).to(BF)


def _attn_decode_fused_ragged(qkv, k_pool, v_pool, bt, max_pages, page, cos_t, sin_t, out, batch, nh, D, pos0, pos_dev,
                              max_T, ldq, ldo, scale, n_split, _ws, _wsb, row_off, _s):
    pos0 = pos0 + _dev_int(pos_dev)
    H, half = nh * D, D // 2
    q = _bfmat(qkv, batch, 3 * H, ldq)
    for b, off in enumerate(_offsets(row_off, batch)):
        c = _from_ptr(cos_t + (pos0 + off) * half * 2, half, BF).float()[None]
        s_ = _from_ptr(sin_t + (pos0 + off) * half * 2, half, BF).float()[None]
        for col0 in (0, H):
            q[b, col0:col0 + H] = _rot(_f(q[b, col0:col0 + H]).view(nh, D), c, s_, False).reshape(H).to(BF)
    _kv_append_ragged(qkv, k_pool, v_pool, bt, max_pages, page, nh, D, batch, 1, pos0, None, ldq, row_off, None)
    _attn_decode_ragged(qkv, k_pool, v_pool, bt, max_pages, page, out, batch, 1, nh, D, pos0, None, max_T, ldq, ldo, scale,
                        n_split, None, 0, row_off, None)


def _event_commit_ragged(ev_t, seq, ev_next, pos_dev, B, T, max_len, row_off, _s):
    pos = _from_ptr(pos_dev, 1, torch.int32)
    p = int(pos[0])
    ev = _from_ptr(ev_t, T * B, torch.int64).view(T, B).t()                # [B, T]
    out = _from_ptr(seq, B * max_len * T, torch.int64).view(B, max_len, T)
    for b, off in enumerate(_offsets(row_off, B)):
        if p + off + 1 < max_len:
            out[b, p + off + 1] = ev[b]
    _from_ptr(ev_next, B * T, torch.int64).view(B, T).copy_(ev)
    pos[0] = p + 1


CALLS = {"b200_kv_append_ragged": _kv_append_ragged, "b200_attn_decode_ragged": _attn_decode_ragged,
         "b200_attn_decode_fused_ragged": _attn_decode_fused_ragged, "b200_event_commit_ragged": _event_commit_ragged}
OPS = MK.OPS + ("rope_qk_ragged_",)


def _call(name, *args):
    if name in CALLS:
        return CALLS[name](*args)
    return MK._call(name, *args)


def install(monkeypatch):
    """mock_kernels.install plus the ragged entries, for the duration of one test."""
    from midi_b200 import lib, ops
    MK.install(monkeypatch)
    monkeypatch.setattr(ops, "rope_qk_", rope_qk_)
    monkeypatch.setattr(ops, "rope_qk_ragged_", rope_qk_ragged_)
    monkeypatch.setattr(lib, "call", _call)


def trace(monkeypatch, fn, names=None):
    """mock_kernels.trace over OPS, which includes rope_qk_ragged_."""
    from midi_b200 import lib, ops
    names = [] if names is None else names
    for name in OPS:
        f = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _f=f, _n=name, **k: (names.append(_n), _f(*a, **k))[1])
    call = lib.call
    monkeypatch.setattr(lib, "call", lambda n, *a: (names.append(n), call(n, *a))[1])
    fn()
    return names
