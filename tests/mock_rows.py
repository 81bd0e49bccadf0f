"""TEST INFRASTRUCTURE: CPU stand-ins for the per-request queue entries (`b200_sample_from_logits_rows`,
`b200_uniform_fill_rows`, `b200_decode_events_queue_rows`), on top of tests/mock_queue.py, so that `generate_many`'s
per-request mode runs in the CPU suite on the host-issued loop and on the persistent kernel's launch protocol.  Semantics
follow include/midi_b200.h.

Unlike the greedy mock layer, the samplers here draw: softmax of logits / temp over the vocabulary, the grammar range and
mask, top-k then top-p on the sorted probabilities, and the uniform picks from the renormalised mass (top_k = 1 is the
mock layer's argmax).  `b200_uniform_fill` writes the counter-based uniforms of the kernels, so a sampled `generate` at
batch 1 and a sampled request draw alike.  Every draw of a sampler is appended to DRAWS as a dict (row, u, temp, top_p,
top_k, denied ids, step, and -- where the caller keyed it -- seed and event j).
"""
import numpy as np
import torch

import mock_kernels as MK
import mock_queue
from mock_kernels import _bfmat, _f, _from_ptr

M64 = (1 << 64) - 1
DRAWS = []


def counter_uniform(seed, c, i):
    """sampler.cuh counter_uniform: draw i of counter value c under `seed`."""
    z = (seed + 0x9E3779B97F4A7C15 * (c * 4096 + i + 1)) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    z ^= z >> 31
    return float(np.float32(z >> 40) * np.float32(1.0 / 16777216.0))


def _range(step, ev, table, n_event_types, eos_id, pad_id):
    if step == 0:
        return eos_id, eos_id + 1 + n_event_types
    e = ev - (eos_id + 1)
    if ev == eos_id or e < 0 or e >= n_event_types:
        return pad_id, pad_id + 1
    lo, hi = int(table[e, step - 1, 0]), int(table[e, step - 1, 1])
    return (lo, hi) if hi > lo else (pad_id, pad_id + 1)


def _draw(lg, lo, hi, mrow, temp, top_p, top_k, u):
    """One row: lg float [V] logits, mrow uint8 [V] or None."""
    allowed = torch.zeros_like(lg, dtype=torch.bool)
    allowed[lo:hi] = True
    if mrow is not None:
        allowed &= mrow != 0
    if top_k == 1:                                          # the mock layer's greedy sampler
        x = lg.clone()
        x[~allowed] = float("-inf")
        return lo + int(torch.argmax(x[lo:hi]))
    p = torch.softmax(lg.double() / temp, 0)
    p[~allowed] = 0
    ids = sorted((i for i in range(lg.numel()) if p[i] > 0), key=lambda i: (-float(p[i]), i))[:top_k]
    if not ids:
        return lo
    keep, cum = [], 0.0
    for i in ids:
        if cum > top_p:
            break
        keep.append(i)
        cum += float(p[i])
    total = sum(float(p[i]) for i in keep)
    run = 0.0
    for i in keep:
        run += float(p[i])
        if run > u * total:
            return i
    return keep[-1]


def _sample(logits, rows, V, ld, temps, top_ps, top_ks, step, event_tok, lut, n_event_types, eos_id, pad_id, dense_mask,
            us, out, out_stride, keys=None):
    lg = _f(_bfmat(logits, rows, V, ld))
    mask = _from_ptr(dense_mask, rows * V, torch.uint8).view(rows, V) if dense_mask else None
    table = _from_ptr(lut, n_event_types * 8 * 2, torch.int32).view(n_event_types, 8, 2)
    ev = _from_ptr(event_tok, rows, torch.int64)
    o = _from_ptr(out, (rows - 1) * out_stride + 1, torch.int64)
    for r in range(rows):
        lo, hi = _range(step, int(ev[r]), table, n_event_types, eos_id, pad_id)
        mrow = mask[r] if mask is not None else None
        o[r * out_stride] = _draw(lg[r], lo, hi, mrow, float(temps[r]), float(top_ps[r]), int(top_ks[r]), float(us[r]))
        rec = dict(row=r, u=float(us[r]), temp=float(temps[r]), top_p=float(top_ps[r]), top_k=int(top_ks[r]), step=step,
                   deny=sorted(torch.nonzero(mrow == 0).flatten().tolist()) if mrow is not None else [])
        if keys is not None:
            rec["seed"], rec["j"] = keys[r]
        DRAWS.append(rec)


def _sample_from_logits(logits, rows, V, ld, temp, top_p, top_k, step, event_tok, lut, n_event_types, eos_id, pad_id,
                        dense_mask, uniforms, out, out_stride, _s):
    us = _from_ptr(uniforms, rows, torch.float32).tolist() if uniforms else [0.0] * rows
    _sample(logits, rows, V, ld, [temp] * rows, [top_p] * rows, [max(1, top_k)] * rows, step, event_tok, lut,
            n_event_types, eos_id, pad_id, dense_mask, us, out, out_stride)


def _uniform_fill(u, n, seed, state, _s):
    st = _from_ptr(state, 2, torch.int64)
    c, key = int(st[0]), (seed ^ int(st[1])) & M64
    _from_ptr(u, n, torch.float32).copy_(torch.tensor([counter_uniform(key, c, i) for i in range(n)]))
    st[0] += 1


_KEYS = {}                  # u pointer -> [(seed, j)] of the last b200_uniform_fill_rows into it


def _row_keys(B, pos, row_off, row_first, row_seed):
    p = int(_from_ptr(pos, 1, torch.int32)[0])
    offs, first = _from_ptr(row_off, B, torch.int32).tolist(), _from_ptr(row_first, B, torch.int32).tolist()
    seeds = _from_ptr(row_seed, B, torch.int64).tolist()
    return [(seeds[b], p + offs[b] - first[b]) for b in range(B)]


def _uniform_fill_rows(u, B, pos_dev, row_off, row_first, row_seed, step, _s):
    keys = _row_keys(B, pos_dev, row_off, row_first, row_seed)
    _from_ptr(u, B, torch.float32).copy_(torch.tensor([counter_uniform(s, 8 * j + step, 0) for s, j in keys]))
    _KEYS[u] = keys


def _sample_from_logits_rows(logits, rows, V, ld, row_temp, row_top_p, row_top_k, step, event_tok, lut, n_event_types,
                             eos_id, pad_id, dense_mask, uniforms, out, out_stride, _s):
    _sample(logits, rows, V, ld, _from_ptr(row_temp, rows, torch.float32).tolist(),
            _from_ptr(row_top_p, rows, torch.float32).tolist(), _from_ptr(row_top_k, rows, torch.int32).tolist(), step,
            event_tok, lut, n_event_types, eos_id, pad_id, dense_mask, _from_ptr(uniforms, rows, torch.float32).tolist(),
            out, out_stride, keys=_KEYS.get(uniforms))


def _decode_events_queue_rows(desc, row_off, row_end, row_last, exit_on_done, n_events, ws, wsb, row_temp, row_top_p,
                              row_top_k, row_seed, row_first, s):
    """mock_queue's persistent stand-in, with each row's settings and keyed draws in its sampler."""
    d = desc._obj
    B = d.batch
    temps = _from_ptr(row_temp, B, torch.float32).tolist()
    top_ps = _from_ptr(row_top_p, B, torch.float32).tolist()
    top_ks = _from_ptr(row_top_k, B, torch.int32).tolist()

    def sampler(logits, rows, V, ld, _t, _p, _k, step, event_tok, lut, n_et, eos_id, pad_id, dense_mask, _u, out, ostr, _s):
        keys = _row_keys(B, d.pos, row_off, row_first, row_seed)
        us = [counter_uniform(sd, 8 * j + step, 0) for sd, j in keys]
        _sample(logits, rows, V, ld, temps, top_ps, top_ks, step, event_tok, lut, n_et, eos_id, pad_id, dense_mask, us,
                out, ostr, keys=keys)

    greedy = MK._sample_from_logits
    MK._sample_from_logits = sampler
    try:
        mock_queue._decode_events_queue(desc, row_off, row_end, row_last, exit_on_done, n_events, ws, wsb, s)
    finally:
        MK._sample_from_logits = greedy


CALLS = {"b200_sample_from_logits": _sample_from_logits, "b200_uniform_fill": _uniform_fill,
         "b200_sample_from_logits_rows": _sample_from_logits_rows, "b200_uniform_fill_rows": _uniform_fill_rows,
         "b200_decode_events_queue_rows": _decode_events_queue_rows}


def _call(name, *args):
    if name in CALLS:
        return CALLS[name](*args)
    return mock_queue._call(name, *args)


def install(monkeypatch, persist=False):
    """mock_queue.install plus the entries above, for the duration of one test."""
    from midi_b200 import lib
    mock_queue.install(monkeypatch, persist=persist)
    monkeypatch.setattr(lib, "call", _call)
    DRAWS.clear()
    _KEYS.clear()
