"""KV-cached inference of the two stacks and the device-side generate() loop.

Replaces hf DynamicCache's per-step `torch.cat` (cache_utils.py:102-121) with a paged KV cache
(pages of 64 positions for the outer stack, 8 for the inner one; per-row block tables) that the
QKV/RoPE step appends to and a split-T single-query attention kernel reads.  The sampling step
(midi_model.py:202-223) -- grammar mask, temperature softmax, top-p / top-k, draw -- is one
kernel per token with the grammar held on the device as id ranges, so the only host<->device
traffic per generated event is the 8-byte-per-row read of the event-type token that the
reference's `end` / early-exit logic needs (midi_model.py:224-237, 248).
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from . import lib, ops
from .engine import StackCfg, StackEngine

BF16 = torch.bfloat16


class PagedKV:
    """Per-stack paged KV cache for `batch` rows and up to `capacity` positions."""

    def __init__(self, cfg: StackCfg, batch: int, capacity: int, page: int, device):
        self.cfg, self.batch, self.page = cfg, batch, page
        self.max_pages = (capacity + page - 1) // page
        self.capacity = self.max_pages * page
        n_pages = batch * self.max_pages
        shape = (n_pages, cfg.n_head, page, cfg.head_dim)
        self.k = [torch.empty(shape, dtype=BF16, device=device) for _ in range(cfg.n_layer)]
        self.v = [torch.empty(shape, dtype=BF16, device=device) for _ in range(cfg.n_layer)]
        # identity block table: row b owns pages [b*max_pages, (b+1)*max_pages)
        self.block_table = torch.arange(n_pages, dtype=torch.int32, device=device).view(batch, self.max_pages).contiguous()
        self.length = 0

    def reset(self):
        self.length = 0

    def row(self, b: int) -> "PagedKV":
        """Row b alone as a batch-1 cache over the same memory (its slice of every pool, an identity block table), empty:
        a request's prefill into its slot runs exactly as a batch-1 prefill does.  Never grown."""
        v = PagedKV.__new__(PagedKV)
        v.cfg, v.batch, v.page, v.max_pages, v.capacity, v.length = self.cfg, 1, self.page, self.max_pages, self.capacity, 0
        rows = slice(b * self.max_pages, (b + 1) * self.max_pages)
        v.k, v.v = [k[rows] for k in self.k], [x[rows] for x in self.v]
        v.block_table = self.block_table[:1]              # row 0 of the identity table: pages 0 .. max_pages - 1
        return v

    def table_row(self, b: int) -> "PagedKV":
        """Row b of the block table as a batch-1 cache over the whole pools, empty: a prefill through it writes the pages
        that row b's entries name, which need not be the row's own range (shared prompts, GraphGenerator.run_queue).
        Never grown."""
        v = PagedKV.__new__(PagedKV)
        v.cfg, v.batch, v.page, v.max_pages, v.capacity, v.length = self.cfg, 1, self.page, self.max_pages, self.capacity, 0
        v.k, v.v = list(self.k), list(self.v)
        v.block_table = self.block_table[b:b + 1]
        return v

    def identity_table(self) -> None:
        """Row b owns pages [b * max_pages, (b+1) * max_pages) again."""
        n = self.batch * self.max_pages
        self.block_table.copy_(torch.arange(n, dtype=torch.int32).view(self.batch, self.max_pages))

    def grow(self, capacity: int) -> None:
        """Re-allocate the pools for at least `capacity` positions, keeping the cached keys / values (row b owns pages
        [b * max_pages, (b+1) * max_pages), so the old pages are copied to the front of each row's new range).  The
        reference's DynamicCache has no capacity (hf cache_utils.py:119-120 keeps concatenating); neither may we."""
        if capacity <= self.capacity:
            return
        old_mp = self.max_pages
        self.max_pages = (max(capacity, 2 * self.capacity) + self.page - 1) // self.page
        self.capacity = self.max_pages * self.page
        c = self.cfg
        dev = self.block_table.device
        shape = (self.batch * self.max_pages, c.n_head, self.page, c.head_dim)
        for pools in (self.k, self.v):
            for li in range(c.n_layer):
                new = torch.empty(shape, dtype=BF16, device=dev)
                new.view(self.batch, self.max_pages, c.n_head, self.page, c.head_dim)[:, :old_mp].copy_(
                    pools[li].view(self.batch, old_mp, c.n_head, self.page, c.head_dim))
                pools[li] = new
        self.block_table = torch.arange(self.batch * self.max_pages, dtype=torch.int32, device=dev).view(
            self.batch, self.max_pages).contiguous()


def _share_keys(prompts, page: int) -> list:
    """Share key of each request of a queue call (prompts: int64 [L, T] tensors): the index of the first request with an
    equal prompt, or None.  Only prompts of at least page + 1 events share, so that at least one whole page is prefilled;
    a prompt that no other request repeats gets None.  A hash of the bytes only picks the candidates: equality is exact."""
    keys = [None] * len(prompts)
    by_shape = {}
    for i, p in enumerate(prompts):
        if p.shape[0] - 1 >= page:
            by_shape.setdefault(tuple(p.shape), []).append(i)
    for idx in by_shape.values():
        if len(idx) < 2:
            continue
        host = {i: prompts[i].cpu().numpy() for i in idx}
        firsts = {}                                  # hash of the bytes -> first requests with those bytes
        for i in idx:
            cands = firsts.setdefault(hash(host[i].tobytes()), [])
            keys[i] = next((j for j in cands if np.array_equal(host[i], host[j])), None)
            if keys[i] is None:
                cands.append(i)
                keys[i] = i
    count = {}
    for k in keys:
        count[k] = count.get(k, 0) + 1
    return [k if k is not None and count[k] > 1 else None for k in keys]


class SharedPages:
    """Page assignment of a queue call in which requests share prompts.  The outer cache keeps its batch * max_pages pages;
    they are handed out from a host free list and each slot's block-table row is written when the slot takes a request.

    A request of L prompt events with share key k reads positions below S = ((L - 1) // page) * page from k's shared
    pages, which the first request of k prefills and the last live one of k gives back.  Every other entry of its row is a
    private page; the one at S, the prompt's tail page, also holds prompt positions S .. L - 2 and is copied for each
    later sharer.  A request has max_pages distinct pages at most and sharing only lowers the total, so the pool suffices.

    An empty slot still appends on the graph and host-issued loops (at positions 0, 1, 2, ... of its row), so every entry
    of its row names one private page of the last request it held; it keeps that page until the call ends.  A slot is
    only left empty when no request waits, so no later admission can be handed that page."""

    def __init__(self, kv: PagedKV):
        self.kv = kv
        self.n_pages = kv.batch * kv.max_pages
        self.free = list(range(self.n_pages - 1, -1, -1))
        self.groups = {}                          # share key -> (shared page ids, live slots)
        self.rows = [None] * kv.batch             # page ids of slot b's block-table row, as written
        self.held = [[] for _ in range(kv.batch)]  # private pages of slot b
        self.key = [None] * kv.batch              # share key of slot b's live request
        self.shared = [0] * kv.batch              # S of slot b's live request (0: nothing shared)

    def _take(self, n: int) -> list:
        if n > len(self.free):
            raise lib.B200Error(f"KV page pool exhausted: {n} pages wanted, {len(self.free)} free")
        return [self.free.pop() for _ in range(n)]

    def _write(self, b: int, row: list) -> None:
        self.rows[b] = row
        self.kv.block_table[b].copy_(torch.tensor(row, dtype=torch.int32))

    def release(self, b: int) -> None:
        """Slot b's request finished: its share of the prompt's pages goes back (with the last live sharer)."""
        k = self.key[b]
        if k is not None:
            pages, live = self.groups[k]
            live.remove(b)
            if not live:
                self.free.extend(reversed(pages))
                del self.groups[k]
        self.key[b], self.shared[b] = None, 0

    def admit(self, b: int, L: int, key) -> Optional[int]:
        """Row b for a request of L prompt events and share key `key` (None: shares nothing).  Returns a live sharer's slot
        whose tail page holds the prompt, or None when the request must be prefilled."""
        self.free.extend(reversed(self.held[b]))
        page, mp = self.kv.page, self.kv.max_pages
        S = (L - 1) // page * page if key is not None else 0
        group = self.groups.get(key) if key is not None else None
        src = group[1][0] if group is not None else None
        if key is not None and group is None:
            group = self.groups[key] = (self._take(S // page), [])
        self.held[b] = self._take(mp - S // page)
        if group is not None:
            group[1].append(b)
        self.key[b], self.shared[b] = key, S
        self._write(b, (group[0] if group is not None else []) + self.held[b])
        return src

    def copy_tail(self, src: int, b: int, L: int) -> None:
        """Prompt positions S .. L - 2 of sharer `src`'s tail page into b's (nothing when L - 1 == S)."""
        if L - 1 == self.shared[b]:
            return
        t = self.shared[b] // self.kv.page
        s, d = self.rows[src][t], self.rows[b][t]
        for pools in (self.kv.k, self.kv.v):
            for pool in pools:
                pool[d].copy_(pool[s])

    def park(self, b: int) -> None:
        """Slot b stays empty: every entry of its row names one private page of its last request (a free one if it never
        held a request)."""
        if not self.held[b]:
            self.held[b] = self._take(1)
        self.free.extend(reversed(self.held[b][1:]))
        self.held[b] = self.held[b][:1]
        self._write(b, self.held[b] * self.kv.max_pages)

    def close(self) -> None:
        """End of the call: every page back on the free list, and the identity table restored."""
        for b in range(self.kv.batch):
            self.release(b)
            self.free.extend(reversed(self.held[b]))
            self.held[b] = []
        self.kv.identity_table()


def _linear(x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None,
            pitch: Optional[int] = None) -> torch.Tensor:
    """nn.Linear on a few rows: weight-streaming skinny GEMM for <= 16 rows, tensor-core GEMM otherwise.  `pitch`: row
    pitch of the output when N is not a multiple of 8 (lm_head, V = 3406 -> 3408)."""
    M, K = x.shape
    N = w.shape[0]
    if M > 16:
        return ops.linear(x, w, residual=residual, pitch=pitch)
    y = torch.empty((M, pitch or N), dtype=BF16, device=x.device)
    lib.call("b200_gemv_bf16", x.data_ptr(), w.data_ptr(), lib.ptr(residual), y.data_ptr(), M, N, K, x.stride(0),
             w.stride(0), residual.stride(0) if residual is not None else 0, y.stride(0), lib.stream())
    return y


def _lm_head(x: torch.Tensor, w: torch.Tensor, pitch: int) -> torch.Tensor:
    """Logits projection into rows of `pitch` columns (kept for existing callers; same code path as _linear)."""
    return _linear(x, w, pitch=pitch)


def _gemv_fused(x, w, n_out, *, ids=None, table=None, norm_w=None, eps=0.0, residual=None, swiglu=False, ldy=None):
    """y[B, n_out] = [swiglu]([rmsnorm](x or table[ids]) @ w.T) [+ residual]   (B <= 16 rows, one launch)."""
    B = x.shape[0] if x is not None else ids.shape[0]
    K = w.shape[1]
    y = torch.empty((B, ldy or n_out), dtype=BF16, device=w.device)
    lib.call("b200_gemv_fused", lib.ptr(x), lib.ptr(ids), ids.stride(0) if ids is not None else 0, lib.ptr(table),
             table.shape[0] if table is not None else 0, lib.ptr(norm_w), float(eps), w.data_ptr(), lib.ptr(residual),
             y.data_ptr(), B, n_out, K, x.stride(0) if x is not None else 0, w.stride(0),
             residual.stride(0) if residual is not None else 0, y.stride(0), int(swiglu), lib.stream())
    return y


FUSED_DECODE = __import__("os").environ.get("B200_FUSED_DECODE", "1") != "0"


class CachedStack:
    """Incremental forward of one stack over a PagedKV (inference only)."""

    def __init__(self, eng: StackEngine, max_pos: int, inv_freq: torch.Tensor):
        self.eng = eng
        self.inv_freq = inv_freq
        self.cos, self.sin = ops.rope_table(inv_freq, max_pos)
        self.max_pos = max_pos
        self.version = 0            # bumped when the tables are re-created (captured graphs hold the old addresses)

    def ensure_positions(self, n_pos: int) -> bool:
        """cos/sin tables for positions 0 .. n_pos-1.  `max_position_embeddings` (4096) is only the initial size: hf computes
        the rotation from the position ids on the fly (modeling_llama.py:124-135), so contexts longer than that are legal
        (app.py: max_len = prompt + up to 4096 generated events).  Returns True when the tables were re-created."""
        if n_pos <= self.max_pos:
            return False
        self.max_pos = max(n_pos, 2 * self.max_pos)
        self.cos, self.sin = ops.rope_table(self.inv_freq, self.max_pos)
        self.version += 1
        return True

    def step(self, x: torch.Tensor, kv: PagedKV, s_new: int, pos_dev: Optional[torch.Tensor] = None,
             max_T: Optional[int] = None, final_norm: bool = True, row_off: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x: [batch * s_new, H] new inputs_embeds; appends to kv; returns final-normed hidden for the new rows.
        With `pos_dev` (int32[1] on the device) the number of cached positions is read by the kernels themselves
        (CUDA-graph replay); `max_T` then bounds the context for the split-T decode attention.  `row_off` (int32 [batch]
        on the device, with `pos_dev` only): row b sits at *pos_dev + row_off[b] (ragged generate, the `_ragged` entries)."""
        c = self.eng.cfg
        H, D, nh = c.hidden, c.head_dim, c.n_head
        B = kv.batch
        dev_pos = pos_dev is not None
        past = 0 if dev_pos else kv.length
        T = max_T if dev_pos else past + s_new
        if dev_pos:
            # graph replay: pools and tables were sized by the generator (addresses are baked into the graph)
            if T > kv.capacity or T > self.max_pos:
                raise lib.B200Error(f"KV cache overflow: {T} positions > capacity {min(kv.capacity, self.max_pos)}")
        else:
            self.ensure_positions(T)
            kv.grow(T)
        scale = 1.0 / math.sqrt(D)
        n_split = max(1, min(32, (T + 255) // 256)) if D == 64 else 1
        pd = lib.ptr(pos_dev)
        ws_bytes = lib.query("b200_attn_decode_workspace_bytes", B * s_new, nh, D, n_split)
        if row_off is not None and not dev_pos:
            raise lib.B200Error("row_off needs device-side positions (pos_dev)")
        if FUSED_DECODE and s_new == 1 and B <= 16:
            return self._step_fused(x, kv, past, pos_dev, T, n_split, ws_bytes, final_norm, row_off)
        if not final_norm:
            raise lib.B200Error("final_norm=False is only available on the fused single-token path")
        prefill = not dev_pos and past == 0 and s_new > 1        # prompt into an empty cache: causal attention kernels
        for li, w in enumerate(self.eng.layers):
            n1 = ops.rmsnorm(x, w.ln1, c.eps)
            qkv = _linear(n1, w.qkv)
            if row_off is not None:
                ops.rope_qk_ragged_(qkv, self.cos, self.sin, s_new, H, D, row_off, pos0=past, pos0_dev=pos_dev)
                lib.call("b200_kv_append_ragged", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                         kv.block_table.data_ptr(), kv.max_pages, kv.page, nh, D, B, s_new, past, pd, qkv.stride(0),
                         row_off.data_ptr(), lib.stream())
            else:
                ops.rope_qk_(qkv, self.cos, self.sin, s_new, H, D, pos0=past, pos0_dev=pos_dev)
                lib.call("b200_kv_append", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(), kv.block_table.data_ptr(),
                         kv.max_pages, kv.page, nh, D, B, s_new, past, pd, qkv.stride(0), lib.stream())
            if prefill and D == 64:
                attn, _ = ops.attn_causal_fwd(qkv, B, s_new, nh, D, want_lse=False)
            elif prefill and D == 256 and s_new <= 8:
                attn = ops.attn_tiny_fwd(qkv, B, s_new, nh, D)
            else:
                # the cached length is `past` (host) or *pos_dev (graph replay, past = 0)
                attn = torch.empty((B * s_new, H), dtype=BF16, device=x.device)
                ws = ops._ws("attn_decode", ws_bytes, x.device)
                if row_off is not None:
                    lib.call("b200_attn_decode_ragged", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                             kv.block_table.data_ptr(), kv.max_pages, kv.page, attn.data_ptr(), B, s_new, nh, D, past, pd, T,
                             qkv.stride(0), H, scale, n_split, ws.data_ptr(), ws.numel(), row_off.data_ptr(), lib.stream())
                else:
                    lib.call("b200_attn_decode", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                             kv.block_table.data_ptr(), kv.max_pages, kv.page, attn.data_ptr(), B, s_new, nh, D, past, pd, T,
                             qkv.stride(0), H, scale, n_split, ws.data_ptr(), ws.numel(), lib.stream())
            h = _linear(attn, w.o, residual=x)
            n2 = ops.rmsnorm(h, w.ln2, c.eps)
            gu = _linear(n2, w.gu)
            act = ops.swiglu(gu)
            x = _linear(act, w.down, residual=h)
        if not dev_pos:
            kv.length = T
        return ops.rmsnorm(x, self.eng.norm, c.eps)


    def _step_fused(self, x, kv, past, pos_dev, T, n_split, ws_bytes, final_norm=True, row_off=None):
        """Single-token step with 5 launches per layer: norm+QKV, RoPE+append+attention, o_proj+residual,
        norm+gate/up+SwiGLU, down+residual.  Same rounding points as the unfused kernels (bit-identical)."""
        c = self.eng.cfg
        H, D, nh = c.hidden, c.head_dim, c.n_head
        B = kv.batch
        scale = 1.0 / math.sqrt(D)
        pd = lib.ptr(pos_dev)
        ws = ops._ws("attn_decode", ws_bytes, kv.block_table.device)
        for li, w in enumerate(self.eng.layers):
            qkv = _gemv_fused(x, w.qkv, 3 * H, norm_w=w.ln1, eps=c.eps)
            attn = torch.empty((B, H), dtype=BF16, device=qkv.device)
            if row_off is not None:
                lib.call("b200_attn_decode_fused_ragged", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                         kv.block_table.data_ptr(), kv.max_pages, kv.page, self.cos.data_ptr(), self.sin.data_ptr(),
                         attn.data_ptr(), B, nh, D, past, pd, T, qkv.stride(0), H, scale, n_split, ws.data_ptr(),
                         ws.numel(), row_off.data_ptr(), lib.stream())
            else:
                lib.call("b200_attn_decode_fused", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                         kv.block_table.data_ptr(), kv.max_pages, kv.page, self.cos.data_ptr(), self.sin.data_ptr(),
                         attn.data_ptr(), B, nh, D, past, pd, T, qkv.stride(0), H, scale, n_split, ws.data_ptr(), ws.numel(),
                         lib.stream())
            h = _gemv_fused(attn, w.o, H, residual=x)
            act = _gemv_fused(h, w.gu, c.inner, norm_w=w.ln2, eps=c.eps, swiglu=True)
            x = _gemv_fused(act, w.down, H, residual=h)
        if pos_dev is None:
            kv.length = T
        if not final_norm:
            return x                                  # caller fuses the final norm into the next projection (lm_head)
        return ops.rmsnorm(x, self.eng.norm, c.eps)


class GrammarLUT:
    """Device copy of the tokenizer grammar as id ranges (midi_tokenizer.py:517-535)."""

    def __init__(self, tok, device):
        self.eos, self.pad = tok.eos_id, tok.pad_id
        ev_ids = sorted(tok.event_ids.values())
        if ev_ids != list(range(self.eos + 1, self.eos + 1 + len(ev_ids))):
            raise lib.B200Error("event ids are not contiguous after eos: the range-based grammar does not apply")
        self.n_event_types = len(ev_ids)
        lut = np.zeros((self.n_event_types, 8, 2), dtype=np.int32)
        self.n_params = {}
        for name, params in tok.events.items():
            e = tok.event_ids[name] - (self.eos + 1)
            self.n_params[tok.event_ids[name]] = len(params)
            for i, pn in enumerate(params):
                ids = tok.parameter_ids[pn]
                if list(ids) != list(range(ids[0], ids[0] + len(ids))):
                    raise lib.B200Error(f"parameter ids of {pn} are not contiguous")
                lut[e, i] = (ids[0], ids[-1] + 1)
        self.lut = torch.from_numpy(lut).to(device)


def sample_from_logits(logits: torch.Tensor, V: int, temp: float, top_p: float, top_k: int, step: int,
                       event_tok: torch.Tensor, g: GrammarLUT, uniforms: torch.Tensor, out: torch.Tensor,
                       dense_mask: Optional[torch.Tensor] = None):
    """logits [B, pitch] bf16 -> out[:, step] (int64 [B, 8] event buffer)."""
    B = logits.shape[0]
    lib.call("b200_sample_from_logits", logits.data_ptr(), B, V, logits.stride(0), temp, top_p, top_k, step,
             event_tok.data_ptr(), g.lut.data_ptr(), g.n_event_types, g.eos, g.pad, lib.ptr(dense_mask), uniforms.data_ptr(),
             out.data_ptr() + 8 * step, out.stride(0), lib.stream())


class GraphGenerator:
    """Device-resident generate loop: ONE CUDA graph = one generated event (the event-level decode step, the 8
    token-level decode steps with their sampler launches, and the bookkeeping), replayed once per event.

    State lives on the device: `pos` (events already in the KV cache), `ev_in` (the event fed to the event-level
    stack next), `seq` (the output), the RNG counter.  Every inner step always runs (tokens past an event's last
    parameter are forced to pad by the grammar, exactly what the reference pads with, midi_model.py:239-241), so
    no host decision is needed inside an event; the reference's stop rule -- all rows emitted EOS in the same
    event (midi_model.py:248) -- is applied on the host every `check_every` events and the output truncated there.

    Ragged prompts (`lengths`, set per call): row b continues its own first L_b events.  The shared `pos` stays the loop's
    counter (its exit, the attention's chunk grid and the events per launch stay uniform) and row b sits at
    pos + row_off[b], row_off[b] = L_b - max(L) <= 0, through the `_ragged` kernel entries; that mode has its own graph.
    """

    def __init__(self, outer: CachedStack, inner: CachedStack, lm_head: torch.Tensor, pitch: int, V: int, tok,
                 grammar: GrammarLUT, batch: int, max_len: int, temp: float, top_p: float, top_k: int, seed: int):
        dev = lm_head.device
        self.outer, self.inner, self.lm_head, self.pitch, self.V = outer, inner, lm_head, pitch, V
        self.tok, self.g, self.B, self.max_len = tok, grammar, batch, max_len
        self.T = tok.max_token_seq
        outer.ensure_positions(max_len)            # max_len may exceed max_position_embeddings (app.py: prompt + 4096 new events)
        self.table_version = outer.version
        self.temp, self.top_p, self.top_k, self.seed = float(temp), float(top_p), int(top_k), int(seed) & ((1 << 63) - 1)
        self.kv1 = PagedKV(outer.eng.cfg, batch, max_len, 64, dev)
        self.kv2 = PagedKV(inner.eng.cfg, batch, self.T, self.T, dev)
        self.pos = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ev_in = torch.zeros((batch, self.T), dtype=torch.long, device=dev)
        self.ev_t = torch.zeros((self.T, batch), dtype=torch.long, device=dev)
        self.seq = torch.full((batch, max_len, self.T), tok.pad_id, dtype=torch.long, device=dev)
        self.u = torch.zeros(batch, dtype=torch.float32, device=dev)
        self.counter = torch.zeros(2, dtype=torch.int64, device=dev)   # {call counter, seed} read by the RNG kernel
        # extra sampling mask ANDed with the grammar ranges (app.py:27-34,73-87: disable_patch_change /
        # disable_control_change / disable_channels); its address is baked into the graph, its contents are not
        self.mask = torch.ones((batch, V), dtype=torch.uint8, device=dev)
        self.row_off = torch.zeros(batch, dtype=torch.int32, device=dev)    # ragged mode: row b at pos + row_off[b]
        self.lengths = None             # ragged mode of the current call: int64 [B] prompt lengths on the device, else None
        # request-queue mode (run_queue): row b stops at its own EOS or at seq index row_end[b]; row_last[b] is -1 while
        # the row is live, then the seq index of its last event (-2: empty slot)
        self.queue = False
        self.row_end = torch.zeros(batch, dtype=torch.int32, device=dev)
        self.row_last = torch.full((batch,), -2, dtype=torch.int32, device=dev)
        # per-request queue (run_queue with `settings`): slot b's request samples with its own temp / top_p / top_k and
        # draws hash(row_seed[b], 8 j + t, 0) at its new event j = pos + row_off[b] - row_first[b] (the `_rows` entries);
        # the arrays are allocated by the first per-request call (alloc_rows)
        self.rows = False
        self.req_top_k = []             # top_k of every request of the current per-request call (persistent_ok)
        self.row_temp = self.row_top_p = self.row_top_k = self.row_seed = self.row_first = None
        self.graph = None
        self.graph_ragged = None
        self.graph_queue = None
        self.graph_queue_rows = None
        self.stream = torch.cuda.Stream(device=dev)
        self._persist = None            # (descriptor, pointer tables, workspace) of the persistent kernel, built on first use

    def alloc_rows(self) -> None:
        """The per-request arrays, allocated by the first per-request call: a loop that only runs scalar settings does
        not carry them."""
        if self.row_temp is None:
            dev, B = self.pos.device, self.B
            self.row_temp = torch.ones(B, dtype=torch.float32, device=dev)
            self.row_top_p = torch.ones(B, dtype=torch.float32, device=dev)
            self.row_top_k = torch.ones(B, dtype=torch.int32, device=dev)
            self.row_seed = torch.zeros(B, dtype=torch.int64, device=dev)
            self.row_first = torch.zeros(B, dtype=torch.int32, device=dev)

    # ------------------------------------------------------------------ persistent kernel (csrc/decode_persist.cu)
    def persistent_ok(self) -> bool:
        """Whether the persistent kernel runs this loop's current call: at most 32 slots in per-request mode (the `_rows`
        kernels run their rows in groups of 16), 16 otherwise, every top_k in 1..128, and a model it is built for."""
        c1, c2 = self.outer.eng.cfg, self.inner.eng.cfg
        top_ks = self.req_top_k if self.rows else [self.top_k]
        return (self.B <= (32 if self.rows else 16) and all(1 <= k <= 128 for k in top_ks)
                and c1.hidden == 1024 and c2.hidden == 1024 and c1.head_dim == 64 and c2.head_dim == 256
                and c1.inner % 256 == 0 and c2.inner % 256 == 0 and self.T == 8 and self.kv1.page % 32 == 0)

    def _persistent(self):
        """b200_decode_desc for this loop's state: whole events run inside ONE cooperative kernel (one CTA per SM, grid
        barriers between the dependent phases) instead of ~210 launches per event."""
        if self._persist is not None and self._persist[0] == self.outer.version:
            return self._persist[1:]
        import ctypes
        dev = self.lm_head.device

        def table(eng):
            rows = [[w.qkv.data_ptr(), w.o.data_ptr(), w.gu.data_ptr(), w.down.data_ptr(), w.ln1.data_ptr(), w.ln2.data_ptr()]
                    for w in eng.layers]
            return torch.tensor(rows, dtype=torch.int64, device=dev)

        t_outer, t_inner = table(self.outer.eng), table(self.inner.eng)
        t_kv = torch.tensor([[k.data_ptr(), v.data_ptr()] for k, v in zip(self.kv1.k, self.kv1.v)], dtype=torch.int64, device=dev)
        c1, c2 = self.outer.eng.cfg, self.inner.eng.cfg
        d = lib.DecodeDesc()
        d.outer_w, d.inner_w, d.n_outer, d.n_inner = t_outer.data_ptr(), t_inner.data_ptr(), c1.n_layer, c2.n_layer
        d.outer_norm, d.inner_norm = self.outer.eng.norm.data_ptr(), self.inner.eng.norm.data_ptr()
        d.lm_head, d.emb_outer, d.emb_inner = self.lm_head.data_ptr(), self.outer.eng.embed.data_ptr(), self.inner.eng.embed.data_ptr()
        d.H, d.I_outer, d.I_inner, d.nh_outer, d.nh_inner = c1.hidden, c1.inner, c2.inner, c1.n_head, c2.n_head
        d.V, d.pitch, d.eps = self.V, self.pitch, c1.eps
        d.kv_outer, d.block_table = t_kv.data_ptr(), self.kv1.block_table.data_ptr()
        d.max_pages, d.page = self.kv1.max_pages, self.kv1.page
        d.cos_outer, d.sin_outer = self.outer.cos.data_ptr(), self.outer.sin.data_ptr()
        d.cos_inner, d.sin_inner = self.inner.cos.data_ptr(), self.inner.sin.data_ptr()
        d.pos, d.ev_in, d.seq, d.max_len = self.pos.data_ptr(), self.ev_in.data_ptr(), self.seq.data_ptr(), self.max_len
        d.rng_state, d.dense_mask, d.lut = self.counter.data_ptr(), self.mask.data_ptr(), self.g.lut.data_ptr()
        d.n_event_types, d.eos_id, d.pad_id = self.g.n_event_types, self.g.eos, self.g.pad
        d.temp, d.top_p, d.top_k, d.batch = self.temp, self.top_p, max(1, self.top_k), self.B
        self.prof = None
        if __import__("os").environ.get("B200_DECODE_PROFILE"):
            self.prof = torch.zeros(128, dtype=torch.int64, device=dev)
            d.prof = self.prof.data_ptr()
        nbytes = lib.load().b200_decode_events_workspace_bytes(ctypes.byref(d))
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        off = (-ws.data_ptr()) % 256
        self._persist = (self.outer.version, d, ws[off:off + nbytes], (t_outer, t_inner, t_kv))
        return self._persist[1:]

    def _events_persistent(self, n: int) -> None:
        """Run `n` generated events in one launch (stops early inside the kernel at max_len)."""
        import ctypes
        d, ws, _ = self._persistent()
        if self.lengths is not None:
            lib.call("b200_decode_events_ragged", ctypes.byref(d), self.row_off.data_ptr(), int(n), ws.data_ptr(), ws.numel(),
                     lib.stream())
        else:
            lib.call("b200_decode_events", ctypes.byref(d), int(n), ws.data_ptr(), ws.numel(), lib.stream())

    def _events_queue(self, n: int, exit_on_done: bool) -> None:
        """Queue mode: up to `n` events in one launch, which also ends when no row is live or, with `exit_on_done`, after
        the event in which a row finished."""
        import ctypes
        d, ws, _ = self._persistent()
        if self.rows:
            lib.call("b200_decode_events_queue_rows", ctypes.byref(d), self.row_off.data_ptr(), self.row_end.data_ptr(),
                     self.row_last.data_ptr(), int(exit_on_done), int(n), ws.data_ptr(), ws.numel(),
                     self.row_temp.data_ptr(), self.row_top_p.data_ptr(), self.row_top_k.data_ptr(),
                     self.row_seed.data_ptr(), self.row_first.data_ptr(), lib.stream())
        else:
            lib.call("b200_decode_events_queue", ctypes.byref(d), self.row_off.data_ptr(), self.row_end.data_ptr(),
                     self.row_last.data_ptr(), int(exit_on_done), int(n), ws.data_ptr(), ws.numel(), lib.stream())

    def set_deny(self, ids) -> None:
        """Token ids that may never be sampled (empty = plain grammar)."""
        self.mask.fill_(1)
        ids = sorted(set(int(i) for i in ids))
        if ids:
            self.mask[:, torch.tensor(ids, dtype=torch.long, device=self.mask.device)] = 0

    def _event(self):
        B, T = self.B, self.T
        emb_o, emb_i = self.outer.eng.embed, self.inner.eng.embed
        ragged = self.lengths is not None or self.queue
        e = ops.embed_sum(self.ev_in, emb_o)
        hidden = self.outer.step(e, self.kv1, 1, pos_dev=self.pos, max_T=self.max_len,
                                 row_off=self.row_off if ragged else None)
        self.kv2.reset()
        for i in range(T):
            if i == 0:
                xin = ops.inner_input(hidden, None, emb_i)
            else:
                xin = ops.inner_input(None, self.ev_t[i - 1].view(B, 1), emb_i)
            if FUSED_DECODE and B <= 16:
                hs = self.inner.step(xin, self.kv2, 1, final_norm=False)      # final norm fused into the lm_head GEMV
                logits = _gemv_fused(hs, self.lm_head, self.V, norm_w=self.inner.eng.norm, eps=self.inner.eng.cfg.eps,
                                     ldy=self.pitch)
            else:
                hs = self.inner.step(xin, self.kv2, 1)
                logits = _linear(hs, self.lm_head, pitch=self.pitch)
            if self.rows:
                lib.call("b200_uniform_fill_rows", self.u.data_ptr(), B, self.pos.data_ptr(), self.row_off.data_ptr(),
                         self.row_first.data_ptr(), self.row_seed.data_ptr(), i, lib.stream())
                lib.call("b200_sample_from_logits_rows", logits.data_ptr(), B, self.V, logits.stride(0),
                         self.row_temp.data_ptr(), self.row_top_p.data_ptr(), self.row_top_k.data_ptr(), i,
                         self.ev_t.data_ptr(), self.g.lut.data_ptr(), self.g.n_event_types, self.g.eos, self.g.pad,
                         self.mask.data_ptr(), self.u.data_ptr(), self.ev_t.data_ptr() + 8 * B * i, 1, lib.stream())
                continue
            lib.call("b200_uniform_fill", self.u.data_ptr(), B, 0, self.counter.data_ptr(), lib.stream())
            lib.call("b200_sample_from_logits", logits.data_ptr(), B, self.V, logits.stride(0), self.temp, self.top_p,
                     self.top_k, i, self.ev_t.data_ptr(), self.g.lut.data_ptr(), self.g.n_event_types, self.g.eos, self.g.pad,
                     self.mask.data_ptr(), self.u.data_ptr(), self.ev_t.data_ptr() + 8 * B * i, 1, lib.stream())
        if self.queue:
            lib.call("b200_event_commit_queue", self.ev_t.data_ptr(), self.seq.data_ptr(), self.ev_in.data_ptr(),
                     self.pos.data_ptr(), B, T, self.max_len, self.row_off.data_ptr(), self.row_end.data_ptr(),
                     self.row_last.data_ptr(), self.g.eos, lib.stream())
        elif ragged:
            lib.call("b200_event_commit_ragged", self.ev_t.data_ptr(), self.seq.data_ptr(), self.ev_in.data_ptr(),
                     self.pos.data_ptr(), B, T, self.max_len, self.row_off.data_ptr(), lib.stream())
        else:
            lib.call("b200_event_commit", self.ev_t.data_ptr(), self.seq.data_ptr(), self.ev_in.data_ptr(),
                     self.pos.data_ptr(), B, T, self.max_len, lib.stream())

    def _set_state(self, prompt: torch.Tensor):
        """prompt [B, P, T]: events 0..P-2 are prefilled into the KV cache; event P-1 is fed by the first replay.
        Ragged mode (P = max(L)): events >= L_b of row b are set to pad first; the rectangular prefill is still exact, since
        attention is causal (no real event reads a later pad event) and the slot a pad event fills in row b is >= L_b - 1,
        which the decode step writes before it first reads it.  Row b's first fed event is its event L_b - 1."""
        P = prompt.shape[1]
        if self.lengths is not None:
            past = torch.arange(P, device=prompt.device)[None, :] >= self.lengths[:, None]
            prompt = prompt.masked_fill(past[:, :, None], self.tok.pad_id)
        self.seq.fill_(self.tok.pad_id)
        self.seq[:, :P] = prompt
        self.kv1.reset()
        if P > 1:
            e = ops.embed_sum(prompt[:, :P - 1].reshape(self.B * (P - 1), self.T).contiguous(), self.outer.eng.embed)
            self.outer.step(e, self.kv1, P - 1)
        self.pos.fill_(P - 1)
        if self.lengths is not None:
            self.ev_in.copy_(prompt[torch.arange(self.B, device=prompt.device), self.lengths - 1])
            self.row_off.copy_(self.lengths - P)
        else:
            self.ev_in.copy_(prompt[:, P - 1])
        self.counter.copy_(torch.tensor([0, self.seed], dtype=torch.int64))

    def _set_lengths(self, prompt: torch.Tensor, lengths) -> None:
        """Ragged mode for this call (`lengths`: B ints in [1, P], max(lengths) == P, checked by the caller) or not (None)."""
        if lengths is None:
            self.lengths = None
            return
        if len(lengths) != self.B or max(lengths) != prompt.shape[1] or min(lengths) < 1:
            raise lib.B200Error(f"lengths {list(lengths)} do not fit a prompt of {prompt.shape[1]} events and {self.B} rows")
        self.lengths = torch.tensor(list(lengths), dtype=torch.int64).to(self.seq.device)

    def _graph(self):
        if self.queue:
            return self.graph_queue_rows if self.rows else self.graph_queue
        return self.graph_ragged if self.lengths is not None else self.graph

    def _capture(self, use_graph, set_state) -> None:
        """Capture the per-event graph of the current mode on first use (current stream = self.stream); `set_state()`
        loads the call's state and undoes the warm-up's changes to it."""
        set_state()
        if self.table_version != self.outer.version:    # RoPE tables were re-created: the captured addresses are stale
            self.graph, self.table_version = None, self.outer.version
            self.graph_ragged = self.graph_queue = self.graph_queue_rows = None
        if use_graph == "persist":
            return
        if use_graph and self._graph() is None:
            self._event()                       # warm-up (allocations, function attributes) outside capture
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                self._event()
            if self.queue and self.rows:
                self.graph_queue_rows = g
            elif self.queue:
                self.graph_queue = g
            elif self.lengths is not None:
                self.graph_ragged = g
            else:
                self.graph = g
            set_state()

    def _prepare(self, prompt: torch.Tensor, use_graph, lengths=None) -> None:
        """Load the prompt into the device state; capture the per-event graph of this mode (rectangular or ragged) on first
        use (current stream = self.stream)."""
        self.queue = self.rows = False
        self._set_lengths(prompt, lengths)
        self._capture(use_graph, lambda: self._set_state(prompt))

    def _mode(self, use_graph):
        """True / "graph": CUDA-graph replay per event; False: the same launches issued from the host; "persist": the
        persistent kernel (falls back to the graph loop for shapes it is not built for)."""
        if use_graph == "persist" and not self.persistent_ok():
            return True
        return use_graph

    def events(self, prompt: torch.Tensor, use_graph=True, lengths=None):
        """Generator form (app.py:27-120): yields each new event as an int64 [B, T] CPU tensor right after its graph
        replay / kernel -- one device->host copy per EVENT, none per token -- and stops after the event in which every row
        emitted EOS (app.py:119) or at max_len.  `lengths`: ragged prompt (see run); row b's i-th new event is its event
        L_b + i."""
        use_graph = self._mode(use_graph)
        P = prompt.shape[1]
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self._prepare(prompt, use_graph, lengths)
            rows = torch.arange(self.B, device=self.seq.device) if self.lengths is not None else None
        for i in range(self.max_len - P):
            with torch.cuda.stream(self.stream):          # not held across the yield
                if use_graph == "persist":
                    self._events_persistent(1)
                elif use_graph:
                    self._graph().replay()
                else:
                    self._event()
                if self.lengths is not None:
                    ev = self.seq[rows, self.lengths + i].cpu()
                else:
                    ev = self.seq[:, P + i].cpu()          # synchronises on this event only
            yield ev
            if bool((ev[:, 0] == self.tok.eos_id).all()):
                break
        cur.wait_stream(self.stream)

    def run(self, prompt: torch.Tensor, use_graph=True, check_every: int = 32, progress=None,
            stop_on_eos: bool = True, max_new: Optional[int] = None, lengths=None) -> torch.Tensor:
        """`max_new` stops after that many generated events although the pools (and the split-T attention) are sized for
        max_len: a serving process keeps ONE loop with full-context pools and cuts individual requests short.
        `lengths` (B ints, max(lengths) == P): ragged prompt, row b being its first L_b events.  Every row gets the same
        number n of new events; the result is the data.collate layout [B, P + n, T]: row b's L_b prompt events, its n new
        events, then pad events."""
        P = prompt.shape[1]
        n_new = self.max_len - P
        if max_new is not None:
            n_new = min(n_new, int(max_new))
        use_graph = self._mode(use_graph)
        if n_new <= 0:
            return prompt
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self._prepare(prompt, use_graph, lengths)
            graph = self._graph()
            done = 0
            stop_at = None
            while done < n_new:
                n = min(check_every, n_new - done)
                if use_graph == "persist":
                    self._events_persistent(n)           # one launch for the whole block of events
                else:
                    for _ in range(n):
                        if use_graph:
                            graph.replay()
                        else:
                            self._event()
                done += n
                if progress is not None:
                    progress(n)
                if not stop_on_eos:
                    continue
                if self.lengths is not None:                             # row b's generated events are at L_b + j
                    idx = self.lengths[:, None] + torch.arange(done, device=self.seq.device)[None, :]
                    first = self.seq[:, :, 0].gather(1, idx)
                else:
                    first = self.seq[:, P:P + done, 0]                   # event-type token of every generated event
                all_eos = (first == self.tok.eos_id).all(dim=0)          # one small D2H sync per `check_every` events
                hit = torch.nonzero(all_eos)
                if hit.numel() > 0:
                    stop_at = P + int(hit[0].item()) + 1                 # the all-EOS event itself is kept
                    break
            out = self.seq[:, :(stop_at if stop_at is not None else P + done)].clone()
            if self.lengths is not None:
                # rows end at L_b + n_done: events a row generated past the stop point (same check_every block) become pad
                pad_past(out, self.lengths + (out.shape[1] - P), self.tok.pad_id)
        cur.wait_stream(self.stream)
        return out

    # ------------------------------------------------------------------ request queue (continuous batching)
    def _set_queue_state(self) -> None:
        """Every slot empty, the shared counter at 0, the RNG counter at its start."""
        self.seq.fill_(self.tok.pad_id)
        self.ev_in.fill_(self.tok.pad_id)
        self.pos.zero_()
        self.row_off.zero_()
        self.row_end.zero_()
        self.row_last.fill_(-2)
        self.counter.copy_(torch.tensor([0, self.seed], dtype=torch.int64))

    def _admit(self, b: int, prompt: torch.Tensor, setting=None, pages: Optional[SharedPages] = None, key=None) -> None:
        """Request `prompt` (int64 [L, T] on the device) into slot b: events 0 .. L-2 prefilled at batch 1 into the slot's
        pages (nothing for a one-event prompt), event L-1 fed to the next event.  Per-request mode: `setting` = (temp, top_p,
        top_k, seed, denied token ids) becomes slot b's settings, RNG key (row_first = L-1: its new event j is at seq index
        L + j) and mask row.  With `pages` (a call that shares prompts) slot b's row is written first and the prefill goes
        through it; a request whose prompt a live request of the same share `key` already holds is not prefilled, it only
        gets its own copy of the prompt's tail page."""
        L = prompt.shape[0]
        if setting is not None:
            temp, top_p, top_k, seed, deny = setting
            self.row_temp[b], self.row_top_p[b], self.row_top_k[b] = temp, top_p, top_k
            self.row_seed[b], self.row_first[b] = seed, L - 1
            self.mask[b].fill_(1)
            if deny:
                self.mask[b, torch.tensor(sorted(deny), dtype=torch.long, device=self.mask.device)] = 0
        self.seq[b].fill_(self.tok.pad_id)
        self.seq[b, :L] = prompt
        src = pages.admit(b, L, key) if pages is not None else None
        if src is not None:
            pages.copy_tail(src, b, L)
        elif L > 1:
            kv = self.kv1.row(b) if pages is None else self.kv1.table_row(b)
            self.outer.step(ops.embed_sum(prompt[:L - 1].contiguous(), self.outer.eng.embed), kv, L - 1)
        self.ev_in[b] = prompt[L - 1]

    def run_queue(self, prompts, budgets, use_graph=True, settings=None) -> list:
        """Continuous batching: requests i = 0 .. N-1 (prompts[i]: int64 [L_i, T] on the device, L_i >= 1; budgets[i] >= 1
        new events) through this loop's B slots.  Request i ends after its first new event whose event type is EOS (that
        event is kept) or after budgets[i] new events, and its slot is refilled with the next waiting request.  Returns
        request i's prompt and new events, int64 [L_i + n_i, T] on the device, in input order.

        Row b sits at pos + row_off[b], as in ragged mode.  Between launches a finished slot takes the next request (its
        batch-1 prefill) or becomes empty, and the rows are rebased: pos = the largest live position, row_off[b] = r_b - pos
        <= 0, an empty slot at position 0.  So the kernel's `pos + 1 >= max_len` exit never comes before a budget, and an
        empty slot's position stays below a live row's.  The persistent kernel runs until a row finishes while requests
        wait (exit_on_done), else until no row is live; the graph and host-issued loops check after every event.

        `settings` (per-request mode): one (temp, top_p, top_k, seed, denied token ids) per request, with temp > 0,
        0 < top_p <= 1, top_k >= 1 (checked by the caller).  Request i then samples with its own settings and mask row and
        draws what a batch-1 loop seeded `seed` draws, through the `_rows` entries; the persistent kernel needs every top_k
        <= 128 and at most 32 slots.  Without it, every slot shares this loop's settings, seed stream and mask.

        Requests with equal prompts of at least 65 events (`_share_keys`) share the KV pages of the prompt's whole pages
        (SharedPages): the first one resident is prefilled, a later one only copies the prompt's tail page from a live
        sharer.  Every kernel addresses the cache through the block table, so no request's result changes by a bit.  A call
        without such a pair keeps the identity block table and prefills every request into its slot's own pages."""
        self.rows = settings is not None
        self.req_top_k = [s[2] for s in settings] if self.rows else []
        if self.rows:
            self.alloc_rows()
        use_graph = self._mode(use_graph)
        N, B = len(prompts), self.B
        ends = [p.shape[0] - 1 + int(n) for p, n in zip(prompts, budgets)]     # seq index of each request's last event
        if max(ends) >= self.max_len:
            raise lib.B200Error(f"a request ends at event {max(ends)}, past this loop's max_len {self.max_len}")
        out = [None] * N
        slot = [None] * B                  # request held by slot b (None: empty)
        posn = [0] * B                     # position of slot b's row: the seq index of the event it feeds next
        nxt = 0
        keys = _share_keys(prompts, self.kv1.page)
        # a call without a shared prompt keeps the identity block table and each slot's own pages
        pages = SharedPages(self.kv1) if any(k is not None for k in keys) else None
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self.queue, self.lengths = True, None
            self._capture(use_graph, self._set_queue_state)
            graph = self._graph()
            free = list(range(B))
            try:
                while True:
                    if free:
                        if pages is not None:
                            for b in free:
                                pages.release(b)       # all before any admission: a finished group's pages may be reused
                        for b in free:
                            slot[b] = None
                            if nxt < N:
                                self._admit(b, prompts[nxt], settings[nxt] if self.rows else None, pages, keys[nxt])
                                slot[b], posn[b] = nxt, prompts[nxt].shape[0] - 1
                                nxt += 1
                            elif pages is not None:
                                pages.park(b)
                        live = [b for b in range(B) if slot[b] is not None]
                        if not live:
                            break
                        pos = max(posn[b] for b in live)
                        offs = [posn[b] - pos if slot[b] is not None else -pos for b in range(B)]
                        self.pos.fill_(pos)
                        self.row_off.copy_(torch.tensor(offs, dtype=torch.int32))
                        self.row_end.copy_(torch.tensor([ends[s] if s is not None else 0 for s in slot], dtype=torch.int32))
                        self.row_last.copy_(torch.tensor([-1 if s is not None else -2 for s in slot], dtype=torch.int32))
                    if use_graph == "persist":
                        self._events_queue(max(ends[slot[b]] - posn[b] for b in live), exit_on_done=nxt < N)
                    elif use_graph:
                        graph.replay()
                    else:
                        self._event()
                    state = torch.cat([self.pos, self.row_last]).cpu()          # one small device->host copy per launch
                    p_now, last = int(state[0]), state[1:].tolist()
                    free = []
                    for b in live:
                        if last[b] >= 0:
                            out[slot[b]] = self.seq[b, :last[b] + 1].clone()
                            free.append(b)
                        else:
                            posn[b] = p_now + offs[b]
                    live = [b for b in live if b not in free]
            finally:
                if pages is not None:
                    pages.close()
        cur.wait_stream(self.stream)
        return out


def pad_past(x: torch.Tensor, ends: torch.Tensor, pad_id: int) -> torch.Tensor:
    """In place on [B, S, T] events: row b's events >= ends[b] become pad events (the data.collate layout)."""
    past = torch.arange(x.shape[1], device=x.device)[None, :] >= ends.to(x.device)[:, None]
    return x.masked_fill_(past[:, :, None], pad_id)
