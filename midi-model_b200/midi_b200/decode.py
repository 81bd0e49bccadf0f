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


def _linear(x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """nn.Linear on a few rows: weight-streaming skinny GEMM for <= 16 rows, tensor-core GEMM otherwise."""
    M, K = x.shape
    N = w.shape[0]
    if M > 16:
        return ops.linear(x, w, residual=residual)
    y = torch.empty((M, N), dtype=BF16, device=x.device)
    lib.call("b200_gemv_bf16", x.data_ptr(), w.data_ptr(), lib.ptr(residual), y.data_ptr(), M, N, K, x.stride(0),
             w.stride(0), residual.stride(0) if residual is not None else 0, N, lib.stream())
    return y


def _lm_head(x: torch.Tensor, w: torch.Tensor, pitch: int) -> torch.Tensor:
    M, K = x.shape
    N = w.shape[0]
    if M > 16:
        return ops.linear(x, w, pitch=pitch)
    y = torch.empty((M, pitch), dtype=BF16, device=x.device)
    lib.call("b200_gemv_bf16", x.data_ptr(), w.data_ptr(), None, y.data_ptr(), M, N, K, x.stride(0), w.stride(0), 0, pitch,
             lib.stream())
    return y


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
             max_T: Optional[int] = None, final_norm: bool = True) -> torch.Tensor:
        """x: [batch * s_new, H] new inputs_embeds; appends to kv; returns final-normed hidden for the new rows.
        With `pos_dev` (int32[1] on the device) the number of cached positions is read by the kernels themselves
        (CUDA-graph replay); `max_T` then bounds the context for the split-T decode attention."""
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
        if FUSED_DECODE and s_new == 1 and B <= 16:
            return self._step_fused(x, kv, past, pos_dev, T, n_split, ws_bytes, final_norm)
        if not final_norm:
            raise lib.B200Error("final_norm=False is only available on the fused single-token path")
        for li, w in enumerate(self.eng.layers):
            n1 = ops.rmsnorm(x, w.ln1, c.eps)
            qkv = _linear(n1, w.qkv)
            ops.rope_qk_(qkv, self.cos, self.sin, s_new, H, D, pos0=past, pos0_dev=pos_dev)
            lib.call("b200_kv_append", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(), kv.block_table.data_ptr(),
                     kv.max_pages, kv.page, nh, D, B, s_new, past, pd, qkv.stride(0), lib.stream())
            if dev_pos:
                attn = torch.empty((B * s_new, H), dtype=BF16, device=x.device)
                ws = ops._ws("attn_decode", ws_bytes, x.device)
                lib.call("b200_attn_decode", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                         kv.block_table.data_ptr(), kv.max_pages, kv.page, attn.data_ptr(), B, s_new, nh, D, 0, pd, T,
                         qkv.stride(0), H, scale, n_split, ws.data_ptr(), ws.numel(), lib.stream())
            elif past == 0 and s_new > 1 and D == 64:
                attn, _ = ops.attn_causal_fwd(qkv, B, s_new, nh, D, want_lse=False)
            elif past == 0 and s_new > 1 and D == 256 and s_new <= 8:
                attn = ops.attn_tiny_fwd(qkv, B, s_new, nh, D)
            else:
                attn = torch.empty((B * s_new, H), dtype=BF16, device=x.device)
                ws = ops._ws("attn_decode", ws_bytes, x.device)
                lib.call("b200_attn_decode", qkv.data_ptr(), kv.k[li].data_ptr(), kv.v[li].data_ptr(),
                         kv.block_table.data_ptr(), kv.max_pages, kv.page, attn.data_ptr(), B, s_new, nh, D, past, None, T,
                         qkv.stride(0), H, scale, n_split, ws.data_ptr(), ws.numel(), lib.stream())
            h = _linear(attn, w.o, residual=x)
            n2 = ops.rmsnorm(h, w.ln2, c.eps)
            gu = _linear(n2, w.gu)
            act = ops.swiglu(gu)
            x = _linear(act, w.down, residual=h)
        if not dev_pos:
            kv.length = T
        return ops.rmsnorm(x, self.eng.norm, c.eps)


    def _step_fused(self, x, kv, past, pos_dev, T, n_split, ws_bytes, final_norm=True):
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
        self.graph = None
        self.stream = torch.cuda.Stream(device=dev)
        self._persist = None            # (descriptor, pointer tables, workspace) of the persistent kernel, built on first use

    # ------------------------------------------------------------------ persistent kernel (csrc/decode_persist.cu)
    def persistent_ok(self) -> bool:
        c1, c2 = self.outer.eng.cfg, self.inner.eng.cfg
        return (self.B <= 16 and 1 <= self.top_k <= 64 and c1.hidden == 1024 and c2.hidden == 1024 and c1.head_dim == 64 and c2.head_dim == 256
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
        lib.call("b200_decode_events", ctypes.byref(d), int(n), ws.data_ptr(), ws.numel(), lib.stream())

    def set_deny(self, ids) -> None:
        """Token ids that may never be sampled (empty = plain grammar)."""
        self.mask.fill_(1)
        ids = sorted(set(int(i) for i in ids))
        if ids:
            self.mask[:, torch.tensor(ids, dtype=torch.long, device=self.mask.device)] = 0

    def _event(self):
        B, T = self.B, self.T
        emb_o, emb_i = self.outer.eng.embed, self.inner.eng.embed
        e = ops.embed_sum(self.ev_in, emb_o)
        hidden = self.outer.step(e, self.kv1, 1, pos_dev=self.pos, max_T=self.max_len)
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
                logits = _lm_head(hs, self.lm_head, self.pitch)
            lib.call("b200_uniform_fill", self.u.data_ptr(), B, 0, self.counter.data_ptr(), lib.stream())
            lib.call("b200_sample_from_logits", logits.data_ptr(), B, self.V, logits.stride(0), self.temp, self.top_p,
                     self.top_k, i, self.ev_t.data_ptr(), self.g.lut.data_ptr(), self.g.n_event_types, self.g.eos, self.g.pad,
                     self.mask.data_ptr(), self.u.data_ptr(), self.ev_t.data_ptr() + 8 * B * i, 1, lib.stream())
        lib.call("b200_event_commit", self.ev_t.data_ptr(), self.seq.data_ptr(), self.ev_in.data_ptr(), self.pos.data_ptr(),
                 B, T, self.max_len, lib.stream())

    def _set_state(self, prompt: torch.Tensor):
        """prompt [B, P, T]: events 0..P-2 are prefilled into the KV cache; event P-1 is fed by the first replay."""
        P = prompt.shape[1]
        self.seq.fill_(self.tok.pad_id)
        self.seq[:, :P] = prompt
        self.kv1.reset()
        if P > 1:
            e = ops.embed_sum(prompt[:, :P - 1].reshape(self.B * (P - 1), self.T).contiguous(), self.outer.eng.embed)
            self.outer.step(e, self.kv1, P - 1)
        self.pos.fill_(P - 1)
        self.ev_in.copy_(prompt[:, P - 1])
        self.counter.copy_(torch.tensor([0, self.seed], dtype=torch.int64))

    def _prepare(self, prompt: torch.Tensor, use_graph) -> None:
        """Load the prompt into the device state; capture the per-event graph on first use (current stream = self.stream)."""
        self._set_state(prompt)
        if self.table_version != self.outer.version:    # RoPE tables were re-created: the captured addresses are stale
            self.graph, self.table_version = None, self.outer.version
        if use_graph == "persist":
            return
        if use_graph and self.graph is None:
            self._event()                       # warm-up (allocations, function attributes) outside capture
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                self._event()
            self.graph = g
            self._set_state(prompt)             # undo the warm-up's state changes

    def _mode(self, use_graph):
        """True / "graph": CUDA-graph replay per event; False: the same launches issued from the host; "persist": the
        persistent kernel (falls back to the graph loop for shapes it is not built for)."""
        if use_graph == "persist" and not self.persistent_ok():
            return True
        return use_graph

    def events(self, prompt: torch.Tensor, use_graph=True):
        """Generator form (app.py:27-120): yields each new event as an int64 [B, T] CPU tensor right after its graph
        replay / kernel -- one device->host copy per EVENT, none per token -- and stops after the event in which every row
        emitted EOS (app.py:119) or at max_len."""
        use_graph = self._mode(use_graph)
        P = prompt.shape[1]
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self._prepare(prompt, use_graph)
        for i in range(self.max_len - P):
            with torch.cuda.stream(self.stream):          # not held across the yield
                if use_graph == "persist":
                    self._events_persistent(1)
                elif use_graph:
                    self.graph.replay()
                else:
                    self._event()
                ev = self.seq[:, P + i].cpu()              # synchronises on this event only
            yield ev
            if bool((ev[:, 0] == self.tok.eos_id).all()):
                break
        cur.wait_stream(self.stream)

    def run(self, prompt: torch.Tensor, use_graph=True, check_every: int = 32, progress=None,
            stop_on_eos: bool = True, max_new: Optional[int] = None) -> torch.Tensor:
        """`max_new` stops after that many generated events although the pools (and the split-T attention) are sized for
        max_len: a serving process keeps ONE loop with full-context pools and cuts individual requests short."""
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
            self._prepare(prompt, use_graph)
            done = 0
            stop_at = None
            while done < n_new:
                n = min(check_every, n_new - done)
                if use_graph == "persist":
                    self._events_persistent(n)           # one launch for the whole block of events
                else:
                    for _ in range(n):
                        if use_graph:
                            self.graph.replay()
                        else:
                            self._event()
                done += n
                if progress is not None:
                    progress(n)
                if not stop_on_eos:
                    continue
                first = self.seq[:, P:P + done, 0]                       # event-type token of every generated event
                all_eos = (first == self.tok.eos_id).all(dim=0)          # one small D2H sync per `check_every` events
                hit = torch.nonzero(all_eos)
                if hit.numel() > 0:
                    stop_at = P + int(hit[0].item()) + 1                 # the all-EOS event itself is kept
                    break
            out = self.seq[:, :(stop_at if stop_at is not None else P + done)].clone()
        cur.wait_stream(self.stream)
        return out
