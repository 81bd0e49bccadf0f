"""Layer-by-layer execution of the two Llama stacks of MIDIModel on the sm_90a kernels.

`ParamStore` keeps every parameter (and gradient) of the model as a view into ONE flat bf16
buffer, in `named_parameters()` order.  Because q/k/v and gate/up projections are adjacent in
that order, the fused `[3H, H]` QKV and `[2I, H]` gate|up weights are *views* -- the reference's
`state_dict` keys stay the source of truth and no packed
copies exist.  One flat gradient buffer means one all-reduce and one AdamW launch per step.

`StackEngine` runs forward (saving exactly what backward needs) and an explicit backward; there
is no autograd graph inside -- `autograd.Function`s in midi_model.py wrap whole stacks.
Math per layer: hf modeling_llama.py:303-332; rounding points: DESIGN.md 3.3.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from . import lib, ops
from . import lora as _lora

import os

BF16 = torch.bfloat16
# RoPE backward is fused into the attention backward kernels (B200_FUSE_ROPE=0 -> stand-alone kernel).
# The forward fusion into the QKV GEMM epilogue exists (ops.linear_rope, bit-identical) but is OFF by default
# (B200_FUSE_ROPE_FWD=1 turns it on).
FUSE_ROPE = os.environ.get("B200_FUSE_ROPE", "1") != "0"
FUSE_ROPE_FWD = os.environ.get("B200_FUSE_ROPE_FWD", "0") != "0"
# SwiGLU formed in the epilogue of the gate|up GEMM (ops.linear_swiglu, bit-identical to GEMM + stand-alone kernel): ON.
# It removes the stand-alone kernel and its round trip of the [rows, 2I] activation through HBM.
# B200_FUSE_SWIGLU=0 restores GEMM + kernel.
FUSE_SWIGLU = os.environ.get("B200_FUSE_SWIGLU", "1") != "0"
# Weight-gradient GEMMs on a second stream: dW = dY^T X is off the backward's critical path, so it can run
# under the HBM-bound kernels that follow on the main stream (SwiGLU / RMSNorm backward leave the tensor pipe idle, and an
# elementwise CTA fits next to a GEMM CTA on an SM).  B200_WGRAD_STREAM=0 keeps everything on one stream.
WGRAD_STREAM = os.environ.get("B200_WGRAD_STREAM", "1") != "0"
_side_streams: dict = {}


def _side_stream(device) -> torch.cuda.Stream:
    s = _side_streams.get(device.index)
    if s is None:
        s = torch.cuda.Stream(device=device, priority=0)     # main work keeps the default (same) priority class
        _side_streams[device.index] = s
    return s


def _wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, accumulate: bool, side, hold=None) -> None:
    """dW (+)= dY^T X, on `side` when given: ordered after everything queued so far on the current stream; the caller
    joins `side` back before the gradients are consumed.  The operands must outlive the side GEMM: `hold` (a list) takes a
    reference the caller drops only after an event recorded on `side` has been waited for; with hold=None the caller
    guarantees the lifetime itself.  (Tensor.record_stream would also do, but it makes the caching allocator unable to
    reuse those blocks while the host runs ahead of the device: the 0.9 GB logits / dlogits block of every step then
    triggers fresh cudaMallocs -- measured +5 ms per step.)"""
    if side is None:
        ops.linear_wgrad(dy, x, dw, accumulate)
        return
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.linear_wgrad(dy, x, dw, accumulate)
    if hold is not None:
        hold.append((dy, x))


ALIGN = 256   # elements; AdamW's no-decay flags are per 256-element block


def _require_device(n: str, p: torch.Tensor, dev) -> None:
    if p.device != dev or p.dtype != BF16 or not p.is_cuda:
        raise lib.B200Error(f"parameter {n} is {p.dtype} on {p.device}: the native path needs the whole model in "
                            "bfloat16 on one CUDA device (model.to('cuda', dtype=torch.bfloat16)); no fallback")


class ParamStore:
    def __init__(self, module: torch.nn.Module):
        named = list(module.named_parameters())
        if not named:
            raise lib.B200Error("model has no parameters")
        dev = named[0][1].device
        for n, p in named:
            _require_device(n, p, dev)
        # Flat layout: the base parameters in named_parameters() order (q|k|v and gate|up adjacent), then -- when LoRA
        # adapters are injected (midi_b200/lora.py, train.py:439-449) -- every adapter matrix, grouped per layer with the A
        # matrices of q|k|v and gate|up adjacent.  The trainable parameters of a LoRA run are then ONE contiguous tail
        # [base_numel, numel): one all-reduce slice, one AdamW launch, moments only for the adapters.
        base = [(n, p) for n, p in named if ".lora_" not in n]
        lora = sorted(((n, p) for n, p in named if ".lora_" in n), key=lambda t: _lora.flat_order_key(t[0]))
        named = base + lora
        self.device = dev
        self.names = [n for n, _ in named]
        self.offsets = {}
        off = 0
        self.base_numel = None
        for n, p in named:
            if self.base_numel is None and ".lora_" in n:
                self.base_numel = off
            self.offsets[n] = off
            off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        if self.base_numel is None:
            self.base_numel = off
        self.flat = torch.zeros(off, dtype=BF16, device=dev)
        self.gflat = torch.zeros(off, dtype=BF16, device=dev)
        self.views = {}
        self.gviews = {}
        with torch.no_grad():
            for n, p in named:
                o = self.offsets[n]
                v = self.flat[o:o + p.numel()].view(p.shape)
                v.copy_(p.data)
                p.data = v
                self.views[n] = v
                self.gviews[n] = self.gflat[o:o + p.numel()].view(p.shape)
        self._params = dict(named)
        self.rg_sig = tuple(p.requires_grad for _, p in named)
        # [train_lo, train_hi): the span of the flat buffer that holds every trainable parameter; `train_dense` when no
        # frozen parameter sits inside it (full training: everything; LoRA: the adapter tail) -- what the fused optimizer
        # and the data-parallel gradient average run over
        tr = [n for n, p in named if p.requires_grad]
        if tr:
            self.train_lo = self.offsets[tr[0]]
            self.train_hi = self._end(tr[-1])
            inside = [n for n in self.names if self.train_lo <= self.offsets[n] < self.train_hi]
            self.train_dense = all(self._params[n].requires_grad for n in inside)
        else:
            self.train_lo = self.train_hi = 0
            self.train_dense = True
        # no-decay flags (train.py:123-131: names containing 'bias' or 'norm')
        flags = torch.zeros(off // ALIGN, dtype=torch.uint8)
        for n, p in named:
            if "bias" in n or "norm" in n:
                o = self.offsets[n] // ALIGN
                flags[o:o + (p.numel() + ALIGN - 1) // ALIGN] = 1
        self.nodecay = flags.to(dev)

    def _end(self, name: str) -> int:
        return self.offsets[name] + (self.views[name].numel() + ALIGN - 1) // ALIGN * ALIGN

    def valid(self) -> bool:
        """False once somebody re-created or re-pointed ANY parameter (.to(dtype), .cuda(), p.data = ..., ...): the
        engine reads the flat buffer, so a parameter living elsewhere would silently be ignored.  Also False when a
        parameter's requires_grad changed (model.requires_grad_(False), train.py:440): which gradients are computed, and the
        span the fused optimizer updates, are decided when the runtime is built."""
        views, params = self.views, self._params
        for n, rg in zip(self.names, self.rg_sig):
            p = params[n]
            if p.data_ptr() != views[n].data_ptr() or p.requires_grad != rg:
                return False
        return True

    def trainable(self, name: str) -> bool:
        return self._params[name].requires_grad

    def wname(self, path: str) -> str:
        """Parameter name of the weight of the Linear at `path` (peft / midi_b200.lora wrap it as `.base_layer`)."""
        n = path + ".weight"
        if n in self.views:
            return n
        n = path + ".base_layer.weight"
        if n in self.views:
            return n
        raise lib.B200Error(f"no weight parameter for module {path}")

    def fused(self, names: List[str]) -> torch.Tensor:
        """[sum(rows), cols] view over adjacent 2-D parameters (q|k|v or gate|up)."""
        first = self.views[names[0]]
        o = self.offsets[names[0]]
        rows = 0
        for n in names:
            v = self.views[n]
            if self.offsets[n] != o + rows * first.shape[1] or v.shape[1] != first.shape[1]:
                raise lib.B200Error(f"parameters {names} are not adjacent in the flat buffer")
            rows += v.shape[0]
        return self.flat[o:o + rows * first.shape[1]].view(rows, first.shape[1])

    def fused_grad(self, names: List[str]) -> torch.Tensor:
        first = self.views[names[0]]
        o = self.offsets[names[0]]
        rows = sum(self.views[n].shape[0] for n in names)
        return self.gflat[o:o + rows * first.shape[1]].view(rows, first.shape[1])

    def publish_grads(self):
        """Expose the flat gradient buffer as `.grad` of every parameter (for train.py / torch optimizers)."""
        for n, p in self._params.items():
            if p.requires_grad:
                p.grad = self.gviews[n]

    def zero_grad(self):
        self.gflat.zero_()


@dataclass
class StackCfg:
    prefix: str
    n_layer: int
    n_head: int
    hidden: int
    inner: int
    eps: float

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_head


class LoraW:
    """One adapted projection of one layer: y = x W^T + scale * (x A^T) B^T  (peft lora/layer.py Linear.forward)."""
    __slots__ = ("A", "B", "scale", "r", "a_name", "b_name")


class LayerW:
    """Weights of one decoder layer (views into the flat buffer).  `tr_*`: does the base weight get a gradient (False for
    the frozen base of a LoRA run, train.py:440); `lora`: projection key ("q","k","v","o","gate","up","down") -> LoraW."""
    __slots__ = ("qkv", "o", "gu", "down", "ln1", "ln2", "tr_qkv", "tr_o", "tr_gu", "tr_down", "tr_ln1", "tr_ln2", "lora")


class LayerG:
    __slots__ = ("qkv", "o", "gu", "down", "ln1", "ln2", "lora")


_LORA_KEYS = (("q", "self_attn.q_proj"), ("k", "self_attn.k_proj"), ("v", "self_attn.v_proj"), ("o", "self_attn.o_proj"),
              ("gate", "mlp.gate_proj"), ("up", "mlp.up_proj"), ("down", "mlp.down_proj"))


class StackGrads:
    """Gradient views of one stack.  `spans` = [(buffer or None, lo, hi)]: flat-layout ranges [lo, hi) and the buffer that
    backs each of them (the store's own gradient buffer at offset 0, or a private buffer starting at `lo`); a parameter
    whose range has no buffer -- or that does not require a gradient -- has the view None and its gradient is not computed."""

    def __init__(self, eng: "StackEngine", spans):
        store, cfg = eng.store, eng.cfg
        self.store, self.spans = store, spans
        p = cfg.prefix
        H = cfg.hidden

        def view(name, rows=None, need=True):
            if not need:
                return None
            v = store.views[name]
            o = store.offsets[name]
            for buf, lo, hi in spans:
                if lo <= o < hi:
                    if buf is None:
                        return None
                    if rows is None:
                        return buf[o - lo:o - lo + v.numel()].view(v.shape)
                    return buf[o - lo:o - lo + rows * v.shape[1]].view(rows, v.shape[1])
            return None

        self._view = view
        self.layers = []
        for l, w in enumerate(eng.layers):
            a = f"{p}.layers.{l}.self_attn."
            m = f"{p}.layers.{l}.mlp."
            g = LayerG()
            g.qkv = view(store.wname(a + "q_proj"), 3 * H, w.tr_qkv)
            g.o = view(store.wname(a + "o_proj"), None, w.tr_o)
            g.gu = view(store.wname(m + "gate_proj"), 2 * cfg.inner, w.tr_gu)
            g.down = view(store.wname(m + "down_proj"), None, w.tr_down)
            g.ln1 = view(f"{p}.layers.{l}.input_layernorm.weight", None, w.tr_ln1)
            g.ln2 = view(f"{p}.layers.{l}.post_attention_layernorm.weight", None, w.tr_ln2)
            g.lora = {}
            for key, lw in w.lora.items():
                ga = view(lw.a_name, None, store.trainable(lw.a_name))
                gb = view(lw.b_name, None, store.trainable(lw.b_name))
                g.lora[key] = (ga, gb)
            self.layers.append(g)
        self.norm = view(f"{p}.norm.weight", None, eng.tr_norm)
        self.embed = view(f"{p}.embed_tokens.weight", None, eng.tr_embed)

    def named(self, names):
        """name -> gradient view (None for parameters without a gradient), for handing gradients back to autograd."""
        return [self._view(n, None, self.store.trainable(n)) for n in names]


class StackEngine:
    """One Llama stack (outer `net`: causal over events; inner `net_token`: causal over <= 8 tokens per event)."""

    def __init__(self, store: ParamStore, cfg: StackCfg, tiny_attention: bool, lora_sites=None):
        self.cfg = cfg
        self.store = store
        self.tiny = tiny_attention
        lora_sites = lora_sites or {}
        p = cfg.prefix
        self.layers: List[LayerW] = []
        self.has_lora = False
        for l in range(cfg.n_layer):
            a = f"{p}.layers.{l}.self_attn."
            m = f"{p}.layers.{l}.mlp."
            w = LayerW()
            qkv_n = [store.wname(a + "q_proj"), store.wname(a + "k_proj"), store.wname(a + "v_proj")]
            gu_n = [store.wname(m + "gate_proj"), store.wname(m + "up_proj")]
            o_n, down_n = store.wname(a + "o_proj"), store.wname(m + "down_proj")
            ln1_n, ln2_n = f"{p}.layers.{l}.input_layernorm.weight", f"{p}.layers.{l}.post_attention_layernorm.weight"
            w.qkv = store.fused(qkv_n)
            w.gu = store.fused(gu_n)
            w.o = store.views[o_n]
            w.down = store.views[down_n]
            w.ln1 = store.views[ln1_n]
            w.ln2 = store.views[ln2_n]
            # a fused weight gets its gradient GEMM when any of its parts is trainable (frozen parts are never published)
            w.tr_qkv = any(store.trainable(n) for n in qkv_n)
            w.tr_gu = any(store.trainable(n) for n in gu_n)
            w.tr_o, w.tr_down = store.trainable(o_n), store.trainable(down_n)
            w.tr_ln1, w.tr_ln2 = store.trainable(ln1_n), store.trainable(ln2_n)
            w.lora = {}
            for key, sub in _LORA_KEYS:
                site = lora_sites.get(f"{p}.layers.{l}.{sub}")
                if site is None:
                    continue
                lw = LoraW()
                lw.A, lw.B = store.views[site.a_name], store.views[site.b_name]
                lw.scale, lw.r, lw.a_name, lw.b_name = site.scale, site.r, site.a_name, site.b_name
                w.lora[key] = lw
                self.has_lora = True
            self.layers.append(w)
        self.norm = store.views[f"{p}.norm.weight"]
        self.embed = store.views[f"{p}.embed_tokens.weight"]
        self.tr_norm = store.trainable(f"{p}.norm.weight")
        self.tr_embed = store.trainable(f"{p}.embed_tokens.weight")
        self.names = [n for n in store.names if n.startswith(p + ".")]
        base_names = [n for n in self.names if ".lora_" not in n]
        lora_names = [n for n in self.names if ".lora_" in n]
        self.seg_start = store.offsets[base_names[0]]
        self.seg_end = store._end(base_names[-1])
        self.lora_start = store.offsets[lora_names[0]] if lora_names else 0
        self.lora_end = store._end(lora_names[-1]) if lora_names else 0
        self.base_trainable = any(store.trainable(n) for n in base_names)
        self.lora_trainable = any(store.trainable(n) for n in lora_names)
        self.any_trainable = self.base_trainable or self.lora_trainable
        self.main_grads = StackGrads(self, [(store.gflat, 0, store.numel)])
        if tiny_attention and cfg.head_dim != 256:
            raise lib.B200Error(f"inner stack head_dim {cfg.head_dim} unsupported (kernels are built for 256)")
        if not tiny_attention and cfg.head_dim != 64:
            raise lib.B200Error(f"outer stack head_dim {cfg.head_dim} unsupported (kernels are built for 64)")

    def fresh_grads(self) -> StackGrads:
        """Private gradient buffers for this stack (autograd mode hands these tensors to torch): one over the base
        parameters when any of them trains, one over the stack's LoRA matrices when it has trainable adapters."""
        dev = self.store.device
        spans = []
        if self.base_trainable:
            spans.append((torch.empty(self.seg_end - self.seg_start, dtype=BF16, device=dev), self.seg_start, self.seg_end))
        if self.lora_trainable:
            spans.append((torch.empty(self.lora_end - self.lora_start, dtype=BF16, device=dev), self.lora_start, self.lora_end))
        return StackGrads(self, spans)

    # ------------------------------------------------------------------ LoRA (train.py:439-449; peft lora/layer.py)
    @staticmethod
    def _lora_fwd(lw: LoraW, x: torch.Tensor, y: torch.Tensor, col0: int, out_f: int) -> torch.Tensor:
        """y[:, col0:col0+out_f] += (scale * (x A^T)) B^T, in place through the GEMM's residual epilogue; returns the
        scaled down-projection ts = scale * x A^T  [rows, r] (saved: it is the B-gradient's operand)."""
        rows = x.shape[0]
        t = ops.linear(x, lw.A)
        ts = ops.scale(t, lw.scale)
        yv = y[:, col0:col0 + out_f]
        ops.gemm(ts, lw.B, rows, out_f, lw.r, lda=ts.stride(0), ldb=lw.B.stride(0), out=yv, ldc=y.stride(0), residual=yv)
        return ts

    @staticmethod
    def _lora_bwd(lw: LoraW, g, dy: torch.Tensor, col0: int, out_f: int, x: torch.Tensor, ts: torch.Tensor,
                  dx: torch.Tensor, accumulate: bool) -> None:
        """Backward of _lora_fwd for upstream gradient dy[:, col0:col0+out_f]:  dB (+)= dy^T ts,  dt = scale * dy B,
        dA (+)= dt^T x,  dx += dt A  (dx already holds dy W from the base projection's dgrad)."""
        rows, in_f = x.shape
        r = lw.r
        dyv = dy[:, col0:col0 + out_f]
        ga, gb = g
        if gb is not None:
            ops.gemm(dyv, ts, out_f, r, rows, lda=dy.stride(0), ldb=ts.stride(0), a_mn=True, b_mn=True, out=gb, ldc=r,
                     accumulate=accumulate, allow_split=True)
        dts = ops.gemm(dyv, lw.B, rows, r, out_f, lda=dy.stride(0), ldb=lw.B.stride(0), b_mn=True)
        dt = ops.scale(dts, lw.scale)
        if ga is not None:
            ops.gemm(dt, x, r, in_f, rows, lda=dt.stride(0), ldb=x.stride(0), a_mn=True, b_mn=True, out=ga, ldc=in_f,
                     accumulate=accumulate, allow_split=True)
        ops.gemm(dt, lw.A, rows, in_f, r, lda=dt.stride(0), ldb=lw.A.stride(0), b_mn=True, out=dx, ldc=dx.stride(0),
                 residual=dx)

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor, n_seq: int, S: int, inv_freq: torch.Tensor, save: bool):
        """x: [n_seq * S, H] inputs_embeds (row-major, sequences contiguous) -> (final-normed hidden, saved)."""
        c = self.cfg
        H, D, nh, I = c.hidden, c.head_dim, c.n_head, c.inner
        cos, sin = ops.rope_table(inv_freq, S)
        saved = [] if save else None
        # Residual adds are fused into the norm that follows them (x + y is formed, rounded to bf16 and written by
        # the norm kernel), so every GEMM keeps the plain store epilogue.
        pending = None                                   # output of the previous layer's down_proj, not yet added
        for w in self.layers:
            lo = w.lora
            lsv = {}                                     # projection key -> scaled LoRA down-projection (backward operand)
            if pending is None:
                n1, rstd1 = ops.rmsnorm(x, w.ln1, c.eps, want_rstd=True)
            else:
                x, n1, rstd1 = ops.add_rmsnorm(x, pending, w.ln1, c.eps)
            fuse_tiny = self.tiny and FUSE_ROPE and not FUSE_ROPE_FWD     # token-level stack: RoPE inside the attention kernel
            qkv_lora = any(k in lo for k in ("q", "k", "v"))
            if FUSE_ROPE_FWD and not qkv_lora:
                qkv = ops.linear_rope(n1, w.qkv, cos, sin, S, D)      # QKV GEMM with RoPE in the epilogue
            else:
                qkv = ops.linear(n1, w.qkv)
                for j, key in enumerate(("q", "k", "v")):              # adapters add to the projections BEFORE the rotation
                    if key in lo:
                        lsv[key] = self._lora_fwd(lo[key], n1, qkv, j * H, H)
                if not fuse_tiny:
                    ops.rope_qk_(qkv, cos, sin, S, H, D)
            if self.tiny:
                attn, lse = ops.attn_tiny_fwd(qkv, n_seq, S, nh, D, rope=(cos, sin) if fuse_tiny else None), None
            else:
                attn, lse = ops.attn_causal_fwd(qkv, n_seq, S, nh, D, want_lse=save)
            y1 = ops.linear(attn, w.o)
            if "o" in lo:
                lsv["o"] = self._lora_fwd(lo["o"], attn, y1, 0, H)
            h, n2, rstd2 = ops.add_rmsnorm(x, y1, w.ln2, c.eps)
            del y1
            if FUSE_SWIGLU and I % 128 == 0 and "gate" not in lo and "up" not in lo:
                gu, act = ops.linear_swiglu(n2, w.gu)
            else:
                gu = ops.linear(n2, w.gu)
                if "gate" in lo:
                    lsv["gate"] = self._lora_fwd(lo["gate"], n2, gu, 0, I)
                if "up" in lo:
                    lsv["up"] = self._lora_fwd(lo["up"], n2, gu, I, I)
                act = ops.swiglu(gu)
            pending = ops.linear(act, w.down)
            if "down" in lo:
                lsv["down"] = self._lora_fwd(lo["down"], act, pending, 0, H)
            if save:
                saved.append((x, n1, rstd1, qkv, attn, lse, h, n2, rstd2, gu, act, lsv))
            x = h
        x, y, rstd_f = ops.add_rmsnorm(x, pending, self.norm, c.eps)
        sv = dict(layers=saved, x_last=x, rstd_f=rstd_f, n_seq=n_seq, S=S, cos=cos, sin=sin) if save else None
        return y, sv

    # ------------------------------------------------------------------ backward
    def layer_range(self, li: int):
        """[start, end) of layer `li`'s base parameters inside the flat parameter / gradient buffers."""
        p = self.cfg.prefix
        first = self.store.offsets[self.store.wname(f"{p}.layers.{li}.self_attn.q_proj")]
        if li + 1 < self.cfg.n_layer:
            end = self.store.offsets[self.store.wname(f"{p}.layers.{li + 1}.self_attn.q_proj")]
        else:
            end = self.store.offsets[f"{p}.norm.weight"]
        return first, end

    def backward(self, sv: dict, dy: torch.Tensor, grads: StackGrads, accumulate: bool = False,
                 layer_done=None) -> torch.Tensor:
        """dy: grad of the final-normed output.  Writes (or accumulates) the gradient of every trainable weight of the
        stack into `grads` (a frozen weight -- view None -- costs no gradient GEMM: the base of a LoRA run) and returns the
        gradient w.r.t. the stack input (inputs_embeds)."""
        c = self.cfg
        H, D, nh, I = c.hidden, c.head_dim, c.n_head, c.inner
        if sv is None or sv["layers"] is None:
            raise lib.B200Error("backward called without a saved forward")
        n_seq, S, cos, sin = sv["n_seq"], sv["S"], sv["cos"], sv["sin"]
        side = _side_stream(dy.device) if WGRAD_STREAM else None
        pending = []          # (event on the side stream, operands of the wgrads issued before it), released one layer late
        dx = ops.rmsnorm_bwd(dy, sv["x_last"], self.norm, sv["rstd_f"], None, grads.norm, accumulate)
        for li in range(len(self.layers) - 1, -1, -1):
            w = self.layers[li]
            g = grads.layers[li]
            lo = w.lora
            hold = []
            x, n1, rstd1, qkv, attn, lse, h, n2, rstd2, gu, act, lsv = sv["layers"][li]
            sv["layers"][li] = None   # free as we go
            # ---- MLP block: x_out = h + down(act)
            dact = ops.linear_dgrad(dx, w.down)
            if g.down is not None:
                _wgrad(dx, act, g.down, accumulate, side, hold)
            if "down" in lo:
                self._lora_bwd(lo["down"], g.lora["down"], dx, 0, H, act, lsv["down"], dact, accumulate)
            del act
            dgu = ops.swiglu_bwd(gu, dact)
            del dact, gu
            dn2 = ops.linear_dgrad(dgu, w.gu)
            if g.gu is not None:
                _wgrad(dgu, n2, g.gu, accumulate, side, hold)
            if "gate" in lo:
                self._lora_bwd(lo["gate"], g.lora["gate"], dgu, 0, I, n2, lsv["gate"], dn2, accumulate)
            if "up" in lo:
                self._lora_bwd(lo["up"], g.lora["up"], dgu, I, I, n2, lsv["up"], dn2, accumulate)
            del dgu, n2
            dh = ops.rmsnorm_bwd(dn2, h, w.ln2, rstd2, dx, g.ln2, accumulate)
            del dn2, h, dx
            # ---- attention block: h = x + o(attn)
            dattn = ops.linear_dgrad(dh, w.o)
            if g.o is not None:
                _wgrad(dh, attn, g.o, accumulate, side, hold)
            if "o" in lo:
                self._lora_bwd(lo["o"], g.lora["o"], dh, 0, H, attn, lsv["o"], dattn, accumulate)
            rope = (cos, sin) if FUSE_ROPE else None
            if self.tiny:
                dqkv = ops.attn_tiny_bwd(qkv, dattn, n_seq, S, nh, D, rope=rope)
            else:
                dqkv = ops.attn_causal_bwd(qkv, attn, dattn, lse, n_seq, S, nh, D, rope=rope)
            del dattn, attn, qkv
            if not FUSE_ROPE:
                ops.rope_qk_(dqkv, cos, sin, S, H, D, backward=True)
            dn1 = ops.linear_dgrad(dqkv, w.qkv)
            if g.qkv is not None:
                _wgrad(dqkv, n1, g.qkv, accumulate, side, hold)
            for j, key in enumerate(("q", "k", "v")):
                if key in lo:
                    self._lora_bwd(lo[key], g.lora[key], dqkv, j * H, H, n1, lsv[key], dn1, accumulate)
            del dqkv, n1, lsv
            dx = ops.rmsnorm_bwd(dn1, x, w.ln1, rstd1, dh, g.ln1, accumulate)
            del dn1, dh, x
            if side is not None:
                ev = torch.cuda.Event()
                ev.record(side)
                pending.append((ev, hold))
                if len(pending) > 1:          # the previous layer's wgrads have long finished: no stall, memory bounded
                    old_ev, old_hold = pending.pop(0)
                    torch.cuda.current_stream().wait_event(old_ev)
                    old_hold.clear()
            if layer_done is not None:
                if side is not None:
                    torch.cuda.current_stream().wait_stream(side)     # this layer's weight gradients are complete
                layer_done(li)
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)
            pending.clear()
        sv["layers"] = None
        return dx


class MergedStack:
    """Inference view of a stack whose LoRA adapters are folded into private copies of the adapted weights:
    W' = W + scale * B A, one rounding per element (what `merge_and_unload` / load_merge_lora compute, midi_model.py:109-114).
    Quacks like StackEngine for midi_b200.decode (cfg, layers[i].{ln1,qkv,o,ln2,gu,down}, norm, embed), so `generate`
    works on a model with injected adapters -- train.py:216-233 samples examples from the LoRA model while it trains."""

    def __init__(self, eng: StackEngine):
        self.cfg, self.norm, self.embed = eng.cfg, eng.norm, eng.embed
        self.store = eng.store
        H, I = eng.cfg.hidden, eng.cfg.inner
        self.layers = []
        for w in eng.layers:
            m = LayerW()
            for f in ("qkv", "o", "gu", "down", "ln1", "ln2"):
                setattr(m, f, getattr(w, f))
            m.lora = {}
            lo = w.lora
            if any(k in lo for k in ("q", "k", "v")):
                m.qkv = w.qkv.clone()
                for j, key in enumerate(("q", "k", "v")):
                    if key in lo:
                        self._fold(lo[key], m.qkv[j * H:(j + 1) * H])
            if "o" in lo:
                m.o = w.o.clone()
                self._fold(lo["o"], m.o)
            if "gate" in lo or "up" in lo:
                m.gu = w.gu.clone()
                if "gate" in lo:
                    self._fold(lo["gate"], m.gu[:I])
                if "up" in lo:
                    self._fold(lo["up"], m.gu[I:])
            if "down" in lo:
                m.down = w.down.clone()
                self._fold(lo["down"], m.down)
            self.layers.append(m)

    @staticmethod
    def _fold(lw: LoraW, W: torch.Tensor) -> None:
        """W[out, in] += (scale * B)[out, r] . A[r, in]  (A as stored = the GEMM's MN-major B operand)."""
        out_f, in_f = W.shape
        sB = ops.scale(lw.B, lw.scale)
        ops.gemm(sB, lw.A, out_f, in_f, lw.r, lda=sB.stride(0), ldb=lw.A.stride(0), b_mn=True, out=W, ldc=W.stride(0),
                 residual=W)
