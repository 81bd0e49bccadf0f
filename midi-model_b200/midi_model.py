"""Drop-in `midi_model` module: CUDA-native MIDIModel (H100, sm_90a).

Place this directory ahead of the reference checkout on `sys.path`; `train.py` / `app.py` then do
`from midi_model import MIDIModel, MIDIModelConfig, config_name_list` and get this implementation
(reference: `midi_model.py:14-250`).  What is kept verbatim is the *contract*: constructor, module
tree and `state_dict` keys (`net.*`, `net_token.*`, `lm_head.weight` -- the HF `LlamaModel`s are used
as parameter containers only, so seeded init, the four dtype-following RoPE `inv_freq` buffers and
peft/LoRA affordances behave exactly like the reference), and the signatures / semantics of
`forward`, `forward_token`, `sample_top_p_k`, `generate`.  What is new is everything that computes:
all arithmetic runs in hand-written sm_90a kernels behind the C ABI in `include/midi_b200.h`
(`midi_b200/lib.py`).  There is no PyTorch / CPU fallback: parameters must be bfloat16 on a CUDA
device, otherwise the call raises.

LoRA (`train.py --task lora`, train.py:439-449): `add_adapter` injects adapters in peft's layout (transformers' mixin when
peft is installed, midi_b200/lora.py otherwise); the engine then computes y = W x + (lora_alpha / r) B A x, trains A and B
only, and `generate` reads merged copies.

Extra (non-reference) entry points used by the fused trainer and the benchmark: `training_loss(batch)`,
`fused_optimizer_step(...)`, `optimizer_state_dict()` / `load_optimizer_state_dict()`, `generate_stream(...)`
(app.py:27-120), `load_adapter_weights(dir)`.
"""
from __future__ import annotations

import json
import math
import os
import threading
from typing import Any, Dict, Optional, Union

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
import tqdm
from transformers import DynamicCache, LlamaConfig, LlamaModel, PretrainedConfig, PreTrainedModel

from midi_b200 import decode as _dec
from midi_b200 import engine as _engine
from midi_b200 import lib as _lib
from midi_b200 import lora as _lora
from midi_b200 import ops as _ops
from midi_b200.engine import MergedStack, ParamStore, StackCfg, StackEngine
from midi_b200.tokenizer_tables import make_tokenizer

config_name_list = ["tv1-medium", "tv2-medium", "tv2o-medium", "tv2-large", "tv2o-large"]

_SIZES = {"medium": dict(n_layer=12, n_head=16, n_embd=1024, n_inner=4096),
          "large": dict(n_layer=24, n_head=16, n_embd=1024, n_inner=4096)}


class MIDIModelConfig(PretrainedConfig):
    """Same public surface as the reference config (midi_model.py:17-96)."""
    model_type = "midi_model"

    def __init__(self, tokenizer=None, net_config: Union[LlamaConfig, Dict, None] = None,
                 net_token_config: Union[LlamaConfig, Dict, None] = None, **kwargs):
        super().__init__(**kwargs)
        if isinstance(tokenizer, dict):
            tok = make_tokenizer(tokenizer["version"])
            tok.set_optimise_midi(tokenizer["optimise_midi"])
            tokenizer = tok
        self.tokenizer = tokenizer if tokenizer else make_tokenizer()

        def as_llama(c):
            if isinstance(c, dict):
                return LlamaConfig(**c)
            return c if c else LlamaConfig()

        self.net_config = as_llama(net_config)
        self.net_token_config = as_llama(net_token_config)
        self.n_embd = self.net_token_config.hidden_size   # midi_model.py:48

    def to_dict(self) -> Dict[str, Any]:
        d = super().to_dict()
        d["tokenizer"] = self.tokenizer.to_dict()
        return d

    def __str__(self):
        return json.dumps({"net": self.net_config.to_json_string(use_diff=False),
                           "net_token": self.net_token_config.to_json_string(use_diff=False)}, indent=4)

    @staticmethod
    def get_config(tokenizer_ver="v2", optimise_midi=True, n_layer=12, n_head=16, n_embd=1024, n_inner=4096):
        tok = make_tokenizer(tokenizer_ver)
        tok.set_optimise_midi(optimise_midi)
        common = dict(vocab_size=tok.vocab_size, hidden_size=n_embd, pad_token_id=tok.pad_id,
                      max_position_embeddings=4096, use_cache=False)
        outer = LlamaConfig(num_attention_heads=n_head, num_hidden_layers=n_layer, intermediate_size=n_inner, **common)
        # the token-level stack is a quarter of the event-level one in heads, depth and MLP width (midi_model.py:71-75)
        inner = LlamaConfig(num_attention_heads=n_head // 4, num_hidden_layers=n_layer // 4,
                            intermediate_size=n_inner // 4, **common)
        return MIDIModelConfig(tok, outer, inner)

    @staticmethod
    def from_name(name="tv2o-medium"):
        tv, size = name.split("-")
        tv = tv[1:]
        optimise = tv.endswith("o")
        if optimise:
            tv = tv[:-1]
        if tv not in ("v1", "v2"):
            raise ValueError(f"Unknown tokenizer version {tv}")
        if size not in _SIZES:
            raise ValueError(f"Unknown model size {size}")
        return MIDIModelConfig.get_config(tokenizer_ver=tv, optimise_midi=optimise, **_SIZES[size])


# ---------------------------------------------------------------------------------------------
# runtime: flat parameter store + the two stack engines, (re)built lazily
# ---------------------------------------------------------------------------------------------
class _Runtime:
    def __init__(self, model: "MIDIModel"):
        # LoRA adapters injected by peft or by MIDIModel.add_adapter (train.py:439-449): projection path -> A, B, scaling
        self.lora_sites = _lora.find_sites(model)
        for path in self.lora_sites:
            if not (path.startswith("net.layers.") or path.startswith("net_token.layers.")):
                raise _lib.B200Error(f"LoRA on {path} is not supported (adapters go on the decoder layers' projections)")
        self.store = ParamStore(model)
        nc, tc = model.config.net_config, model.config.net_token_config
        self.outer = StackEngine(self.store, StackCfg("net", nc.num_hidden_layers, nc.num_attention_heads, nc.hidden_size,
                                                      nc.intermediate_size, nc.rms_norm_eps), tiny_attention=False,
                                 lora_sites=self.lora_sites)
        self.inner = StackEngine(self.store, StackCfg("net_token", tc.num_hidden_layers, tc.num_attention_heads,
                                                      tc.hidden_size, tc.intermediate_size, tc.rms_norm_eps),
                                 tiny_attention=True, lora_sites=self.lora_sites)
        self.has_lora = self.outer.has_lora or self.inner.has_lora
        self.peft_flag = bool(getattr(model, "_hf_peft_config_loaded", False))
        self.lora_params = [p for n, p in model.named_parameters() if ".lora_" in n]
        self.lora_step = 0                      # bumped by the fused optimizer (raw-pointer updates have no _version)
        self.merged_version = None              # adapter version the merged decode weights were folded at
        self.lm_head = self.store.views["lm_head.weight"]
        self.tr_lm_head = self.store.trainable("lm_head.weight")
        self.g_lm_head = self.store.gviews["lm_head.weight"] if self.tr_lm_head else None
        self.V = self.lm_head.shape[0]
        self.pitch = (self.V + 7) // 8 * 8
        self.H = nc.hidden_size
        self.cached_outer = None
        self.cached_inner = None
        self.grammar = None
        # Device-resident generate loops (decode.GraphGenerator: KV pools, CUDA graph, RNG / position state, own stream).
        # gradio serves app.generate from up to 10 worker threads sharing one model (app.py:496) and may resume a
        # suspended generator from another thread, so no thread-owned lock is ever held across a `yield`: a generation
        # CHECKS OUT a generator (creating one when none is idle), owns it exclusively until it finishes or is closed,
        # then returns it.  `pool_lock` only guards the free list.
        self.gen_pool = {}                      # key -> [idle GraphGenerator]
        self.pool_lock = threading.Lock()

    def lora_version(self):
        """Changes whenever an adapter matrix was updated (torch optimizers bump _version; the fused AdamW bumps lora_step)."""
        return (self.lora_step, sum(p._version for p in self.lora_params))


def _flat_ids(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.long).contiguous()


class _OuterFn(torch.autograd.Function):
    """forward(): embed-sum + event-level stack, as one autograd node (parameters are inputs so that
    torch's AccumulateGrad / DDP hooks see their gradients)."""

    @staticmethod
    def forward(ctx, model, x_ids, *params):
        rt = model._rt()
        B, S, T = x_ids.shape
        ids = _flat_ids(x_ids).view(B * S, T)
        need = any(ctx.needs_input_grad)   # (grad mode is off inside Function.forward; this is the reliable signal)
        e = _ops.embed_sum(ids, rt.outer.embed)
        y, sv = rt.outer.forward(e, B, S, model.net.rotary_emb.inv_freq, save=need)
        ctx.model, ctx.sv, ctx.ids, ctx.shape = model, sv, ids, (B, S, T)
        return y.view(B, S, -1)

    @staticmethod
    def backward(ctx, dy):
        model = ctx.model
        rt = model._rt()
        B, S, T = ctx.shape
        g = rt.outer.fresh_grads()
        dy2 = dy.reshape(B * S, -1).to(torch.bfloat16).contiguous()
        de = rt.outer.backward(ctx.sv, dy2, g, accumulate=False)
        if g.embed is not None:
            _ops.embed_bwd(ctx.ids.view(-1), de, g.embed, per_row=T, row_stride=1, row_inner=0, row_off=0,
                           pad_id=model.config.net_config.pad_token_id, accumulate=False)
        ctx.sv = None
        return (None, None, *g.named(rt.outer.names))


class _InnerFn(torch.autograd.Function):
    """forward_token() without cache: [hidden, embed(x)] -> token-level stack -> lm_head logits."""

    @staticmethod
    def forward(ctx, model, hidden, x_ids, *params):
        rt = model._rt()
        N = hidden.shape[0] if hidden is not None else x_ids.shape[0]
        ids = _flat_ids(x_ids) if x_ids is not None else None
        n_ids = 0 if ids is None else ids.shape[1]
        L = n_ids + (1 if hidden is not None else 0)
        need = any(ctx.needs_input_grad)
        hid = hidden.to(torch.bfloat16).contiguous() if hidden is not None else None
        xin = _ops.inner_input(hid, ids, rt.inner.embed)
        hs, sv = rt.inner.forward(xin, N, L, model.net_token.rotary_emb.inv_freq, save=need)
        logits = _ops.linear(hs, rt.lm_head, pitch=rt.pitch)          # [N*L, pitch]
        ctx.model, ctx.sv, ctx.ids, ctx.hs = model, sv, ids, (hs if need else None)
        ctx.dims = (N, L, n_ids, hidden is not None)
        return logits.view(N, L, rt.pitch)[:, :, :rt.V]

    @staticmethod
    def backward(ctx, dlogits):
        model = ctx.model
        rt = model._rt()
        N, L, n_ids, has_hidden = ctx.dims
        dl = _as_pitched(dlogits, N * L, rt.pitch)
        if dl is None:
            # caller gradients arrive dense [N, L, V]; the kernels want 16-byte row pitch
            dl = torch.zeros((N * L, rt.pitch), dtype=torch.bfloat16, device=dlogits.device)
            dl[:, :rt.V] = dlogits.reshape(N * L, rt.V)
        g = rt.inner.fresh_grads()
        g_head = torch.empty_like(rt.lm_head) if rt.tr_lm_head else None
        dhidden, = _inner_backward(rt, model, ctx.sv, ctx.hs, dl, ctx.ids, N, L, n_ids, has_hidden, g, g_head, False)
        ctx.sv = ctx.hs = None
        return (None, dhidden, None, *g.named(rt.inner.names), g_head)


def _as_pitched(t: torch.Tensor, rows: int, pitch: int):
    """`t` = [..., V] view (V <= pitch) of a [rows, pitch] bf16 buffer starting at its storage base -> that buffer
    (no copy), else None.  This is how the fused cross entropy hands its in-place gradient back to _InnerFn.backward."""
    if t.dtype != torch.bfloat16 or t.dim() < 2 or t.stride(-1) != 1 or t.stride(-2) != pitch or t.storage_offset() != 0:
        return None
    if t.numel() // t.shape[-1] != rows or t.untyped_storage().nbytes() < rows * pitch * 2 or t.data_ptr() % 16:
        return None
    want = pitch
    for d in range(t.dim() - 2, -1, -1):                     # leading dims must be a plain row enumeration
        if t.shape[d] != 1 and t.stride(d) != want:
            return None
        want *= t.shape[d]
    return torch.as_strided(t.detach(), (rows, pitch), (pitch, 1))


LAZY_CE = os.environ.get("B200_LAZY_CE", "1") != "0"
LAZY_CE_HITS = 0          # how many F.cross_entropy calls were served by the fused kernels (tests read this)


class _LazyCEFn(torch.autograd.Function):
    """F.cross_entropy(logits.view(-1, V), y, reduction="mean", ignore_index=pad) (train.py:180-185) on the pitched logits
    buffer forward_token produced: one read for the loss; the backward overwrites the logits with dlogits in place and
    returns a view of that same buffer, which _InnerFn.backward recognises (no dense [N*L, V] copies in either direction)."""

    @staticmethod
    def forward(ctx, logits2d, buf, targets, V, ignore_index):
        lac, lse = _ops.ce_fwd(buf, targets, V, ignore_index)
        ctx.save_for_backward(buf, targets, lse, lac)
        ctx.V, ctx.ignore = V, ignore_index
        return lac[0].to(logits2d.dtype)

    @staticmethod
    def backward(ctx, dloss):
        buf, targets, lse, lac = ctx.saved_tensors
        # the logits buffer now holds dlogits (in place, through a raw pointer): bump its version counter so that autograd
        # raises if anything else saved these logits for a later backward, instead of silently reading gradients
        _ops.ce_bwd_(buf, targets, lse, lac, ctx.V, ctx.ignore, grad_scale=1.0, grad_scale_dev=dloss)
        torch.autograd.graph.increment_version(buf)
        return buf[:, :ctx.V], None, None, None, None


class LazyLogits(torch.Tensor):
    """What forward_token returns in training: an ordinary dense [N, L, V] logits tensor (every op works on it as before)
    that remembers the pitched buffer behind it, so that the reference's loss expression is served by the fused
    cross-entropy kernels instead of materialising log-softmax and dlogits copies of the 0.9 GB logits."""

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is F.cross_entropy and LAZY_CE:
            out = cls._fused_ce(*args, **kwargs)
            if out is not None:
                return out
        ret = super().__torch_function__(func, types, args, kwargs)
        if func in (torch.Tensor.view, torch.Tensor.reshape, torch.reshape) and isinstance(ret, LazyLogits):
            src = args[0]
            h = getattr(src, "_b200_lazy", None)
            if h is not None and ret.dim() >= 1 and ret.shape[-1] == h[1] and ret.numel() == src.numel():
                ret._b200_lazy = h                      # still the same rows in the same order
        return ret

    @staticmethod
    def _fused_ce(input, target, weight=None, size_average=None, ignore_index=-100, reduce=None, reduction="mean",
                  label_smoothing=0.0):
        h = getattr(input, "_b200_lazy", None)
        if (h is None or weight is not None or reduction != "mean" or label_smoothing != 0.0 or size_average is not None
                or reduce is not None or input.dim() != 2 or not isinstance(target, torch.Tensor) or target.dim() != 1
                or target.dtype != torch.long or target.shape[0] != input.shape[0] or not input.requires_grad):
            return None
        buf, V = h
        if input.shape != (buf.shape[0], V) or _as_pitched(input, buf.shape[0], buf.shape[1]) is None:
            return None
        global LAZY_CE_HITS
        LAZY_CE_HITS += 1
        with torch._C.DisableTorchFunctionSubclass():
            return _LazyCEFn.apply(input, buf, target.contiguous(), V, int(ignore_index))


def _inner_backward(rt, model, sv, hs, dlogits, ids, N, L, n_ids, has_hidden, g, g_head, accumulate):
    """dlogits [N*L, pitch] -> grads of lm_head, the token-level stack, its embedding; returns (dhidden,)."""
    # lm_head weight gradient on the engine's side stream (joined at the end of rt.inner.backward)
    side = _engine._side_stream(dlogits.device) if _engine.WGRAD_STREAM else None
    if g_head is not None:                       # None: lm_head is frozen (LoRA run, train.py:440)
        _engine._wgrad(dlogits, hs, g_head, accumulate, side)
    dhs = _ops.linear_dgrad(dlogits, rt.lm_head)
    dx = rt.inner.backward(sv, dhs, g, accumulate=accumulate)
    if g.embed is None:
        pass
    elif n_ids > 0:
        _ops.embed_bwd(ids.view(-1), dx, g.embed, per_row=n_ids, row_stride=L, row_inner=1, row_off=1 if has_hidden else 0,
                       pad_id=model.config.net_token_config.pad_token_id, accumulate=accumulate)
    else:
        if not accumulate:
            g.embed.zero_()
    dhidden = None
    if has_hidden:
        dhidden = torch.empty((N, rt.H), dtype=torch.bfloat16, device=dx.device)
        _lib.call("b200_inner_input_bwd_hidden", dx.data_ptr(), dhidden.data_ptr(), N, L, rt.H, _lib.stream())
    return (dhidden,)


def _loop_mode(mode: str):
    """B200_GENERATE: "persist" (default: one persistent cooperative kernel per block of events), "graph" (one CUDA-graph
    replay per event), "nograph" (the graph's launches issued from the host), "eager" (host-driven reference-shaped loop)."""
    if mode == "persist":
        return "persist"
    return mode not in ("nograph", "eager")


class _KVState:
    """Paged KV cache hung off the caller's (opaque) DynamicCache object."""

    def __init__(self, kv):
        self.kv = kv


class MIDIModel(PreTrainedModel):
    config_class = MIDIModelConfig

    def __init__(self, config: MIDIModelConfig, *args, **kwargs):
        super(MIDIModel, self).__init__(config, *args, **kwargs)
        self.tokenizer = config.tokenizer
        # HF modules are parameter containers (same construction order as midi_model.py:105-107 => same seeded init)
        self.net = LlamaModel(config.net_config)
        self.net_token = LlamaModel(config.net_token_config)
        self.lm_head = nn.Linear(config.n_embd, self.tokenizer.vocab_size, bias=False)
        self._b200_rt: Optional[_Runtime] = None

    # ------------------------------------------------------------------ plumbing
    def _rt(self) -> _Runtime:
        rt = self.__dict__.get("_b200_rt")
        if rt is None or not rt.store.valid() or rt.peft_flag != bool(getattr(self, "_hf_peft_config_loaded", False)):
            _lib.load()
            rt = _Runtime(self)
            self.__dict__["_b200_rt"] = rt
        return rt

    # ------------------------------------------------------------------ LoRA (train.py:439-449, 234-244, 263-264)
    def add_adapter(self, adapter_config, adapter_name: Optional[str] = None):
        """`model.add_adapter(LoraConfig(...))` as train.py:449 calls it.  With peft installed this is transformers' own
        PeftAdapterMixin.add_adapter; without it the adapter modules are created natively in peft's layout
        (midi_b200/lora.py): either way the engine finds `<proj>.lora_A/.lora_B.<adapter>.weight` next to
        `<proj>.base_layer.weight`, computes y = W x + (lora_alpha / r) B A x in both stacks and trains A, B only."""
        try:
            import peft  # noqa: F401
            have_peft = True
        except ImportError:
            have_peft = False
        if have_peft:
            out = super().add_adapter(adapter_config, adapter_name)
            self.__dict__["_b200_rt"] = None
            return out
        adapter_name = adapter_name or "default"
        cfg = _lora.LoraAdapterConfig.from_any(adapter_config)
        if not self._hf_peft_config_loaded:
            self._hf_peft_config_loaded = True
            self.peft_config = {}
        elif adapter_name in self.peft_config:
            raise ValueError(f"Adapter with name {adapter_name} already exists. Please use a different name.")
        _lora.inject(self, cfg, adapter_name)
        self.peft_config[adapter_name] = cfg
        self.__dict__["_b200_native_lora"] = adapter_name
        self.__dict__["_b200_rt"] = None

    def active_adapters(self):
        if self.__dict__.get("_b200_native_lora") is not None:
            return [self.__dict__["_b200_native_lora"]]
        return super().active_adapters()

    def get_adapter_state_dict(self, adapter_name: Optional[str] = None, *args, **kwargs):
        if self.__dict__.get("_b200_native_lora") is not None:
            return _lora.adapter_state_dict(self, adapter_name or self.active_adapters()[0])
        return super().get_adapter_state_dict(adapter_name, *args, **kwargs)

    def load_adapter_weights(self, adapter_dir_or_state_dict, adapter_name: Optional[str] = None) -> None:
        """Resume LoRA training: load `adapter_model.safetensors` (train.py:241-244) / a state dict into the injected
        adapter WITHOUT merging (load_merge_lora is the inference-side merge)."""
        sd = adapter_dir_or_state_dict
        if not isinstance(sd, dict):
            from safetensors.torch import load_file
            sd = load_file(os.path.join(sd, "adapter_model.safetensors"))
        _lora.load_adapter_state_dict(self, sd, adapter_name or self.active_adapters()[0])
        rt = self.__dict__.get("_b200_rt")
        if rt is not None:
            rt.lora_step += 1

    def load_merge_lora(self, model_id):
        """midi_model.py:109-114: merge a LoRA adapter into the base weights and return the merged model.
        With `peft` installed this is the reference's own sequence; without it (this image) the adapter directory
        (`adapter_config.json` + `adapter_model.safetensors`/`.bin`, as written by train.py:234-244 or by peft) is merged
        natively: W += (B @ A) * scaling, in place on the packed parameter buffer."""
        try:
            from peft import LoraModel, PeftConfig, load_peft_weights, set_peft_model_state_dict
        except ImportError:
            return self._merge_lora_native(model_id)
        peft_config = PeftConfig.from_pretrained(model_id)
        model = LoraModel(self, peft_config, adapter_name="default")
        adapter_state_dict = load_peft_weights(model_id, device=str(self.device))
        set_peft_model_state_dict(self, adapter_state_dict, "default")
        merged = model.merge_and_unload()
        self.__dict__["_b200_rt"] = None
        return merged

    def _merge_lora_native(self, adapter_dir: str):
        """LoRA merge without peft (what LoraModel.merge_and_unload computes for nn.Linear targets): for every target
        module, delta = lora_B @ lora_A scaled by lora_alpha / r (lora_alpha / sqrt(r) with use_rslora; per-module
        rank_pattern / alpha_pattern honoured), accumulated in fp32 and rounded once into the weight's dtype."""
        import json
        import re
        cfg_path = os.path.join(adapter_dir, "adapter_config.json")
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(f"load_merge_lora: {cfg_path} not found (a local adapter directory is required without peft)")
        with open(cfg_path) as f:
            cfg = json.load(f)
        if str(cfg.get("peft_type", "LORA")).upper() != "LORA":
            raise ValueError(f"load_merge_lora: unsupported peft_type {cfg.get('peft_type')}")
        st_path = os.path.join(adapter_dir, "adapter_model.safetensors")
        if os.path.isfile(st_path):
            from safetensors.torch import load_file
            weights = load_file(st_path)
        else:
            weights = torch.load(os.path.join(adapter_dir, "adapter_model.bin"), map_location="cpu", weights_only=True)
        r0, alpha0 = int(cfg["r"]), float(cfg.get("lora_alpha", cfg["r"]))
        rank_pattern, alpha_pattern = cfg.get("rank_pattern") or {}, cfg.get("alpha_pattern") or {}
        rslora, fan_in_fan_out = bool(cfg.get("use_rslora", False)), bool(cfg.get("fan_in_fan_out", False))

        def pattern(table, name, default):
            for k, v in table.items():
                if re.fullmatch(rf"(.*\.)?{k}", name):
                    return v
            return default

        # key = [base_model.model.]<module path>.lora_{A,B}[.<adapter name>].weight
        pairs = {}
        for k, v in weights.items():
            mobj = re.fullmatch(r"(?:base_model\.model\.)?(.+)\.lora_(A|B)(?:\.[^.]+)?\.weight", k)
            if mobj is None:
                if "lora_embedding" in k:
                    raise NotImplementedError("load_merge_lora: LoRA on embeddings is not supported by the native merge")
                continue
            pairs.setdefault(mobj.group(1), {})[mobj.group(2)] = v
        if not pairs:
            raise ValueError("load_merge_lora: no lora_A / lora_B tensors in the adapter")
        modules = dict(self.named_modules())
        with torch.no_grad():
            for name, ab in sorted(pairs.items()):
                if "A" not in ab or "B" not in ab:
                    raise ValueError(f"load_merge_lora: incomplete LoRA pair for {name}")
                mod = modules.get(name)
                if not isinstance(mod, nn.Linear):
                    raise ValueError(f"load_merge_lora: target {name} is not a Linear layer of this model")
                W = mod.weight
                A = ab["A"].to(device=W.device, dtype=torch.float32)       # [r, in]
                Bm = ab["B"].to(device=W.device, dtype=torch.float32)      # [out, r]
                r = int(pattern(rank_pattern, name, r0))
                if A.shape[0] != r or Bm.shape[1] != r:
                    r = A.shape[0]
                alpha = float(pattern(alpha_pattern, name, alpha0))
                scaling = alpha / math.sqrt(r) if rslora else alpha / r
                delta = (Bm @ A) * scaling
                if fan_in_fan_out:
                    delta = delta.t()
                if delta.shape != W.shape:
                    raise ValueError(f"load_merge_lora: {name}: delta {tuple(delta.shape)} vs weight {tuple(W.shape)}")
                W.copy_((W.float() + delta).to(W.dtype))
        self.__dict__["_b200_rt"] = None          # fused views / cached stacks are rebuilt from the merged weights
        return self

    def _kv_for(self, cache, which: str, batch: int):
        rt = self._rt()
        st = getattr(cache, "_b200_" + which, None)
        if st is None or st.kv.batch != batch:
            if which == "outer":
                cfgs, page, cap = rt.outer.cfg, 64, self.config.net_config.max_position_embeddings
            else:
                cfgs, page, cap = rt.inner.cfg, 8, 8
            st = _KVState(_dec.PagedKV(cfgs, batch, cap, page, rt.store.device))
            setattr(cache, "_b200_" + which, st)
        return st.kv

    def _refresh_merged(self, rt) -> None:
        """Inference on a model with injected adapters (train.py:216-233 samples from the LoRA model while it trains): the
        decode kernels read private merged copies W + scale * B A (engine.MergedStack), re-folded whenever an adapter
        changed -- which also retires the idle generate loops built on the old copies."""
        if not rt.has_lora:
            return
        ver = rt.lora_version()
        if rt.merged_version != ver:
            with rt.pool_lock:
                rt.merged_version = ver
                rt.cached_outer = rt.cached_inner = None
                rt.gen_pool.clear()

    def _cached_stack(self, which: str, refresh: bool = True):
        rt = self._rt()
        if refresh:
            self._refresh_merged(rt)
        if which == "outer":
            if rt.cached_outer is None:
                eng = MergedStack(rt.outer) if rt.outer.has_lora else rt.outer
                rt.cached_outer = _dec.CachedStack(eng, self.config.net_config.max_position_embeddings,
                                                   self.net.rotary_emb.inv_freq)
            return rt.cached_outer
        if rt.cached_inner is None:
            eng = MergedStack(rt.inner) if rt.inner.has_lora else rt.inner
            rt.cached_inner = _dec.CachedStack(eng, 8, self.net_token.rotary_emb.inv_freq)
        return rt.cached_inner

    # ------------------------------------------------------------------ reference API
    def forward_token(self, hidden_state=None, x=None, cache=None):
        """
        :param hidden_state: (batch_size, n_embd)
        :param x: (batch_size, token_sequence_length)
        :param cache: Cache
        :return: (batch_size, 1 + token_sequence_length, vocab_size)
        """
        rt = self._rt()
        if cache is None:
            params = [self._b200_param(n) for n in rt.inner.names] + [self.lm_head.weight]
            out = _InnerFn.apply(self, hidden_state, x, *params)
            if LAZY_CE and out.requires_grad:
                buf = _as_pitched(out, out.shape[0] * out.shape[1], rt.pitch)
                if buf is not None:
                    out = out.as_subclass(LazyLogits)
                    out._b200_lazy = (buf, rt.V)
            return out
        # cached (inference) path: midi_model.py:216-221 call modes
        N = hidden_state.shape[0] if hidden_state is not None else x.shape[0]
        kv = self._kv_for(cache, "inner", N)
        ids = _flat_ids(x) if x is not None else None
        hid = hidden_state.to(torch.bfloat16).contiguous() if hidden_state is not None else None
        xin = _ops.inner_input(hid, ids, rt.inner.embed)
        L = xin.shape[0] // N
        hs = self._cached_stack("inner").step(xin, kv, L)
        logits = _dec._lm_head(hs, rt.lm_head, rt.pitch)
        return logits.view(N, L, rt.pitch)[:, :, :rt.V]

    def forward(self, x, cache=None):
        """
        :param x: (batch_size, midi_sequence_length, token_sequence_length)
        :param cache: Cache
        :return: hidden (batch_size, midi_sequence_length, n_embd)
        """
        rt = self._rt()
        _lib.require_cuda(x, "x")
        if cache is None:
            params = [self._b200_param(n) for n in rt.outer.names]
            return _OuterFn.apply(self, x, *params)
        B, S, T = x.shape
        kv = self._kv_for(cache, "outer", B)
        e = _ops.embed_sum(_flat_ids(x).view(B * S, T), rt.outer.embed)
        y = self._cached_stack("outer").step(e, kv, S)
        return y.view(B, S, -1)

    def _b200_param(self, name: str) -> torch.Tensor:
        mod, _, leaf = name.rpartition(".")
        return getattr(self.get_submodule(mod), leaf)

    def sample_top_p_k(self, probs, p, k, generator=None):
        """midi_model.py:152-165 as one kernel.  `probs`: (..., vocab) softmaxed and masked, un-normalised."""
        _lib.require_cuda(probs, "probs")
        shape = probs.shape
        V = shape[-1]
        flat = probs.reshape(-1, V)
        if flat.dtype not in (torch.bfloat16, torch.float32):
            flat = flat.float()
        flat = flat.contiguous()
        rows = flat.shape[0]
        gen_dev = generator.device if generator is not None else probs.device
        u = torch.rand(rows, generator=generator, device=gen_dev, dtype=torch.float32).to(probs.device)
        out = torch.empty(rows, dtype=torch.long, device=probs.device)
        _lib.call("b200_sample_topp_topk", flat.data_ptr(), int(flat.dtype == torch.bfloat16), rows, V, flat.stride(0),
                  float(p), int(k), u.data_ptr(), out.data_ptr(), _lib.stream())
        return out.reshape(*shape[:-1])

    @torch.inference_mode()
    def _prompt_tensor(self, prompt, batch_size: int, dev) -> torch.Tensor:
        """Prompt normalisation of midi_model.py:173-190 / app.py:36-54 -> int64 [B, P, T] on the device."""
        tok = self.tokenizer
        T = tok.max_token_seq
        if prompt is None:
            inp = torch.full((batch_size, 1, T), tok.pad_id, dtype=torch.long, device=dev)
            inp[:, 0, 0] = tok.bos_id
            return inp
        if len(prompt.shape) == 2:
            prompt = np.repeat(prompt[None, :], repeats=batch_size, axis=0)
        elif prompt.shape[0] == 1:
            prompt = np.repeat(prompt, repeats=batch_size, axis=0)
        elif len(prompt.shape) != 3 or prompt.shape[0] != batch_size:
            raise ValueError(f"invalid shape for prompt, {prompt.shape}")
        prompt = prompt[..., :T]
        if prompt.shape[-1] < T:
            prompt = np.pad(prompt, ((0, 0), (0, 0), (0, T - prompt.shape[-1])), mode="constant",
                            constant_values=tok.pad_id)
        return torch.from_numpy(np.ascontiguousarray(prompt)).to(dtype=torch.long, device=dev)

    def _checkout_generator(self, batch_size, max_len, temp, top_p, top_k, generator):
        """Exclusive use of a device-resident generate loop for these settings, reseeded from `generator`; hand it back
        with _return_generator.  Idle generators are reused (graph capture and KV pools are the expensive part)."""
        rt = self._rt()
        gen_dev = generator.device if generator is not None else torch.device("cpu")
        seed = int(torch.randint(0, 2 ** 62, (1,), generator=generator, device=gen_dev).item())
        key = (batch_size, max_len, float(temp), float(top_p), int(top_k))
        self._refresh_merged(rt)
        with rt.pool_lock:
            idle = rt.gen_pool.get(key)
            gg = idle.pop() if idle else None
            if gg is None:
                for k in [k for k in rt.gen_pool if k != key]:      # other settings: drop their idle pools (KV is large)
                    del rt.gen_pool[k]
                if rt.grammar is None:
                    rt.grammar = _dec.GrammarLUT(self.tokenizer, rt.store.device)
                outer, inner = self._cached_stack("outer", refresh=False), self._cached_stack("inner", refresh=False)
        if gg is None:
            gg = _dec.GraphGenerator(outer, inner, rt.lm_head, rt.pitch, rt.V, self.tokenizer, rt.grammar, batch_size,
                                     max_len, temp, top_p, top_k, seed)
        gg.seed = seed & ((1 << 63) - 1)
        return key, gg

    def _return_generator(self, key, gg) -> None:
        rt = self.__dict__.get("_b200_rt")
        if rt is None or gg.outer is not rt.cached_outer:         # the runtime was rebuilt meanwhile: drop it
            return
        with rt.pool_lock:
            idle = rt.gen_pool.setdefault(key, [])
            if len(idle) < 2:                                      # keep at most two idle loops per setting
                idle.append(gg)

    @torch.inference_mode()
    def generate_stream(self, prompt=None, batch_size=1, max_len=512, temp=1.0, top_p=0.98, top_k=20,
                        disable_patch_change=False, disable_control_change=False, disable_channels=None, generator=None):
        """app.py:27-120 (the gradio app's own generate loop) on the device-resident loop: a Python generator that
        yields every new event as an int64 numpy array [batch, max_token_seq], with the app's extra grammar options
        (`disable_patch_change`, `disable_control_change`, `disable_channels` = channel numbers) applied as a device-side
        mask, the app's 4096-event context window (app.py:55) and its stop rule (all rows EOS in the same event).
        One device->host copy per event, no sync per token."""
        tok = self.tokenizer
        rt = self._rt()
        dev = rt.store.device
        deny = []
        if disable_patch_change:
            deny.append(tok.event_ids["patch_change"])
        if disable_control_change:
            deny.append(tok.event_ids["control_change"])
        for c in (disable_channels or []):
            deny.append(tok.parameter_ids["channel"][c])
        inp = self._prompt_tensor(prompt, batch_size, dev)[:, -4096:]
        if inp.shape[1] >= max_len:
            return
        mode = os.environ.get("B200_GENERATE", "persist")
        # this generation owns its loop state (no lock is held across the yields; see _Runtime.gen_pool)
        key, gg = self._checkout_generator(batch_size, max_len, temp, top_p, top_k, generator)
        try:
            gg.set_deny(deny)
            for ev in gg.events(inp, use_graph=_loop_mode(mode)):
                yield ev.numpy()
        finally:
            gg.set_deny(())
            self._return_generator(key, gg)

    def generate(self, prompt=None, batch_size=1, max_len=512, temp=1.0, top_p=0.98, top_k=20, generator=None):
        """midi_model.py:167-250 with the per-token work on the device (see midi_b200/decode.py)."""
        tok = self.tokenizer
        T = tok.max_token_seq
        rt = self._rt()
        dev = rt.store.device
        inp = self._prompt_tensor(prompt, batch_size, dev)
        cur_len = inp.shape[1]
        if cur_len >= max_len:
            return inp.cpu().numpy()
        if rt.grammar is None:
            rt.grammar = _dec.GrammarLUT(tok, dev)
        mode = os.environ.get("B200_GENERATE", "persist")
        if mode != "eager" and max_len - cur_len >= 4:
            # device-resident loop: one CUDA graph replay per event (midi_b200/decode.py::GraphGenerator)
            key, gg = self._checkout_generator(batch_size, max_len, temp, top_p, top_k, generator)
            try:
                gg.set_deny(())
                bar = tqdm.tqdm(desc="generating", total=max_len - cur_len)
                with bar:
                    out = gg.run(inp, use_graph=_loop_mode(mode), progress=bar.update)
            finally:
                self._return_generator(key, gg)
            return out.cpu().numpy()
        seq = torch.full((batch_size, max_len, T), tok.pad_id, dtype=torch.long, device=dev)
        seq[:, :cur_len] = inp
        g = rt.grammar
        n_params = g.n_params
        outer, inner = self._cached_stack("outer"), self._cached_stack("inner")
        kv1 = _dec.PagedKV(rt.outer.cfg, batch_size, max(max_len, 1), 64, dev)
        kv2 = _dec.PagedKV(rt.inner.cfg, batch_size, T, T, dev)
        gen_dev = generator.device if generator is not None else dev
        past_len = 0
        bar = tqdm.tqdm(desc="generating", total=max_len - cur_len)
        with bar:
            while cur_len < max_len:
                s_new = cur_len - past_len
                e = _ops.embed_sum(seq[:, past_len:cur_len].reshape(batch_size * s_new, T), rt.outer.embed)
                hidden = outer.step(e, kv1, s_new).view(batch_size, s_new, -1)[:, -1].contiguous()
                evb = torch.full((batch_size, T), tok.pad_id, dtype=torch.long, device=dev)   # event being generated
                evt0 = evb                               # step-0 tokens (contiguous [B]) once sampled
                kv2.reset()
                n_steps = T
                end = [False] * batch_size
                for i in range(T):
                    if i >= n_steps:
                        break
                    if i == 0:
                        xin = _ops.inner_input(hidden, None, rt.inner.embed)
                    else:
                        xin = _ops.inner_input(None, evb[:, i - 1:i].contiguous(), rt.inner.embed)
                    hs = inner.step(xin, kv2, 1)
                    logits = _dec._lm_head(hs, rt.lm_head, rt.pitch)
                    u = torch.rand(batch_size, generator=generator, device=gen_dev, dtype=torch.float32).to(dev)
                    _dec.sample_from_logits(logits, rt.V, float(temp), float(top_p), int(top_k), i, evt0, g, u, evb)
                    if i == 0:
                        # one small device->host read per event: the reference's `end` / early-exit logic
                        # (midi_model.py:224-237) needs the event types on the host
                        evt0 = evb[:, 0].contiguous()
                        evt = evt0.tolist()
                        end = [t == tok.eos_id for t in evt]
                        lens = {n_params.get(t, 0) for t, e_ in zip(evt, end) if not e_}
                        if len(lens) == 0:
                            n_steps = 2            # all rows ended: reference breaks after i == 1
                        elif len(lens) == 1:
                            n_steps = lens.pop() + 1
                        else:
                            n_steps = T
                seq[:, cur_len] = evb
                past_len = cur_len
                cur_len += 1
                bar.update(1)
                if all(end):
                    break
        return seq[:, :cur_len].cpu().numpy()

    # ------------------------------------------------------------------ fused training path (non-reference API)
    def training_loss(self, batch: torch.Tensor, backward: bool = True, accumulate: bool = False, grad_ready=None):
        """train.py:168-185 (sample_seq=False) fused: x = batch[:, :-1], y = batch[:, 1:], both stacks, lm_head,
        mean CE with ignore_index=pad -- and, if `backward`, every gradient written to the flat gradient buffer
        (`.grad` of each parameter is a view of it).  Returns a 0-dim fp32 tensor (no host sync).
        `grad_ready(start, end)` (optional) is called as soon as a slice of the flat gradient buffer is final --
        first the token-level stack + lm_head, then the event-level stack -- so a data-parallel trainer can start
        the all-reduce of the first slice while the second is still being computed (midi_b200/ddp.py)."""
        rt = self._rt()
        tok = self.tokenizer
        B, S1, T = batch.shape
        S = S1 - 1
        if batch.dtype == torch.int16:
            x, y = _ops.batch_to_xy(batch.contiguous())        # int16 host data path (midi_b200/data.py): one widening pass
        else:
            batch = batch.to(torch.long)
            x = batch[:, :-1].contiguous().view(B * S, T)
            y = batch[:, 1:].contiguous().view(B * S, T)
        e = _ops.embed_sum(x, rt.outer.embed)
        hidden, sv_o = rt.outer.forward(e, B, S, self.net.rotary_emb.inv_freq, save=backward)
        ids_in = y[:, :-1].contiguous()
        xin = _ops.inner_input(hidden, ids_in, rt.inner.embed)
        hs, sv_i = rt.inner.forward(xin, B * S, T, self.net_token.rotary_emb.inv_freq, save=backward)
        del xin
        logits = _ops.linear(hs, rt.lm_head, pitch=rt.pitch)
        targets = y.reshape(-1)
        lac, lse = _ops.ce_fwd(logits, targets, rt.V, tok.pad_id)
        loss = lac[0]
        if backward:
            _ops.ce_bwd_(logits, targets, lse, lac, rt.V, tok.pad_id, 1.0)
            g_i, g_o = rt.inner.main_grads, rt.outer.main_grads
            dhidden, = _inner_backward(rt, self, sv_i, hs, logits, ids_in, B * S, T, T - 1, True, g_i, rt.g_lm_head,
                                       accumulate)
            del logits, hs
            # Gradient hand-over to a data-parallel trainer.  Base parameters that train (full training): slices of the flat
            # buffer as backward finishes them.  Adapter matrices (LoRA, train.py:439-449) sit in the tail
            # [base_numel, numel) and are handed over in one piece at the end (40 MB for r = 64 on tv2o-medium).
            base_sync = grad_ready is not None and (rt.inner.base_trainable or rt.outer.base_trainable or rt.tr_lm_head)
            if base_sync:
                grad_ready(rt.inner.seg_start, rt.store.base_numel)
            layer_done = None
            if base_sync:
                # event-level stack: hand finished gradients over in groups of 3 layers while backward continues
                hi = [rt.inner.seg_start]

                def layer_done(li):
                    # groups of three layers while a lot of backward is still ahead (fewer, larger collectives); the last
                    # three layers one by one, so that only the first layer (33.5 MB) and the embedding table are still
                    # to be reduced when the backward pass ends
                    if li % 3 == 0 or li < 3:
                        lo = rt.outer.layer_range(li)[0]
                        grad_ready(lo, hi[0])
                        hi[0] = lo
            de = rt.outer.backward(sv_o, dhidden, g_o, accumulate=accumulate, layer_done=layer_done)
            if g_o.embed is not None:
                _ops.embed_bwd(x.view(-1), de, g_o.embed, per_row=T, row_stride=1, row_inner=0, row_off=0,
                               pad_id=self.config.net_config.pad_token_id, accumulate=accumulate)
            if base_sync:
                grad_ready(0, hi[0])          # embedding table (+ whatever is left)
            if grad_ready is not None and rt.store.numel > rt.store.base_numel:
                grad_ready(rt.store.base_numel, rt.store.numel)
            rt.store.publish_grads()
        return loss

    def _opt_state(self, rt):
        """AdamW moments (fp32) over the trainable span of the flat parameter buffer -- everything in full training, the
        adapter tail in a LoRA run.  They live on the MODEL, not on the runtime, so they survive a runtime rebuild (the flat
        layout is a function of named_parameters() only); a model whose trainable span changed gets fresh moments and says
        so."""
        store = rt.store
        if not store.train_dense:
            raise _lib.B200Error("fused optimizer: frozen parameters sit between trainable ones in the flat buffer (it "
                                 "supports full training and LoRA-only training); use a torch optimizer on "
                                 "model.parameters() for other mixes")
        st = self.__dict__.get("_b200_opt")
        lo, hi, dev = store.train_lo, store.train_hi, store.device
        n = hi - lo
        if st is not None and (st["m"].numel() != n or st.get("span") != (lo, hi) or st["m"].device != dev):
            if st["m"].numel() != n or st.get("span") != (lo, hi):
                import warnings
                warnings.warn("fused AdamW: the set of trainable parameters changed; optimizer moments restart from zero")
                st = None
            else:
                st = {k: (v.to(dev) if isinstance(v, torch.Tensor) and k != "step" else v) for k, v in st.items()}
                self.__dict__["_b200_opt"] = st
        if st is None:
            st = dict(m=torch.zeros(n, dtype=torch.float32, device=dev), v=torch.zeros(n, dtype=torch.float32, device=dev),
                      nc=torch.zeros(2, dtype=torch.float32, device=dev), step=torch.zeros(1, dtype=torch.int64),
                      span=(lo, hi))
            self.__dict__["_b200_opt"] = st
        return st

    def fused_optimizer_step(self, lr: float, step: int, weight_decay: float = 0.01, betas=(0.9, 0.99), eps: float = 1e-8,
                             max_grad_norm: float = 1.0):
        """Global-norm clip (train.py:464) + AdamW with the no-decay split (train.py:121-138) over the trainable span of
        the flat parameter / gradient buffers: two small reductions and one update launch."""
        rt = self._rt()
        st = self._opt_state(rt)
        lo, hi = st["span"]
        n = hi - lo
        if n == 0:
            raise _lib.B200Error("fused optimizer: the model has no trainable parameters")
        align = _engine.ALIGN
        parts = _lib.query("b200_gradnorm_parts")
        ws = _ops._ws("gradnorm", parts * 4, rt.store.device)
        gptr, pptr = rt.store.gflat.data_ptr() + 2 * lo, rt.store.flat.data_ptr() + 2 * lo
        _lib.call("b200_grad_clip_coef", gptr, n, float(max_grad_norm), st["nc"].data_ptr(),
                  ws.data_ptr(), ws.numel(), _lib.stream())
        _lib.call("b200_adamw_step", pptr, gptr, st["m"].data_ptr(),
                  st["v"].data_ptr(), rt.store.nodecay.data_ptr() + lo // align, n, float(lr), float(betas[0]), float(betas[1]),
                  float(eps), float(weight_decay), int(step), st["nc"].data_ptr(), _lib.stream())
        st["step"][0] = int(step)
        rt.lora_step += 1
        return st["nc"]

    def optimizer_state_dict(self) -> Dict[str, Any]:
        """Checkpointable state of the fused AdamW, in torch.optim's vocabulary: {"step": int, "state": {parameter name:
        {"exp_avg", "exp_avg_sq"}}} (fp32 CPU tensors shaped like the parameter).  Empty before the first step."""
        st = self.__dict__.get("_b200_opt")
        if st is None:
            return {"step": 0, "state": {}}
        rt = self._rt()
        lo, hi = st["span"]
        out = {}
        for name in rt.store.names:
            o, v = rt.store.offsets[name] - lo, rt.store.views[name]
            if not (lo <= rt.store.offsets[name] < hi):
                continue                                   # frozen (e.g. the base of a LoRA run): no moments
            out[name] = {"exp_avg": st["m"][o:o + v.numel()].view(v.shape).cpu().clone(),
                         "exp_avg_sq": st["v"][o:o + v.numel()].view(v.shape).cpu().clone()}
        return {"step": int(st["step"][0]), "state": out}

    def load_optimizer_state_dict(self, sd: Dict[str, Any]) -> int:
        """Inverse of optimizer_state_dict(); returns the step to resume from (pass step + 1 to fused_optimizer_step)."""
        rt = self._rt()
        st = self._opt_state(rt)
        st["m"].zero_()
        st["v"].zero_()
        lo, hi = st["span"]
        for name, ent in sd.get("state", {}).items():
            if name not in rt.store.offsets:
                raise KeyError(f"load_optimizer_state_dict: unknown parameter {name}")
            if not (lo <= rt.store.offsets[name] < hi):
                raise KeyError(f"load_optimizer_state_dict: {name} is not trainable in this model")
            o, v = rt.store.offsets[name] - lo, rt.store.views[name]
            if tuple(ent["exp_avg"].shape) != tuple(v.shape):
                raise ValueError(f"load_optimizer_state_dict: {name}: shape {tuple(ent['exp_avg'].shape)} vs {tuple(v.shape)}")
            st["m"][o:o + v.numel()].view(v.shape).copy_(ent["exp_avg"])
            st["v"][o:o + v.numel()].view(v.shape).copy_(ent["exp_avg_sq"])
        st["step"][0] = int(sd.get("step", 0))
        return int(sd.get("step", 0))
