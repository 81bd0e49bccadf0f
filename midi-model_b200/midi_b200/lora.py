"""LoRA adapters for MIDIModel in peft's module / state-dict layout, without peft.

The reference trains LoRA through `model.add_adapter(LoraConfig(r=64, lora_alpha=128, target_modules=[q,k,v,o,gate,up,
down]_proj, lora_dropout=0, bias="none"))` (train.py:439-449), saves `adapter_config.json` +
`adapter_model.safetensors` (train.py:234-244) and merges them for inference (midi_model.py:109-114).  peft is not part
of this image, and the native engine never calls a module's `forward` anyway: the HF modules are parameter containers.
So what has to match peft is the *container*: every targeted `nn.Linear` becomes a module with

    <path>.base_layer.weight                 frozen base weight (same Parameter object as before)
    <path>.lora_A.<adapter>.weight  [r, in]  kaiming-uniform(a=sqrt(5))
    <path>.lora_B.<adapter>.weight  [out, r] zeros
    .scaling[<adapter>] = lora_alpha / r     (lora_alpha / sqrt(r) with use_rslora)

which is exactly what peft's `lora.Linear` exposes, so `midi_b200.engine` reads a peft-injected model (peft installed) and a
natively injected one (this file) through the same attributes.  Forward semantics the engine implements
(peft lora/layer.py `Linear.forward`): y = base(x) + lora_B(lora_A(x)) * scaling.
"""
from __future__ import annotations

import json
import math
import os
import re
from typing import Any, Dict, Iterable, List, Optional

import torch
import torch.nn as nn

from .lib import B200Error

PROJ_ORDER = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


class LoraAdapterConfig:
    """The fields of peft.LoraConfig that train.py sets, with peft's `save_pretrained` file format (adapter_config.json).
    Accepts a peft LoraConfig, a dict or keyword arguments; unknown fields are kept and written back."""
    peft_type = "LORA"

    def __init__(self, r: int = 8, lora_alpha: float = 8, target_modules=None, lora_dropout: float = 0.0, bias: str = "none",
                 task_type=None, use_rslora: bool = False, fan_in_fan_out: bool = False, init_lora_weights=True, **extra):
        self.r = int(r)
        self.lora_alpha = lora_alpha
        if target_modules is not None and not isinstance(target_modules, str):
            target_modules = list(target_modules)
        self.target_modules = target_modules
        self.lora_dropout = float(lora_dropout)
        self.bias = bias
        self.task_type = getattr(task_type, "value", task_type)
        self.use_rslora = bool(use_rslora)
        self.fan_in_fan_out = bool(fan_in_fan_out)
        self.init_lora_weights = init_lora_weights
        self.extra = {k: v for k, v in extra.items() if k != "peft_type"}

    @classmethod
    def from_any(cls, cfg) -> "LoraAdapterConfig":
        if isinstance(cfg, LoraAdapterConfig):
            return cfg
        if isinstance(cfg, dict):
            return cls(**cfg)
        fields = ("r", "lora_alpha", "target_modules", "lora_dropout", "bias", "task_type", "use_rslora", "fan_in_fan_out",
                  "init_lora_weights")
        if not hasattr(cfg, "r") or not hasattr(cfg, "target_modules"):
            raise TypeError(f"add_adapter: expected a LoRA config (object or dict with r / target_modules), got {type(cfg)}")
        kind = str(getattr(getattr(cfg, "peft_type", "LORA"), "value", getattr(cfg, "peft_type", "LORA"))).upper()
        if kind != "LORA":
            raise ValueError(f"add_adapter: unsupported peft_type {kind} (LoRA only)")
        return cls(**{f: getattr(cfg, f) for f in fields if hasattr(cfg, f)})

    def scaling(self) -> float:
        return self.lora_alpha / math.sqrt(self.r) if self.use_rslora else self.lora_alpha / self.r

    def to_dict(self) -> Dict[str, Any]:
        tm = self.target_modules
        d = dict(self.extra)
        d.update(peft_type="LORA", task_type=self.task_type, r=self.r, lora_alpha=self.lora_alpha,
                 target_modules=sorted(tm) if isinstance(tm, (list, tuple, set)) else tm, lora_dropout=self.lora_dropout,
                 bias=self.bias, use_rslora=self.use_rslora, fan_in_fan_out=self.fan_in_fan_out,
                 init_lora_weights=self.init_lora_weights, inference_mode=False, base_model_name_or_path=None)
        return d

    def save_pretrained(self, save_directory: str, **_):
        os.makedirs(save_directory, exist_ok=True)
        with open(os.path.join(save_directory, "adapter_config.json"), "w") as f:
            json.dump(self.to_dict(), f, indent=2, sort_keys=True)

    @classmethod
    def from_pretrained(cls, directory: str) -> "LoraAdapterConfig":
        with open(os.path.join(directory, "adapter_config.json")) as f:
            d = json.load(f)
        for k in ("inference_mode", "base_model_name_or_path"):
            d.pop(k, None)
        return cls(**d)


class LoraLinear(nn.Module):
    """Container with the attribute layout of peft's lora.Linear.  It holds parameters; it does not compute (the engine
    does), so calling it raises instead of silently running a PyTorch path."""

    def __init__(self, base_layer: nn.Linear, adapter_name: str, cfg: LoraAdapterConfig):
        super().__init__()
        if not isinstance(base_layer, nn.Linear) or base_layer.bias is not None:
            raise B200Error("LoRA targets must be bias-free nn.Linear layers")
        self.base_layer = base_layer
        self.in_features, self.out_features = base_layer.in_features, base_layer.out_features
        self.lora_A = nn.ModuleDict()
        self.lora_B = nn.ModuleDict()
        self.lora_dropout = nn.ModuleDict()
        self.r: Dict[str, int] = {}
        self.lora_alpha: Dict[str, float] = {}
        self.scaling: Dict[str, float] = {}
        self.use_dora: Dict[str, bool] = {}
        self.active_adapters: List[str] = []
        self.merged = False
        self.disable_adapters = False
        self.update_layer(adapter_name, cfg)

    @property
    def weight(self) -> torch.Tensor:
        return self.base_layer.weight

    def update_layer(self, adapter_name: str, cfg: LoraAdapterConfig):
        if cfg.r <= 0:
            raise ValueError(f"`r` should be a positive integer value but the value passed is {cfg.r}")
        w = self.base_layer.weight
        # peft lora/layer.py update_layer: two default-initialised Linear layers, then reset_lora_parameters
        A = nn.Linear(self.in_features, cfg.r, bias=False)
        Bm = nn.Linear(cfg.r, self.out_features, bias=False)
        if cfg.init_lora_weights is not False:
            nn.init.kaiming_uniform_(A.weight, a=math.sqrt(5))
            nn.init.zeros_(Bm.weight)
        self.lora_A[adapter_name] = A.to(device=w.device, dtype=w.dtype)
        self.lora_B[adapter_name] = Bm.to(device=w.device, dtype=w.dtype)
        self.lora_dropout[adapter_name] = nn.Identity()
        self.r[adapter_name] = cfg.r
        self.lora_alpha[adapter_name] = cfg.lora_alpha
        self.scaling[adapter_name] = cfg.scaling()
        self.use_dora[adapter_name] = False
        self.active_adapters = [adapter_name]

    def forward(self, *args, **kwargs):
        raise B200Error("LoraLinear is a parameter container: MIDIModel computes through the native engine "
                        "(forward / forward_token / training_loss), there is no PyTorch path")


def _is_target(key: str, targets) -> bool:
    if isinstance(targets, str):
        return re.fullmatch(targets, key) is not None
    return key in targets or any(key.endswith("." + t) for t in targets)


def inject(model: nn.Module, cfg: LoraAdapterConfig, adapter_name: str = "default") -> List[str]:
    """What peft's inject_adapter_in_model does for LoRA on Linear targets: wrap every matching layer, then leave only
    the adapter weights trainable (mark_only_lora_as_trainable, bias="none").  Returns the wrapped module paths."""
    if cfg.lora_dropout != 0.0:
        raise B200Error("lora_dropout > 0 is not supported by the native engine (train.py:447 uses 0)")
    if cfg.bias != "none":
        raise B200Error(f"LoRA bias mode {cfg.bias!r} is not supported (train.py:445 uses 'none')")
    if cfg.fan_in_fan_out:
        raise B200Error("fan_in_fan_out LoRA is for Conv1D layers; MIDIModel has nn.Linear projections only")
    if cfg.r % 8:
        raise B200Error(f"LoRA rank {cfg.r}: the tensor-core kernels need r to be a multiple of 8 (16-byte rows)")
    if not cfg.target_modules:
        raise ValueError("add_adapter: target_modules must name the projections to adapt")
    wrapped = []
    for key, mod in list(model.named_modules()):
        if not key or not _is_target(key, cfg.target_modules):
            continue
        if isinstance(mod, LoraLinear):
            mod.update_layer(adapter_name, cfg)
            wrapped.append(key)
            continue
        if not isinstance(mod, nn.Linear):
            continue
        parent_name, _, leaf = key.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, leaf, LoraLinear(mod, adapter_name, cfg))
        wrapped.append(key)
    if not wrapped:
        raise ValueError(f"Target modules {cfg.target_modules} not found in the base model")
    # peft: _mark_only_adapters_as_trainable freezes everything that is not an adapter, set_adapter leaves only the ACTIVE
    # adapter's matrices trainable (an earlier, now inactive adapter must not be decayed by an optimizer that sees no gradient)
    for n, p in model.named_parameters():
        p.requires_grad_(f".lora_A.{adapter_name}." in n or f".lora_B.{adapter_name}." in n)
    return wrapped


def adapter_state_dict(model: nn.Module, adapter_name: str = "default") -> Dict[str, torch.Tensor]:
    """peft.get_peft_model_state_dict for LoRA with bias="none": the lora_A / lora_B tensors with the adapter name removed
    from the key (`...q_proj.lora_A.weight`) -- the file train.py:241-244 writes."""
    out = {}
    for k, v in model.state_dict().items():
        if ".lora_" in k and f".{adapter_name}." in k:
            out[k.replace(f".{adapter_name}", "")] = v
    return out


def load_adapter_state_dict(model: nn.Module, sd: Dict[str, torch.Tensor], adapter_name: str = "default") -> None:
    """Inverse of adapter_state_dict (keys may carry peft's `base_model.model.` prefix)."""
    params = dict(model.named_parameters())
    seen = 0
    with torch.no_grad():
        for k, v in sd.items():
            m = re.fullmatch(r"(?:base_model\.model\.)?(.+)\.lora_(A|B)(?:\.[^.]+)?\.weight", k)
            if m is None:
                continue
            name = f"{m.group(1)}.lora_{m.group(2)}.{adapter_name}.weight"
            if name not in params:
                raise KeyError(f"adapter tensor {k}: the model has no parameter {name}")
            if tuple(params[name].shape) != tuple(v.shape):
                raise ValueError(f"adapter tensor {k}: shape {tuple(v.shape)} vs {tuple(params[name].shape)}")
            params[name].copy_(v)
            seen += 1
    if seen == 0:
        raise ValueError("no lora_A / lora_B tensors in the adapter state dict")


class LoraSite:
    """One adapted projection as the engine sees it: parameter names + scaling."""
    __slots__ = ("path", "a_name", "b_name", "scale", "r")

    def __init__(self, path, a_name, b_name, scale, r):
        self.path, self.a_name, self.b_name, self.scale, self.r = path, a_name, b_name, float(scale), int(r)


def find_sites(model: nn.Module) -> Dict[str, LoraSite]:
    """Module path -> LoraSite for every projection with an ACTIVE, unmerged LoRA adapter -- peft's lora.Linear or the
    LoraLinear above (same attributes).  Raises for adapter features the engine does not implement."""
    sites: Dict[str, LoraSite] = {}
    for path, mod in model.named_modules():
        if not (hasattr(mod, "base_layer") and hasattr(mod, "lora_A") and hasattr(mod, "lora_B") and hasattr(mod, "scaling")):
            continue
        if getattr(mod, "merged", False) or getattr(mod, "disable_adapters", False) or len(mod.lora_A) == 0:
            continue
        active = getattr(mod, "active_adapters", None)
        if callable(active):
            active = active()
        if isinstance(active, str):
            active = [active]
        names = [a for a in (active or list(mod.lora_A.keys())) if a in mod.lora_A]
        if not names:
            continue
        if len(names) != 1:
            raise B200Error(f"{path}: {len(names)} active LoRA adapters; the engine runs one adapter at a time")
        a = names[0]
        if not isinstance(mod.base_layer, nn.Linear) or mod.base_layer.bias is not None:
            raise B200Error(f"{path}: LoRA on {type(mod.base_layer).__name__} is not supported (bias-free Linear only)")
        drop = mod.lora_dropout[a] if hasattr(mod, "lora_dropout") and a in mod.lora_dropout else None
        if drop is not None and not isinstance(drop, nn.Identity) and getattr(drop, "p", 0.0) > 0.0:
            raise B200Error(f"{path}: lora_dropout > 0 is not supported by the native engine")
        use_dora = getattr(mod, "use_dora", {})
        if isinstance(use_dora, dict) and use_dora.get(a, False):
            raise B200Error(f"{path}: DoRA is not supported")
        if getattr(mod.lora_A[a], "bias", None) is not None or getattr(mod.lora_B[a], "bias", None) is not None:
            raise B200Error(f"{path}: lora_bias is not supported")
        r = mod.lora_A[a].weight.shape[0]
        if r % 8:
            raise B200Error(f"{path}: LoRA rank {r} must be a multiple of 8")
        sites[path] = LoraSite(path, f"{path}.lora_A.{a}.weight", f"{path}.lora_B.{a}.weight", mod.scaling[a], r)
    return sites


def flat_order_key(name: str):
    """Sort key that places LoRA parameters after all base parameters of the flat buffer, grouped per layer with the A
    matrices of q|k|v and gate|up adjacent (one fused down-projection GEMM each): (stack, layer, A before B, projection)."""
    m = re.fullmatch(r"(.+?)\.layers\.(\d+)\.(?:self_attn|mlp)\.(\w+)\.lora_(A|B)\..+", name)
    if m is None:
        return (1, name, 0, 0, 0)
    proj = PROJ_ORDER.index(m.group(3)) if m.group(3) in PROJ_ORDER else len(PROJ_ORDER)
    return (0, m.group(1), int(m.group(2)), 0 if m.group(4) == "A" else 1, proj)
