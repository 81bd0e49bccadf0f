"""CPU oracle for the MIDIModel hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain-PyTorch restatement of the reference algorithm (SkyTNT/midi-model,
`midi_model.py:99-250`, `train.py:168-188`) and of the third-party arithmetic
it delegates to (HF transformers 5.5.0 `models/llama/modeling_llama.py`,
un-vendored dependency `transformers>=4.36`, `requirements.txt:6`).

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this module, and only as the checker /
timed CPU baseline.  The product (`midi-model_b200/`) never imports it.

Pinning: the reference has no tests or golden vectors of its own, so this restatement is pinned against outputs of the reference itself,
imported read-only with a 4-name `peft` stub
(`oracle/ref_loader.py`); the generating script is `oracle/make_golden.py` and
the vectors live in `tests/golden/`.  `tests/test_oracle.py` re-checks them.

Everything operates on a flat ``state_dict`` with the reference's key names
(`net.layers.{i}.self_attn.q_proj.weight`, ...) so that the same function can
be fed weights from the reference, from the drop-in class or from a file.
Computation happens in the dtype of the weights: with bf16 weights every torch
op rounds where the reference's eager bf16 path rounds (DESIGN.md 3.3).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------
# configuration of one Llama stack (midi_model.py:63-76)
# --------------------------------------------------------------------------
@dataclass
class StackCfg:
    prefix: str          # "net" or "net_token"
    n_layer: int
    n_head: int
    hidden: int
    inner: int
    eps: float = 1e-6
    theta: float = 10000.0

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_head


@dataclass
class ModelCfg:
    """Mirror of MIDIModelConfig.get_config (midi_model.py:63-76)."""
    vocab: int
    n_layer: int = 12
    n_head: int = 16
    n_embd: int = 1024
    n_inner: int = 4096
    max_token_seq: int = 8
    pad_id: int = 0
    bos_id: int = 1
    eos_id: int = 2

    @property
    def net(self) -> StackCfg:
        return StackCfg("net", self.n_layer, self.n_head, self.n_embd, self.n_inner)

    @property
    def net_token(self) -> StackCfg:
        # midi_model.py:71-75: heads//4, layers//4, inner//4
        return StackCfg("net_token", self.n_layer // 4, self.n_head // 4, self.n_embd, self.n_inner // 4)


def default_inv_freq(head_dim: int, theta: float = 10000.0) -> torch.Tensor:
    """hf modeling_llama.py:117-119 (compute_default_rope_parameters)."""
    return 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float) / head_dim))


# --------------------------------------------------------------------------
# elementary ops (each cites the HF line it restates)
# --------------------------------------------------------------------------
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """hf modeling_llama.py:62-67: fp32 normalise, cast back, then multiply by weight."""
    dt = x.dtype
    xf = x.to(torch.float32)
    var = xf.pow(2).mean(-1, keepdim=True)
    xf = xf * torch.rsqrt(var + eps)
    return w * xf.to(dt)


def rope_cos_sin(inv_freq: torch.Tensor, positions: torch.Tensor, dtype: torch.dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    """hf modeling_llama.py:124-135.  `inv_freq` is the module buffer *as stored*
    (i.e. already rounded to bf16 if the module was cast to bf16); it is upcast
    to fp32, multiplied with fp32 positions, cos/sin taken in fp32, then cast."""
    freqs = positions.to(torch.float32)[:, None] * inv_freq.to(torch.float32)[None, :]   # (S, d/2)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    """hf modeling_llama.py:138-142."""
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """hf modeling_llama.py:146-168; x is (B, h, S, d), cos/sin (S, d)."""
    return (x * cos[None, None]) + (rotate_half(x) * sin[None, None])


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q_pos0: int) -> torch.Tensor:
    """hf integrations/sdpa_attention.py:41-104 with the masks the reference
    produces: causal over absolute positions (query i sits at q_pos0+i and sees
    keys 0..q_pos0+i).  Math: softmax(q k^T / sqrt(d)) v, softmax in fp32.
    q (B,h,Sq,d); k, v (B,h,Sk,d)."""
    d = q.shape[-1]
    scores = torch.matmul(q.to(torch.float32), k.to(torch.float32).transpose(-1, -2)) * (1.0 / math.sqrt(d))
    sq, sk = q.shape[-2], k.shape[-2]
    qi = torch.arange(sq, device=q.device)[:, None] + q_pos0
    kj = torch.arange(sk, device=q.device)[None, :]
    scores = scores.masked_fill(kj > qi, float("-inf"))
    p = torch.softmax(scores, dim=-1)
    return torch.matmul(p.to(v.dtype), v)


def swiglu_mlp(x, wg, wu, wd):
    """hf modeling_llama.py:182-184: down(silu(gate(x)) * up(x))."""
    return F.linear(F.silu(F.linear(x, wg)) * F.linear(x, wu), wd)


# --------------------------------------------------------------------------
# one Llama stack (hf modeling_llama.py:303-332 layer, :375-425 model)
# --------------------------------------------------------------------------
class KV:
    """Minimal stand-in for hf DynamicCache (cache_utils.py:88-135): per-layer
    concatenation of post-RoPE keys and of values along the sequence axis."""

    def __init__(self):
        self.k: List[torch.Tensor] = []
        self.v: List[torch.Tensor] = []

    def seq_len(self) -> int:
        return 0 if not self.k else self.k[0].shape[-2]

    def update(self, layer: int, k: torch.Tensor, v: torch.Tensor):
        if layer == len(self.k):
            self.k.append(k)
            self.v.append(v)
        else:
            self.k[layer] = torch.cat([self.k[layer], k], dim=-2)
            self.v[layer] = torch.cat([self.v[layer], v], dim=-2)
        return self.k[layer], self.v[layer]


def llama_stack(sd: Dict[str, torch.Tensor], cfg: StackCfg, x: torch.Tensor,
                inv_freq: Optional[torch.Tensor] = None, cache: Optional[KV] = None,
                collect: Optional[dict] = None) -> torch.Tensor:
    """x: (B, S, hidden) inputs_embeds -> last_hidden_state (B, S, hidden)."""
    B, S, H = x.shape
    h, d = cfg.n_head, cfg.head_dim
    if inv_freq is None:
        inv_freq = default_inv_freq(d, cfg.theta)
        if x.dtype != torch.float32:          # model.to(bf16) rounds the buffer
            inv_freq = inv_freq.to(x.dtype)
    past = cache.seq_len() if cache is not None else 0
    pos = torch.arange(past, past + S, device=x.device)       # hf :394-397
    cos, sin = rope_cos_sin(inv_freq.to(x.device), pos, x.dtype)
    p = cfg.prefix
    for l in range(cfg.n_layer):
        pre = f"{p}.layers.{l}."
        n1 = rmsnorm(x, sd[pre + "input_layernorm.weight"], cfg.eps)
        q = F.linear(n1, sd[pre + "self_attn.q_proj.weight"]).view(B, S, h, d).transpose(1, 2)
        k = F.linear(n1, sd[pre + "self_attn.k_proj.weight"]).view(B, S, h, d).transpose(1, 2)
        v = F.linear(n1, sd[pre + "self_attn.v_proj.weight"]).view(B, S, h, d).transpose(1, 2)
        q = apply_rope(q, cos, sin)
        k = apply_rope(k, cos, sin)
        if cache is not None:
            k, v = cache.update(l, k, v)
        a = attention(q, k, v, past).transpose(1, 2).reshape(B, S, H)
        x = x + F.linear(a, sd[pre + "self_attn.o_proj.weight"])
        n2 = rmsnorm(x, sd[pre + "post_attention_layernorm.weight"], cfg.eps)
        x = x + swiglu_mlp(n2, sd[pre + "mlp.gate_proj.weight"], sd[pre + "mlp.up_proj.weight"],
                           sd[pre + "mlp.down_proj.weight"])
        if collect is not None:
            collect[f"{p}.layer{l}"] = x
    return rmsnorm(x, sd[f"{p}.norm.weight"], cfg.eps)       # hf :421


# --------------------------------------------------------------------------
# MIDIModel methods
# --------------------------------------------------------------------------
def forward(sd, cfg: ModelCfg, x: torch.Tensor, cache: Optional[KV] = None, inv_freq=None) -> torch.Tensor:
    """midi_model.py:137-150: embed, sum over the token axis, outer stack."""
    e = F.embedding(x, sd["net.embed_tokens.weight"], padding_idx=cfg.pad_id)   # (B,S,T,H); hf :363 padding_idx
    e = e.sum(dim=-2)
    return llama_stack(sd, cfg.net, e, inv_freq, cache)


def forward_token(sd, cfg: ModelCfg, hidden_state: Optional[torch.Tensor], x: Optional[torch.Tensor] = None,
                  cache: Optional[KV] = None, inv_freq=None) -> torch.Tensor:
    """midi_model.py:116-135: [hidden, embed(x)] -> inner stack -> lm_head."""
    if hidden_state is not None:
        hidden_state = hidden_state.unsqueeze(1)
    if x is not None:
        xe = F.embedding(x, sd["net_token.embed_tokens.weight"], padding_idx=cfg.pad_id)
        if hidden_state is not None:
            xe = torch.cat([hidden_state, xe], dim=1)
        hidden_state = xe
    hs = llama_stack(sd, cfg.net_token, hidden_state, inv_freq, cache)
    return F.linear(hs, sd["lm_head.weight"])


def train_loss(sd, cfg: ModelCfg, batch: torch.Tensor) -> torch.Tensor:
    """train.py:168-185 (sample_seq=False): the (event, token) double loss."""
    x = batch[:, :-1].contiguous()
    y = batch[:, 1:].contiguous()
    hidden = forward(sd, cfg, x)
    hidden = hidden.reshape(-1, hidden.shape[-1])
    y = y.reshape(-1, y.shape[-1])
    xin = y[:, :-1]
    logits = forward_token(sd, cfg, hidden, xin)
    return F.cross_entropy(logits.view(-1, cfg.vocab), y.view(-1), reduction="mean", ignore_index=cfg.pad_id)


def lora_effective_sd(sd: Dict[str, torch.Tensor], scaling: float, adapter: str = "default") -> Dict[str, torch.Tensor]:
    """LoRA (train.py:439-449 -> `model.add_adapter(LoraConfig(...))`; merge: midi_model.py:109-114).  The arithmetic lives in
    the un-vendored dependency `peft>=0.13.0` (requirements.txt:5), which is NOT in this image: **parity unpinned** against
    peft itself.  Restated from its published algorithm (Hu et al. 2021, eq. 3; peft `tuners/lora/layer.py`
    `Linear.forward`: `result = base_layer(x) + lora_B(lora_A(dropout(x))) * scaling`, `scaling = lora_alpha / r`,
    `Linear.get_delta_weight`: `B @ A * scaling`): for every `<path>.base_layer.weight` with `<path>.lora_A/B.<adapter>.weight`
    the effective weight `W + scaling * B A` under the reference's key `<path>.weight`.  Differentiable, so autograd through
    it yields the adapter gradients of the unmerged forward (identical in exact arithmetic)."""
    out = {}
    for k, v in sd.items():
        if ".lora_" in k:
            continue
        if k.endswith(".base_layer.weight"):
            path = k[:-len(".base_layer.weight")]
            a, b = sd[f"{path}.lora_A.{adapter}.weight"], sd[f"{path}.lora_B.{adapter}.weight"]
            out[path + ".weight"] = v + scaling * (b @ a)
        else:
            out[k] = v
    return out


def sample_top_p_k(probs: torch.Tensor, p: float, k: int, generator=None, stable: bool = True) -> torch.Tensor:
    """midi_model.py:152-165.  `stable=True` breaks exact ties by ascending id
    (the reference's torch.sort is unstable; its tie order is implementation
    defined)."""
    probs_sort, probs_idx = torch.sort(probs, dim=-1, descending=True, stable=stable)
    probs_sum = torch.cumsum(probs_sort, dim=-1)
    mask = probs_sum - probs_sort > p
    probs_sort[mask] = 0.0
    m = torch.zeros(probs_sort.shape[-1], device=probs_sort.device)
    m[:k] = 1
    probs_sort = probs_sort * m
    probs_sort.div_(probs_sort.sum(dim=-1, keepdim=True))
    shape = probs_sort.shape
    nt = torch.multinomial(probs_sort.reshape(-1, shape[-1]), num_samples=1, generator=generator).reshape(*shape[:-1], 1)
    return torch.gather(probs_idx, -1, nt).reshape(*shape[:-1])


def grammar_tables(tok) -> dict:
    """Flatten the tokenizer grammar used by generate (midi_tokenizer.py:517-535)
    into id ranges: step 0 -> {eos} + event ids; step i -> parameter_ids[...]."""
    ev = {}
    for name, params in tok.events.items():
        ev[tok.event_ids[name]] = [(tok.parameter_ids[pn][0], tok.parameter_ids[pn][-1] + 1) for pn in params]
    return ev


@torch.no_grad()
def _prompt_tensor(tok, prompt, batch_size, dev):
    """Prompt normalisation shared by midi_model.py:173-190 and app.py:36-54."""
    import numpy as np
    T = tok.max_token_seq
    if prompt is None:
        inp = torch.full((1, T), tok.pad_id, dtype=torch.long, device=dev)
        inp[0, 0] = tok.bos_id
        return inp.unsqueeze(0).repeat(batch_size, 1, 1)
    if prompt.ndim == 2:
        prompt = np.repeat(prompt[None, :], batch_size, axis=0)
    elif prompt.shape[0] == 1:
        prompt = np.repeat(prompt, batch_size, axis=0)
    elif prompt.ndim != 3 or prompt.shape[0] != batch_size:
        raise ValueError(f"invalid shape for prompt, {prompt.shape}")
    prompt = prompt[..., :T]
    if prompt.shape[-1] < T:
        prompt = np.pad(prompt, ((0, 0), (0, 0), (0, T - prompt.shape[-1])), constant_values=tok.pad_id)
    return torch.from_numpy(prompt).to(dtype=torch.long, device=dev)


def deny_ids(tok, disable_patch_change=False, disable_control_change=False, disable_channels=None):
    """Token ids app.py:31-34,73-76,86-87 removes from the grammar masks (event-type ids at step 0, channel ids)."""
    deny = set()
    if disable_patch_change:
        deny.add(tok.event_ids["patch_change"])
    if disable_control_change:
        deny.add(tok.event_ids["control_change"])
    for c in (disable_channels or []):
        deny.add(tok.parameter_ids["channel"][c])
    return deny


def generate_stream(sd, cfg: ModelCfg, tok, prompt=None, batch_size=1, max_len=512, temp=1.0, top_p=0.98, top_k=20,
                    generator=None, inv_freq_net=None, inv_freq_tok=None, deny=(), max_context=None):
    """The generate loop of midi_model.py:167-250 / app.py:27-120 restated as a Python generator: yields the first
    (prompt) block [B, P, T] and then one int64 [B, T] event per iteration.  Same quirks: `end` is reset per event and
    the loop exits only when all rows end on the same event.  `deny` = ids removed from every grammar mask
    (app.py's disable_* options, see deny_ids); `max_context` = app.py:55's `input_tensor[:, -4096:]`."""
    T = tok.max_token_seq
    dev = sd["lm_head.weight"].device
    inp = _prompt_tensor(tok, prompt, batch_size, dev)
    if max_context is not None:
        inp = inp[:, -max_context:]
    deny = set(deny)
    yield inp
    cur_len = inp.shape[1]
    cache1 = KV()
    past_len = 0
    V = cfg.vocab
    while cur_len < max_len:
        end = [False] * batch_size
        hidden = forward(sd, cfg, inp[:, past_len:], cache1, inv_freq_net)[:, -1]
        seq = None
        names = [""] * batch_size
        cache2 = KV()
        for i in range(T):
            mask = torch.zeros((batch_size, V), dtype=torch.int64, device=dev)
            for b in range(batch_size):
                if end[b]:
                    mask[b, tok.pad_id] = 1
                    continue
                if i == 0:
                    ids = list(tok.event_ids.values()) + [tok.eos_id]
                else:
                    pn = tok.events[names[b]]
                    if i > len(pn):
                        mask[b, tok.pad_id] = 1
                        continue
                    ids = tok.parameter_ids[pn[i - 1]]
                mask[b, [t for t in ids if t not in deny]] = 1
            mask = mask.unsqueeze(1)
            if i == 0:
                logits = forward_token(sd, cfg, hidden, None, cache2, inv_freq_tok)[:, -1:]
            else:
                logits = forward_token(sd, cfg, None, seq[:, -1:], cache2, inv_freq_tok)[:, -1:]
            scores = torch.softmax(logits / temp, dim=-1) * mask
            samples = sample_top_p_k(scores, top_p, top_k, generator=generator)
            if i == 0:
                seq = samples
                for b in range(batch_size):
                    if end[b]:
                        continue
                    eid = samples[b].item()
                    if eid == tok.eos_id:
                        end[b] = True
                    else:
                        names[b] = tok.id_events[eid]
            else:
                seq = torch.cat([seq, samples], dim=1)
                if all(len(tok.events[names[b]]) == i for b in range(batch_size) if not end[b]):
                    break
        if seq.shape[1] < T:
            seq = F.pad(seq, (0, T - seq.shape[1]), "constant", value=tok.pad_id)
        inp = torch.cat([inp, seq.unsqueeze(1)], dim=1)
        past_len = cur_len
        cur_len += 1
        yield seq
        if all(end):
            break


def generate(sd, cfg: ModelCfg, tok, prompt=None, batch_size=1, max_len=512, temp=1.0, top_p=0.98, top_k=20,
             generator=None, inv_freq_net=None, inv_freq_tok=None, deny=(), max_context=None):
    """midi_model.py:167-250: the whole [B, L, T] result as numpy (prompt + generated events)."""
    blocks = []
    for blk in generate_stream(sd, cfg, tok, prompt, batch_size, max_len, temp, top_p, top_k, generator, inv_freq_net,
                               inv_freq_tok, deny, max_context):
        blocks.append(blk if blk.dim() == 3 else blk.unsqueeze(1))
    return torch.cat(blocks, dim=1).cpu().numpy()


# --------------------------------------------------------------------------
# helpers shared by tests and bench
# --------------------------------------------------------------------------
def cfg_from_hf(config) -> ModelCfg:
    """Build a ModelCfg from a MIDIModelConfig-like object."""
    nc = config.net_config
    tok = config.tokenizer
    return ModelCfg(vocab=tok.vocab_size, n_layer=nc.num_hidden_layers, n_head=nc.num_attention_heads,
                    n_embd=nc.hidden_size, n_inner=nc.intermediate_size, max_token_seq=tok.max_token_seq,
                    pad_id=tok.pad_id, bos_id=tok.bos_id, eos_id=tok.eos_id)


def rel_fro(a: torch.Tensor, b: torch.Tensor) -> float:
    a = a.double()
    b = b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))
