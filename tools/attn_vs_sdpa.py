"""A/B of the attention kernels against torch's F.scaled_dot_product_attention (the reference's backend,
hf integrations/sdpa_attention.py:92-101) at the benchmark shape (8 sequences, 16 heads, 2048 events, head_dim 64,
causal, bf16), forward and backward, plus the token-level shape (16 384 events x 8 tokens, 4 heads of 256).
CUDA events, 3 warm-up + 20 launches.  Writes $MIDI_TOOLS_OUT/attn_vs_sdpa.json.

    python tools/attn_vs_sdpa.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from midi_b200 import ops  # noqa: E402

DEV, BF = "cuda", torch.bfloat16


def time_ms(fn, iters=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    g = torch.Generator(device=DEV).manual_seed(0)
    res = {}
    B, S, nh, D = 8, 2048, 16, 64
    H = nh * D
    qkv = torch.randn(B * S, 3 * H, generator=g, device=DEV).to(BF)
    do = torch.randn(B * S, H, generator=g, device=DEV).to(BF)
    o, lse = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True)
    q, k, v = (qkv.view(B, S, 3, nh, D)[:, :, i].transpose(1, 2).contiguous().requires_grad_(True) for i in range(3))
    do_t = do.view(B, S, nh, D).transpose(1, 2).contiguous()
    fl_f = 4 * B * nh * S * (S + 1) / 2 * D
    t = time_ms(lambda: ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True))
    t_ref = time_ms(lambda: F.scaled_dot_product_attention(q, k, v, is_causal=True))
    res["event_fwd"] = {"ours_ms": t, "sdpa_ms": t_ref, "ours_tflops": fl_f / t / 1e9, "sdpa_tflops": fl_f / t_ref / 1e9, "ratio": t_ref / t}
    t = time_ms(lambda: ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D))
    out_ref = F.scaled_dot_product_attention(q, k, v, is_causal=True)

    def ref_bwd():
        torch.autograd.grad(out_ref, (q, k, v), do_t, retain_graph=True)
    t_ref = time_ms(ref_bwd)
    res["event_bwd"] = {"ours_ms": t, "sdpa_ms": t_ref, "ours_tflops": 2.5 * fl_f / t / 1e9, "sdpa_tflops": 2.5 * fl_f / t_ref / 1e9, "ratio": t_ref / t}
    res["event_fwd_maxabs_vs_sdpa"] = float((o.view(B, S, nh, D).transpose(1, 2).float() - out_ref.float()).abs().max())
    del q, k, v, out_ref, qkv, do
    # token level: 16 384 events x 8 positions, 4 heads x 256 (what hf runs through SDPA as (N, 4, 8, 256))
    N, L, nh, D = 16384, 8, 4, 256
    H = nh * D
    qkv = torch.randn(N * L, 3 * H, generator=g, device=DEV).to(BF)
    do = torch.randn(N * L, H, generator=g, device=DEV).to(BF)
    q, k, v = (qkv.view(N, L, 3, nh, D)[:, :, i].transpose(1, 2).contiguous().requires_grad_(True) for i in range(3))
    t = time_ms(lambda: ops.attn_tiny_fwd(qkv, N, L, nh, D))
    t_ref = time_ms(lambda: F.scaled_dot_product_attention(q, k, v, is_causal=True))
    res["token_fwd"] = {"ours_ms": t, "sdpa_ms": t_ref, "ratio": t_ref / t}
    t = time_ms(lambda: ops.attn_tiny_bwd(qkv, do, N, L, nh, D))
    out_ref = F.scaled_dot_product_attention(q, k, v, is_causal=True)
    do_t = do.view(N, L, nh, D).transpose(1, 2).contiguous()
    t_ref = time_ms(lambda: torch.autograd.grad(out_ref, (q, k, v), do_t, retain_graph=True))
    res["token_bwd"] = {"ours_ms": t, "sdpa_ms": t_ref, "ratio": t_ref / t}
    for k_, v_ in res.items():
        print(k_, json.dumps(v_))
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "attn_vs_sdpa.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
