"""GPU parity checks: every sm_90a kernel (through the C ABI) against the fp32 PyTorch composite it
replaces, and the drop-in MIDIModel against the CPU oracle restatement run on the same device.
Each check returns {metric_name: value} and carries, from `bounded` above its definition, its bound table (metric-name
prefix -> bound) and the names of the metrics it reports without a bound.  test_gpu_parity.py asserts every check of
GROUPS with parity_metrics.check_bounds and tools/run_gpu_checks.py reports them.  Seeds are fixed; sizes are chosen
so the oracle finishes in seconds and so that odd / ragged shapes are covered (S=2047, V=3406, rows not /128, L<8,
empty)."""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

from midi_b200 import lib, ops  # noqa: E402
from oracle import midi_oracle as O  # noqa: E402

import gpu_model as GM  # noqa: E402
import parity_metrics as P  # noqa: E402
from host_model import global_rel, grads  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def randn(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV, dtype=torch.float32) * scale).to(dtype)


def bounded(bounds, info=()):
    """Gives a check its bound table (metric-name prefix -> bound, judged by parity_metrics.check_bounds) and the names
    of the metrics it reports without a bound."""
    def attach(check):
        check.bounds, check.info = bounds, info
        return check
    return attach


# ------------------------------------------------------------------------------------------ GEMM
@bounded([("gemm_vocab_padcols_absmax", 0.0), ("gemm_", 4e-3)])
def check_gemm_fwd():
    out = {}
    for i, (M, N, K) in enumerate([(256, 256, 128), (1000, 1024, 1024), (2048, 3072, 1024), (384, 8192, 1024),
                                   (4096, 1024, 4096), (130, 136, 72)]):
        a, w = randn(M, K, seed=i), randn(N, K, scale=0.05, seed=100 + i)
        y = ops.linear(a, w)
        ref = (a.float() @ w.float().T)
        out[f"gemm_tn_{M}x{N}x{K}"] = rel(y.float(), ref)
    # residual epilogue: bf16(bf16(acc) + r)
    M, N, K = 1024, 1024, 1024
    a, w, r = randn(M, K, seed=7), randn(N, K, scale=0.05, seed=8), randn(M, N, seed=9)
    y = ops.linear(a, w, residual=r)
    ref = ((a.float() @ w.float().T).to(BF).float() + r.float())
    out["gemm_residual"] = rel(y.float(), ref)
    # N = 3406 (vocab): pitch 3408, trailing columns zero
    a, w = randn(520, 1024, seed=11), randn(3406, 1024, scale=0.05, seed=12)
    y = ops.linear(a, w, pitch=3408)
    out["gemm_vocab"] = rel(y[:, :3406].float(), a.float() @ w.float().T)
    out["gemm_vocab_padcols_absmax"] = float(y[:, 3406:].float().abs().max())
    return out


@bounded([("gemm_swiglu", 0.0)])
def check_gemm_swiglu():
    """gate|up GEMM with SwiGLU in the epilogue == plain GEMM + stand-alone SwiGLU kernel, bit for bit."""
    out = {}
    for i, (M, I, K) in enumerate([(300, 1024, 1024), (2048, 4096, 1024), (1000, 128, 256)]):
        x, w = randn(M, K, seed=60 + i), randn(2 * I, K, scale=0.05, seed=70 + i)
        gu, act = ops.linear_swiglu(x, w)
        gu_ref = ops.linear(x, w)
        out[f"gemm_swiglu_gu_mismatch_{M}x{I}"] = float((gu != gu_ref).sum())
        out[f"gemm_swiglu_act_mismatch_{M}x{I}"] = float((act != ops.swiglu(gu_ref)).sum())
    return out


@bounded([("gemm_", 4e-3)])
def check_gemm_dgrad():
    out = {}
    for i, (M, N, K) in enumerate([(256, 256, 128), (1000, 3072, 1024), (2048, 1024, 4096), (520, 3406, 1024)]):
        pitch = (N + 7) // 8 * 8
        dy = torch.zeros(M, pitch, device=DEV, dtype=BF)
        dy[:, :N] = randn(M, N, seed=20 + i)
        w = randn(N, K, scale=0.05, seed=30 + i)
        dx = ops.linear_dgrad(dy, w)
        out[f"gemm_dgrad_{M}x{N}x{K}"] = rel(dx.float(), dy[:, :N].float() @ w.float())
    return out


@bounded([("gemm_", 4e-3)])
def check_gemm_wgrad():
    out = {}
    for i, (M, N, K) in enumerate([(256, 256, 128), (4096, 1024, 1024), (3000, 3072, 1024), (2048, 3406, 1024),
                                   (16384, 1024, 1024)]):
        pitch = (N + 7) // 8 * 8
        dy = torch.zeros(M, pitch, device=DEV, dtype=BF)
        dy[:, :N] = randn(M, N, seed=40 + i)
        x = randn(M, K, seed=50 + i)
        dw = torch.empty(N, K, device=DEV, dtype=BF)
        ops.linear_wgrad(dy, x, dw, accumulate=False)
        ref = dy[:, :N].float().T @ x.float()
        out[f"gemm_wgrad_{M}x{N}x{K}"] = rel(dw.float(), ref)
        if i == 1:
            ops.linear_wgrad(dy, x, dw, accumulate=True)
            out["gemm_wgrad_accumulate"] = rel(dw.float(), 2 * ref)
    return out


# ------------------------------------------------------------------------------------------ elementwise
@bounded([
    ("embed_sum_maxabs", 0.0), ("embed_bwd_padrow_absmax", 0.0), ("embed_bwd", 4e-3), ("inner_input_equal", 0.0),
    ("inner_embed_bwd", 4e-3), ("rmsnorm_fwd_mismatch", 2e-3), ("rmsnorm_fwd", 2e-3), ("rmsnorm_bwd", 4e-3),
    ("rope_table_mismatch", 8.0), ("rope_fwd_mismatch", 64.0), ("rope_bwd_adjoint", 2e-2),
    ("swiglu_fwd_mismatch", 2e-2), ("swiglu_bwd", 4e-3),
])
def check_elementwise():
    out = {}
    V, H = 3406, 1024
    table = randn(V, H, scale=0.02, seed=1)
    ids = torch.randint(0, V, (300, 8), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    ids[5] = 0
    y = ops.embed_sum(ids, table)
    ref = F.embedding(ids, table).float().sum(-2).to(BF)
    out["embed_sum_maxabs"] = float((y.float() - ref.float()).abs().max())
    # embedding backward (outer: 8 ids per gradient row; pad row zero)
    dout = randn(300, H, seed=3)
    dtab = torch.empty(V, H, device=DEV, dtype=BF)
    ops.embed_bwd(ids.view(-1), dout, dtab, per_row=8, row_stride=1, row_inner=0, row_off=0, pad_id=0, accumulate=False)
    t32 = table.float().clone().requires_grad_(True)
    F.embedding(ids, t32, padding_idx=0).sum(-2).backward(dout.float())
    out["embed_bwd"] = rel(dtab.float(), t32.grad)
    out["embed_bwd_padrow_absmax"] = float(dtab[0].float().abs().max())
    # inner input builder + its embedding backward (7 ids per event, rows e*8 + 1 + j)
    hid = randn(40, H, seed=4)
    ids7 = torch.randint(0, V, (40, 7), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    xin = ops.inner_input(hid, ids7, table)
    ref = torch.cat([hid[:, None], F.embedding(ids7, table)], 1).reshape(-1, H)
    out["inner_input_equal"] = float((xin != ref).sum())
    dx = randn(40 * 8, H, seed=6)
    ops.embed_bwd(ids7.view(-1), dx, dtab, per_row=7, row_stride=8, row_inner=1, row_off=1, pad_id=0, accumulate=False)
    t32 = table.float().clone().requires_grad_(True)
    F.embedding(ids7, t32, padding_idx=0).backward(dx.float().view(40, 8, H)[:, 1:])
    out["inner_embed_bwd"] = rel(dtab.float(), t32.grad)
    # rmsnorm
    for M in (1, 300, 5000):
        x, w = randn(M, H, seed=7), (1 + 0.1 * randn(H, seed=8).float()).to(BF)
        y, rstd = ops.rmsnorm(x, w, 1e-6, want_rstd=True)
        ref = O.rmsnorm(x, w, 1e-6)
        out[f"rmsnorm_fwd_mismatch_{M}"] = float((y != ref).float().mean())
        out[f"rmsnorm_fwd_{M}"] = rel(y.float(), ref.float())
        dy, dres = randn(M, H, seed=9), randn(M, H, seed=10)
        dw = torch.empty(H, device=DEV, dtype=BF)
        dx = ops.rmsnorm_bwd(dy, x, w, rstd, dres, dw, False)
        x32, w32 = x.float().requires_grad_(True), w.float().requires_grad_(True)
        v = x32.pow(2).mean(-1, keepdim=True)
        (w32 * (x32 * torch.rsqrt(v + 1e-6))).backward(dy.float())
        out[f"rmsnorm_bwd_dx_{M}"] = rel(dx.float(), x32.grad + dres.float())
        out[f"rmsnorm_bwd_dw_{M}"] = rel(dw.float(), w32.grad)
    # rope (bf16-rounded inv_freq, as after model.to(bf16)) on packed qkv
    for (S, nh, D) in ((37, 16, 64), (8, 4, 256)):
        Hh = nh * D
        inv = O.default_inv_freq(D).to(BF).to(DEV)
        cos, sin = ops.rope_table(inv, S)
        rc, rs = O.rope_cos_sin(inv, torch.arange(S, device=DEV), BF)
        out[f"rope_table_mismatch_D{D}"] = float((cos != rc[:, :D // 2]).sum() + (sin != rs[:, :D // 2]).sum())
        qkv = randn(3 * S, 3 * Hh, seed=11)
        q0 = qkv.clone()
        ops.rope_qk_(qkv, cos, sin, S, Hh, D)
        q = q0[:, :Hh].view(3, S, nh, D).transpose(1, 2)
        k = q0[:, Hh:2 * Hh].view(3, S, nh, D).transpose(1, 2)
        rq = O.apply_rope(q, rc, rs).transpose(1, 2).reshape(3 * S, Hh)
        rk = O.apply_rope(k, rc, rs).transpose(1, 2).reshape(3 * S, Hh)
        out[f"rope_fwd_mismatch_D{D}"] = float((qkv[:, :Hh] != rq).sum() + (qkv[:, Hh:2 * Hh] != rk).sum()
                                               + (qkv[:, 2 * Hh:] != q0[:, 2 * Hh:]).sum())
        # backward == transpose of the rotation: <R x, y> == <x, R^T y>
        d = randn(3 * S, 3 * Hh, seed=12)
        d_in = d.clone()
        ops.rope_qk_(d_in, cos, sin, S, Hh, D, backward=True)
        c32 = torch.cat([cos, cos], -1).float()
        s32 = torch.cat([sin, sin], -1).float()

        def rot32(t):
            t4 = t.float().view(3, S, nh, D)
            return (t4 * c32[None, :, None] + O.rotate_half(t4) * s32[None, :, None]).reshape(3 * S, Hh)
        lhs = (rot32(q0[:, :Hh]) * d[:, :Hh].float()).sum()
        rhs = (q0[:, :Hh].float() * d_in[:, :Hh].float()).sum()
        out[f"rope_bwd_adjoint_D{D}"] = float((lhs - rhs).abs() / lhs.abs().clamp_min(1e-6))
    # swiglu
    gu = randn(777, 2 * 1024, seed=13)
    act = ops.swiglu(gu)
    ref = F.silu(gu[:, :1024]) * gu[:, 1024:]
    out["swiglu_fwd_mismatch"] = float((act != ref).float().mean())
    dact = randn(777, 1024, seed=14)
    dgu = ops.swiglu_bwd(gu, dact)
    g32 = gu.float().requires_grad_(True)
    (F.silu(g32[:, :1024]) * g32[:, 1024:]).backward(dact.float())
    out["swiglu_bwd"] = rel(dgu.float(), g32.grad)
    return out


# ------------------------------------------------------------------------------------------ attention
def _sdpa_ref(q, k, v, off):
    # q (B,h,Sq,d) fp32; causal with offset
    Sq, Sk = q.shape[-2], k.shape[-2]
    s = q @ k.transpose(-1, -2) / math.sqrt(q.shape[-1])
    m = torch.arange(Sk, device=q.device)[None] > (torch.arange(Sq, device=q.device)[:, None] + off)
    s = s.masked_fill(m, float("-inf"))
    return torch.softmax(s, -1) @ v


@bounded([("flash_fwd", 6e-3), ("flash_lse", 1e-4), ("flash_bwd", 1.2e-2)])
def check_attn_flash():
    out = {}
    for (B, S, nh) in ((2, 64, 4), (1, 200, 16), (2, 2047, 16)):
        D, H = 64, nh * 64
        qkv = randn(B * S, 3 * H, seed=S)
        o, lse = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True, impl="mma")
        q32 = qkv.float().view(B, S, 3, nh, D).permute(2, 0, 3, 1, 4).clone().requires_grad_(True)
        ref = _sdpa_ref(q32[0], q32[1], q32[2], 0)
        out[f"flash_fwd_S{S}"] = rel(o.float().view(B, S, nh, D).transpose(1, 2), ref)
        sc = (q32[0] @ q32[1].transpose(-1, -2)) / 8.0
        msk = torch.triu(torch.ones(S, S, device=DEV, dtype=torch.bool), 1)
        out[f"flash_lse_S{S}"] = rel(lse, torch.logsumexp(sc.masked_fill(msk, float("-inf")), -1))
        do = randn(B * S, H, seed=S + 1)
        dqkv = ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D, impl="mma")
        ref.backward(do.float().view(B, S, nh, D).transpose(1, 2))
        g = q32.grad.permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
        out[f"flash_bwd_dq_S{S}"] = rel(dqkv[:, :H].float(), g[:, :H])
        out[f"flash_bwd_dk_S{S}"] = rel(dqkv[:, H:2 * H].float(), g[:, H:2 * H])
        out[f"flash_bwd_dv_S{S}"] = rel(dqkv[:, 2 * H:].float(), g[:, 2 * H:])
    return out


@bounded([("wg_vs_mma_bwd", 8e-3), ("wg_bwd", 1.2e-2), ("wg_vs_mma", 4e-3), ("wg_fwd", 6e-3)],
         info=("time_ms_bwd_wgmma", "time_ms_bwd_mma", "time_ms_wgmma", "tflops_wgmma", "time_ms_mma", "tflops_mma"))
def check_attn_wgmma():
    """wgmma / TMA attention (the training path) vs fp32 SDPA and vs the mma.sync kernels (same semantics)."""
    out = {}
    for (B, S, nh) in ((1, 128, 4), (2, 384, 16), (1, 200, 16), (2, 2047, 16), (8, 2048, 16)):
        D, H = 64, nh * 64
        qkv = randn(B * S, 3 * H, seed=S + B)
        o, lse = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True, impl="wgmma")
        o2, lse2 = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True, impl="mma")
        torch.cuda.synchronize()
        out[f"wg_vs_mma_fwd_B{B}_S{S}"] = rel(o.float(), o2.float())
        out[f"wg_vs_mma_lse_B{B}_S{S}"] = rel(lse, lse2)
        if B * S <= 4096:
            q32 = qkv.float().view(B, S, 3, nh, D).permute(2, 0, 3, 1, 4)
            ref = _sdpa_ref(q32[0], q32[1], q32[2], 0)
            out[f"wg_fwd_S{S}"] = rel(o.float().view(B, S, nh, D).transpose(1, 2), ref)
    # backward: wgmma kernels vs the mma.sync kernels and vs fp32 autograd
    for (B, S, nh) in ((1, 128, 4), (2, 384, 16), (1, 200, 16), (2, 2047, 16)):
        D, H = 64, nh * 64
        qkv = randn(B * S, 3 * H, seed=S + B + 7)
        do = randn(B * S, H, seed=S + B + 8)
        o, lse = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=True, impl="mma")
        g_wg = ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D, impl="wgmma")
        g_mm = ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D, impl="mma")
        torch.cuda.synchronize()
        out[f"wg_vs_mma_bwd_dq_S{S}"] = rel(g_wg[:, :H].float(), g_mm[:, :H].float())
        out[f"wg_vs_mma_bwd_dk_S{S}"] = rel(g_wg[:, H:2 * H].float(), g_mm[:, H:2 * H].float())
        out[f"wg_vs_mma_bwd_dv_S{S}"] = rel(g_wg[:, 2 * H:].float(), g_mm[:, 2 * H:].float())
        q32 = qkv.float().view(B, S, 3, nh, D).permute(2, 0, 3, 1, 4).clone().requires_grad_(True)
        _sdpa_ref(q32[0], q32[1], q32[2], 0).backward(do.float().view(B, S, nh, D).transpose(1, 2))
        g = q32.grad.permute(1, 3, 0, 2, 4).reshape(B * S, 3 * H)
        out[f"wg_bwd_S{S}"] = rel(g_wg.float(), g)
        # with the RoPE backward fused
        inv = O.default_inv_freq(D).to(BF).to(DEV)
        cos, sin = ops.rope_table(inv, S)
        a = ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D, rope=(cos, sin), impl="wgmma")
        bref = ops.attn_causal_bwd(qkv, o, do, lse, B, S, nh, D, rope=(cos, sin), impl="mma")
        out[f"wg_vs_mma_bwd_rope_S{S}"] = rel(a.float(), bref.float())
    # timing at the benchmark shape (B=8, S=2048, 16 heads): CUDA events, 10 launches each
    qkv = randn(8 * 2048, 3 * 1024, seed=1)
    do = randn(8 * 2048, 1024, seed=2)
    o, lse = ops.attn_causal_fwd(qkv, 8, 2048, 16, 64, want_lse=True, impl="mma")
    for impl in ("wgmma", "mma"):
        for _ in range(3):
            ops.attn_causal_bwd(qkv, o, do, lse, 8, 2048, 16, 64, impl=impl)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attn_causal_bwd(qkv, o, do, lse, 8, 2048, 16, 64, impl=impl)
        e1.record()
        torch.cuda.synchronize()
        out[f"time_ms_bwd_{impl}"] = e0.elapsed_time(e1) / 10
    for impl in ("wgmma", "mma"):
        for _ in range(3):
            ops.attn_causal_fwd(qkv, 8, 2048, 16, 64, want_lse=True, impl=impl)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attn_causal_fwd(qkv, 8, 2048, 16, 64, want_lse=True, impl=impl)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        out[f"time_ms_{impl}"] = ms
        out[f"tflops_{impl}"] = 4 * 8 * 16 * 2048 * 2049 / 2 * 64 / (ms * 1e-3) / 1e12
    return out


@bounded([("tiny_fwd", 6e-3), ("tiny_bwd", 1.2e-2)])
def check_attn_tiny():
    out = {}
    nh, D = 4, 256
    H = nh * D
    for (N, L) in ((50, 8), (33, 5), (7, 1)):
        qkv = randn(N * L, 3 * H, seed=L)
        o = ops.attn_tiny_fwd(qkv, N, L, nh, D)
        q32 = qkv.float().view(N, L, 3, nh, D).permute(2, 0, 3, 1, 4).clone().requires_grad_(True)
        ref = _sdpa_ref(q32[0], q32[1], q32[2], 0)
        out[f"tiny_fwd_L{L}"] = rel(o.float().view(N, L, nh, D).transpose(1, 2), ref)
        do = randn(N * L, H, seed=L + 1)
        dqkv = ops.attn_tiny_bwd(qkv, do, N, L, nh, D)
        ref.backward(do.float().view(N, L, nh, D).transpose(1, 2))
        g = q32.grad.permute(1, 3, 0, 2, 4).reshape(N * L, 3 * H)
        out[f"tiny_bwd_L{L}"] = rel(dqkv.float(), g)
    return out


@bounded([("linear_rope_mismatch", 0.0), ("tiny_fused_rope", 0.0), ("attn_bwd_fused_rope_v_mismatch", 0.0),
          ("attn_bwd_fused_rope", 5e-3)])
def check_fused_rope():
    """RoPE fused into the QKV GEMM epilogue (bit-identical to GEMM + stand-alone rope kernel: same rounding
    points, same accumulation order) and into the attention backward kernels (one rounding fewer)."""
    out = {}
    for (nseq, S, nh, D) in ((3, 200, 16, 64), (40, 8, 4, 256)):
        H = nh * D
        inv = O.default_inv_freq(D).to(BF).to(DEV)
        cos, sin = ops.rope_table(inv, S)
        x, w = randn(nseq * S, 1024, seed=S), randn(3 * H, 1024, scale=0.05, seed=S + 1)
        fused = ops.linear_rope(x, w, cos, sin, S, D)
        ref = ops.linear(x, w)
        ops.rope_qk_(ref, cos, sin, S, H, D)
        out[f"linear_rope_mismatch_D{D}"] = float((fused != ref).sum())
        # backward: attention bwd with fused inverse rotation vs attention bwd + stand-alone rope backward
        do = randn(nseq * S, H, seed=S + 2)
        if D == 64:
            o, lse = ops.attn_causal_fwd(ref, nseq, S, nh, D, want_lse=True)
            a = ops.attn_causal_bwd(ref, o, do, lse, nseq, S, nh, D, rope=(cos, sin))
            b = ops.attn_causal_bwd(ref, o, do, lse, nseq, S, nh, D)
        else:
            a = ops.attn_tiny_bwd(ref, do, nseq, S, nh, D, rope=(cos, sin))
            b = ops.attn_tiny_bwd(ref, do, nseq, S, nh, D)
        ops.rope_qk_(b, cos, sin, S, H, D, backward=True)
        out[f"attn_bwd_fused_rope_D{D}"] = rel(a.float(), b.float())
        out[f"attn_bwd_fused_rope_v_mismatch_D{D}"] = float((a[:, 2 * H:] != b[:, 2 * H:]).sum())
        if D == 256:   # forward: RoPE fused into the token-level attention kernel (in-place rotation) == rope kernel + attention
            pre = ops.linear(x, w)
            o_f = ops.attn_tiny_fwd(pre, nseq, S, nh, D, rope=(cos, sin))
            o_r = ops.attn_tiny_fwd(ref, nseq, S, nh, D)
            out["tiny_fused_rope_out_mismatch"] = float((o_f != o_r).sum())
            out["tiny_fused_rope_qkv_mismatch"] = float((pre != ref).sum())
    return out


# ------------------------------------------------------------------------------------------ loss / optimizer
@bounded([
    ("ce_loss_abs", 2e-3), ("ce_count_abs", 0.0), ("ce_bwd_padcols_absmax", 0.0), ("ce_bwd", 6e-3),
    ("ce_all_ignored_loss", 0.0), ("gradnorm_rel", 1e-4), ("adamw_maxabs", 2e-3),
])
def check_loss_optim():
    out = {}
    V, pitch, R = 3406, 3408, 1000
    logits = torch.zeros(R, pitch, device=DEV, dtype=BF)
    logits[:, :V] = randn(R, V, scale=2.0, seed=1)
    tg = torch.randint(0, V, (R,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    tg[::5] = 0
    lac, lse = ops.ce_fwd(logits, tg, V, 0)
    l32 = logits[:, :V].float().requires_grad_(True)
    ref = F.cross_entropy(l32, tg, ignore_index=0)
    out["ce_loss_abs"] = float((lac[0] - ref).abs())
    out["ce_count_abs"] = float((lac[1] - (tg != 0).sum()).abs())
    ref.backward()
    ops.ce_bwd_(logits, tg, lse, lac, V, 0, 1.0)
    out["ce_bwd"] = rel(logits[:, :V].float(), l32.grad)
    out["ce_bwd_padcols_absmax"] = float(logits[:, V:].float().abs().max())
    # all-ignored rows -> loss 0, zero grads
    tg0 = torch.zeros(R, dtype=torch.long, device=DEV)
    lac0, _ = ops.ce_fwd(logits, tg0, V, 0)
    out["ce_all_ignored_loss"] = float(lac0[0].abs())
    # AdamW + clip vs torch.optim.AdamW (fp32 reference on the bf16-rounded values)
    n = 256 * 1000
    p = randn(n, scale=0.05, seed=3)
    g = randn(n, scale=0.5, seed=4)
    nodecay = torch.zeros(n // 256, dtype=torch.uint8, device=DEV)
    nodecay[500:] = 1
    pr = p.float().clone()
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    nc = torch.zeros(2, device=DEV)
    ws = torch.empty(lib.query("b200_gradnorm_parts") * 4, dtype=torch.uint8, device=DEV)
    pa = torch.nn.Parameter(pr[: 500 * 256].clone())
    pb = torch.nn.Parameter(pr[500 * 256:].clone())
    opt = torch.optim.AdamW([dict(params=[pa], weight_decay=0.01), dict(params=[pb], weight_decay=0.0)], lr=1e-3,
                            betas=(0.9, 0.99), eps=1e-8)
    pcur = p.clone()
    for step in (1, 2, 3):
        lib.call("b200_grad_clip_coef", g.data_ptr(), n, 1.0, nc.data_ptr(), ws.data_ptr(), ws.numel(), lib.stream())
        lib.call("b200_adamw_step", pcur.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), nodecay.data_ptr(), n, 1e-3,
                 0.9, 0.99, 1e-8, 0.01, step, nc.data_ptr(), lib.stream())
        pa.grad = g.float()[: 500 * 256].clone()
        pb.grad = g.float()[500 * 256:].clone()
        torch.nn.utils.clip_grad_norm_([pa, pb], 1.0)
        opt.step()
        # the kernel rounds the parameter to bf16 each step; mirror that in the reference
        with torch.no_grad():
            pa.copy_(pa.to(BF).float())
            pb.copy_(pb.to(BF).float())
    out["gradnorm_rel"] = float((nc[0] - g.float().norm()).abs() / g.float().norm())
    out["adamw_maxabs"] = float((pcur.float() - torch.cat([pa, pb]).detach()).abs().max())
    return out


# ------------------------------------------------------------------------------------------ decode kernels
@bounded([("sampler_greedy_mismatch", 0.0), ("logits_sampler_", 0.0), ("sampler_topk_outside", 0.0),
          ("sampler_dist_l1", 0.12)])
def check_decode():
    out = {}
    from midi_b200 import decode as dec
    # (the skinny projections and the paged KV append / attention are scored per element / per row by the gemv_matrix
    # and decode_attn_edges groups)
    # sampler: greedy == argmax; top-k support; distribution sanity
    V = 3406
    g = torch.Generator(device=DEV).manual_seed(5)
    probs = torch.softmax(torch.randn(64, V, generator=g, device=DEV) * 3, -1)
    mask = torch.zeros(V, device=DEV)
    mask[9:137] = 1
    probs = (probs * mask)
    u = torch.rand(64, generator=g, device=DEV)
    o1 = torch.empty(64, dtype=torch.long, device=DEV)
    lib.call("b200_sample_topp_topk", probs.data_ptr(), 0, 64, V, V, 0.98, 1, u.data_ptr(), o1.data_ptr(), lib.stream())
    out["sampler_greedy_mismatch"] = float((o1 != probs.argmax(-1)).sum())
    lib.call("b200_sample_topp_topk", probs.data_ptr(), 0, 64, V, V, 0.98, 20, u.data_ptr(), o1.data_ptr(), lib.stream())
    top20 = probs.topk(20, -1).indices
    out["sampler_topk_outside"] = float((~(top20 == o1[:, None]).any(-1)).sum())
    # fused logits sampler (temperature softmax + grammar range + top-p/top-k) incl. the histogram top-k preselection:
    # greedy == argmax inside the allowed range, top-20 draws stay inside the 20 largest, for narrow and 2048-wide ranges
    from midi_b200.tokenizer_tables import TokenizerTables
    tokz = TokenizerTables("v2")
    glut = dec.GrammarLUT(tokz, DEV)
    logits = torch.zeros(64, 3408, device=DEV, dtype=BF)
    logits[:, :V] = (torch.randn(64, V, generator=g, device=DEV) * 2.5).to(BF)
    uu = torch.rand(64, generator=g, device=DEV)
    ev = torch.full((64,), tokz.event_ids["note"], dtype=torch.long, device=DEV)
    for step, pname in ((1, "time1"), (7, "duration"), (5, "pitch")):
        lo, hi = tokz.parameter_ids[pname][0], tokz.parameter_ids[pname][-1] + 1
        outb = torch.zeros(64, 8, dtype=torch.long, device=DEV)
        dec.sample_from_logits(logits, V, 1.0, 0.98, 1, step, ev, glut, uu, outb)
        ref_arg = logits[:, lo:hi].float().argmax(-1) + lo
        pr = torch.softmax(logits[:, :V].float(), -1).to(BF)
        # ties in bf16 probabilities are broken towards the lowest id: compare probabilities, not ids
        got = outb[:, step]
        out[f"logits_sampler_greedy_{pname}"] = float((pr.gather(1, got[:, None]) != pr.gather(1, ref_arg[:, None])).sum()
                                                       + ((got < lo) | (got >= hi)).sum())
        dec.sample_from_logits(logits, V, 1.0, 1.0, 20, step, ev, glut, uu, outb)
        got = outb[:, step]
        kth = pr[:, lo:hi].float().topk(20, -1).values[:, -1]
        out[f"logits_sampler_top20_{pname}"] = float((pr.gather(1, got[:, None])[:, 0].float() < kth).sum()
                                                      + ((got < lo) | (got >= hi)).sum())
    # empirical distribution of one row vs the reference algorithm's renormalised top-p/top-k weights
    row = probs[:1].repeat(4096, 1).contiguous()
    u = torch.rand(4096, generator=g, device=DEV)
    o2 = torch.empty(4096, dtype=torch.long, device=DEV)
    lib.call("b200_sample_topp_topk", row.data_ptr(), 0, 4096, V, V, 0.9, 8, u.data_ptr(), o2.data_ptr(), lib.stream())
    ps, pi = torch.sort(probs[0], descending=True)
    cs = torch.cumsum(ps, 0)
    ps = torch.where(cs - ps > 0.9, torch.zeros_like(ps), ps)
    ps[8:] = 0
    ps = ps / ps.sum()
    want = torch.zeros(V, device=DEV).scatter(0, pi, ps)
    emp = torch.bincount(o2, minlength=V).float() / 4096
    out["sampler_dist_l1"] = float((emp - want).abs().sum())
    return out


# ------------------------------------------------------------------------------------------ model level
def _sd(model, dtype, device=DEV):
    return {k: v.detach().to(device=device, dtype=dtype) for k, v in model.state_dict().items()}


@bounded([
    ("min:inv_freq_is_bf16", 1.0), ("margin_filtered_argmax_mismatch", 0.0), ("hidden_new_vs_oracle16", 3e-2),
    ("logits_new_vs_oracle16", 4e-2), ("logits_teacher_forced_vs_oracle16", 2e-2),
    ("hidden_new_vs_fp32_minus_1.25x_floor", 0.0), ("logits_new_vs_fp32_minus_1.25x_floor", 0.0),
], info=("hidden_new_vs_fp32", "hidden_oracle16_vs_fp32", "logits_new_vs_fp32", "logits_oracle16_vs_fp32",
         "argmax_agree_new_fp32", "argmax_agree_oracle16_fp32", "margin_filtered_fraction"))
def check_model_forward():
    """forward + forward_token logits vs the oracle (fp32 and bf16 on the same device): noise-floor protocol
    (per-layer teacher-forced bounds, end to end against the oracle's own bf16-vs-fp32 distance)."""
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    sd32 = _sd(model, torch.float32)
    model = model.to(DEV, dtype=BF).eval()
    sd16 = _sd(model, BF)
    inv_n = model.net.rotary_emb.inv_freq
    inv_t = model.net_token.rotary_emb.inv_freq
    out["inv_freq_is_bf16"] = float(inv_n.dtype == BF)
    batch = synth_batch(model.tokenizer, 2, 130, seed=1234).to(DEV)
    x, y = batch[:, :-1], batch[:, 1:]
    with torch.no_grad():
        h = model.forward(x)
        lg = model.forward_token(h.reshape(-1, 1024), y.reshape(-1, 8)[:, :-1])
        h32 = O.forward(sd32, ocfg, x)
        l32 = O.forward_token(sd32, ocfg, h32.reshape(-1, 1024), y.reshape(-1, 8)[:, :-1])
        h16 = O.forward(sd16, ocfg, x, inv_freq=inv_n)
        l16 = O.forward_token(sd16, ocfg, h16.reshape(-1, 1024), y.reshape(-1, 8)[:, :-1], inv_freq=inv_t)
    out["hidden_new_vs_fp32"] = rel(h.float(), h32)
    out["hidden_oracle16_vs_fp32"] = rel(h16.float(), h32)
    out["hidden_new_vs_oracle16"] = rel(h.float(), h16.float())
    out["logits_new_vs_fp32"] = rel(lg.float(), l32)
    out["logits_oracle16_vs_fp32"] = rel(l16.float(), l32)
    out["logits_new_vs_oracle16"] = rel(lg.float(), l16.float())
    out["argmax_agree_new_fp32"] = float((lg.float().argmax(-1) == l32.argmax(-1)).float().mean())
    out["argmax_agree_oracle16_fp32"] = float((l16.float().argmax(-1) == l32.argmax(-1)).float().mean())
    # teacher-forced greedy ids: wherever the fp32 oracle's top-1 margin exceeds the bf16 noise floor by a wide
    # factor, the argmax must agree exactly)
    top2 = l32.topk(2, -1).values
    margin = top2[..., 0] - top2[..., 1]
    noise = float((l16.float() - l32).abs().max())
    sel = margin > 4 * noise
    out["margin_filtered_fraction"] = float(sel.float().mean())
    out["margin_filtered_argmax_mismatch"] = float((lg.float().argmax(-1)[sel] != l32.argmax(-1)[sel]).sum())
    # teacher-forced inner stack: feed the oracle's bf16 hidden
    with torch.no_grad():
        lg_tf = model.forward_token(h16.reshape(-1, 1024), y.reshape(-1, 8)[:, :-1])
    out["logits_teacher_forced_vs_oracle16"] = rel(lg_tf.float(), l16.float())
    # the bf16 oracle's own distance to fp32 is the noise floor: this implementation may sit at most 1.25x as far
    for t in ("hidden", "logits"):
        out[f"{t}_new_vs_fp32_minus_1.25x_floor"] = out[f"{t}_new_vs_fp32"] - 1.25 * out[f"{t}_oracle16_vs_fp32"]
    return out


@bounded([("outer_layer_tf", 6e-3), ("inner_layer_tf", 6e-3)])
def check_model_layer_teacher_forced():
    """One decoder layer at a time, fed the oracle's own bf16 input (tier 1: <= 1e-3 on GEMM-dominated ops)."""
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).eval()
    sd16 = _sd(model, BF)
    rt = model._rt()
    B, S = 2, 96
    x_in = randn(B * S, 1024, seed=3)
    # oracle: a 1-layer stack built from layer 0's weights
    one = O.StackCfg("net", 1, 16, 1024, 4096)
    inv = model.net.rotary_emb.inv_freq
    sd1 = {k: v for k, v in sd16.items() if k.startswith("net.layers.0.") or k == "net.norm.weight"}
    with torch.no_grad():
        ref = O.llama_stack(sd1, one, x_in.view(B, S, 1024), inv)
    eng = rt.outer
    keep = eng.layers
    eng.layers = keep[:1]
    y, _ = eng.forward(x_in, B, S, inv, save=False)
    eng.layers = keep
    out["outer_layer_tf"] = rel(y.float().view(B, S, 1024), ref.float())
    one_t = O.StackCfg("net_token", 1, 4, 1024, 1024)
    sd1 = {k: v for k, v in sd16.items() if k.startswith("net_token.layers.0.") or k == "net_token.norm.weight"}
    inv_t = model.net_token.rotary_emb.inv_freq
    x_in = randn(64 * 8, 1024, seed=4)
    with torch.no_grad():
        ref = O.llama_stack(sd1, one_t, x_in.view(64, 8, 1024), inv_t)
    eng = rt.inner
    keep = eng.layers
    eng.layers = keep[:1]
    y, _ = eng.forward(x_in, 64, 8, inv_t, save=False)
    eng.layers = keep
    out["inner_layer_tf"] = rel(y.float().view(64, 8, 1024), ref.float())
    return out


SAMPLE_SEQ_LOSS_ABS, SAMPLE_SEQ_GRAD_REL = 5e-2, 6e-2
INT16_PATH_GRAD_REL = 1e-3


@bounded([
    ("sample_seq_loss_abs", SAMPLE_SEQ_LOSS_ABS), ("sample_seq_grad_global_rel", SAMPLE_SEQ_GRAD_REL),
    ("loss_abs", 3e-2), ("grad_global_rel", 6e-2), ("grad_pad_row", 0.0), ("autograd_loss_abs", 5e-2),
    ("autograd_grad_global_rel", 6e-2), ("min:lazy_ce_hits", 1.0), ("xy_split_mismatch", 0.0), ("prefetch_mismatch", 0.0),
    ("int16_path_loss_mismatch", 0.0), ("int16_path_grad_rel", INT16_PATH_GRAD_REL),
], info=("loss_ref", "grad_worst_rel"))
def check_model_train():
    """Fused loss + all gradients vs the oracle under torch autograd (fp32 weights = the bf16 weights upcast)."""
    import midi_model as mm
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    batch = synth_batch(model.tokenizer, 2, 66, seed=77, pad_tail=3).to(DEV)
    sd = {k: v.detach().float().requires_grad_(True) for k, v in model.state_dict().items()}
    ref = O.train_loss(sd, ocfg, batch)
    ref.backward()
    loss = model.training_loss(batch)
    out["loss_abs"] = float((loss - ref.detach()).abs())
    out["loss_ref"] = float(ref.detach())
    fused = grads(model)
    sd_grads = {n: sd[n].grad for n in fused}
    out["grad_global_rel"] = global_rel(fused, sd_grads)
    worst_name = max(fused, key=lambda n: rel(fused[n].float(), sd_grads[n]))
    out["grad_worst_rel"] = rel(fused[worst_name].float(), sd_grads[worst_name])
    print("worst grad tensor:", worst_name, out["grad_worst_rel"])
    out["grad_pad_row_outer"] = float(model.net.embed_tokens.weight.grad[0].float().abs().max())
    out["grad_pad_row_inner"] = float(model.net_token.embed_tokens.weight.grad[0].float().abs().max())
    # autograd (drop-in) path == fused path
    for p in model.parameters():
        p.grad = None
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
    hits0 = mm.LAZY_CE_HITS
    hidden = model.forward(x)
    hidden = hidden.reshape(-1, hidden.shape[-1])
    yy = y.reshape(-1, y.shape[-1])
    logits = model.forward_token(hidden, yy[:, :-1])
    l2 = F.cross_entropy(logits.view(-1, model.tokenizer.vocab_size), yy.view(-1), reduction="mean",
                         ignore_index=model.tokenizer.pad_id)
    l2.backward()
    out["lazy_ce_hits"] = float(mm.LAZY_CE_HITS - hits0)          # the reference's loss expression hit the fused CE (8 f2)
    out["autograd_loss_abs"] = float((l2.float() - ref.detach()).abs())
    out["autograd_grad_global_rel"] = global_rel(grads(model), sd_grads)
    # int16 host data path (midi_b200/data.py): device-side widening + x/y split, prefetcher, same loss bit for bit
    from midi_b200 import data as hostdata
    b16 = hostdata.collate(list(batch.cpu().numpy()), pad_id=model.tokenizer.pad_id)
    xs, ys = ops.batch_to_xy(b16.to(DEV))
    out["xy_split_mismatch"] = float((xs.view(2, -1, 8) != batch[:, :-1]).sum() + (ys.view(2, -1, 8) != batch[:, 1:]).sum())
    fed = list(hostdata.Prefetcher([b16, b16, b16], DEV))
    out["prefetch_mismatch"] = float(sum((f.to(torch.long) != batch).sum() for f in fed)) + abs(len(fed) - 3)
    for p in model.parameters():
        p.grad = None
    loss16 = model.training_loss(fed[0])
    out["int16_path_loss_mismatch"] = float((loss16 - loss).abs())
    # (gradients: the backward accumulates dQ / embedding rows with fp32 reductions whose order is not fixed -> rel. error)
    out["int16_path_grad_rel"] = global_rel(grads(model), fused)
    tok = model.tokenizer
    # --sample-seq (train.py:172-175): forward_token on a random subset of event rows, gradients through the fancy index
    for p_ in model.parameters():
        p_.grad = None
    tb = synth_batch(tok, 2, 130, seed=5).to(DEV)
    xx, yy = tb[:, :-1].contiguous(), tb[:, 1:].contiguous()
    rand_idx = GM.rand_idx(yy.shape[1])
    hidden = model.forward(xx)[:, rand_idx]
    ys = yy[:, rand_idx].reshape(-1, 8)
    lg = model.forward_token(hidden.reshape(-1, 1024), ys[:, :-1])
    l_s = F.cross_entropy(lg.view(-1, tok.vocab_size), ys.reshape(-1), reduction="mean", ignore_index=tok.pad_id)
    l_s.backward()
    g_new = grads(model)
    sdg = {k_: v_.detach().float().requires_grad_(True) for k_, v_ in model.state_dict().items()}
    h_o = O.forward(sdg, ocfg, xx, inv_freq=model.net.rotary_emb.inv_freq)[:, rand_idx]
    l_o = F.cross_entropy(O.forward_token(sdg, ocfg, h_o.reshape(-1, 1024), ys[:, :-1], inv_freq=model.net_token.rotary_emb.inv_freq).view(-1, tok.vocab_size), ys.reshape(-1),
                          reduction="mean", ignore_index=tok.pad_id)
    l_o.backward()
    out["sample_seq_loss_abs"] = float((l_s.float() - l_o.detach()).abs())
    out["sample_seq_grad_global_rel"] = global_rel(g_new, {n_: sdg[n_].grad for n_ in g_new})
    return out


@bounded([
    ("cached_vs_full_hidden", 3e-2), ("inner_cached_vs_full_logits", 3e-2), ("min:greedy_token_agree", 0.6),
    ("min:greedy_persist_vs_graph_agree", 0.6), ("sampled_invalid_events", 0.0), ("greedy_graph_vs_nograph_mismatch", 0.0),
    ("fused_decode_mismatch", 0.0), ("fused_lm_head_mismatch", 0.0),
], info=("greedy_len_new", "greedy_len_ref", "greedy_eager_vs_graph_agree"))
def check_model_generate():
    """Greedy (top_k=1) generate and the KV-cached forward vs the oracle."""
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).eval()
    sd16 = _sd(model, BF)
    tok = model.tokenizer
    batch = synth_batch(tok, 2, 40, seed=5).to(DEV)
    from transformers import DynamicCache
    with torch.no_grad():
        full = model.forward(batch)
        c = DynamicCache()
        parts = [model.forward(batch[:, :17], cache=c), model.forward(batch[:, 17:18], cache=c),
                 model.forward(batch[:, 18:23], cache=c)]
        for t in range(23, 40):
            parts.append(model.forward(batch[:, t:t + 1], cache=c))
    out["cached_vs_full_hidden"] = rel(torch.cat(parts, 1).float(), full.float())
    # fused single-token decode step (norm+QKV, RoPE+append+attention, ..., 5 launches/layer) == unfused kernels, bit for bit
    from midi_b200 import decode as dec
    outs = {}
    for fused in (True, False):
        dec.FUSED_DECODE = fused
        with torch.no_grad():
            c = DynamicCache()
            hs = [model.forward(batch[:, :17], cache=c)]
            for t in range(17, 30):
                hs.append(model.forward(batch[:, t:t + 1], cache=c))
        outs[fused] = torch.cat(hs, 1)
    dec.FUSED_DECODE = True
    out["fused_decode_mismatch"] = float((outs[True] != outs[False]).sum())
    # final norm fused into the lm_head GEMV == rmsnorm kernel + GEMV
    rt = model._rt()
    xpre = randn(4, 1024, seed=9)
    a = dec._gemv_fused(xpre, rt.lm_head, rt.V, norm_w=rt.inner.norm, eps=1e-6, ldy=rt.pitch)[:, :rt.V]
    bref = dec._lm_head(ops.rmsnorm(xpre, rt.inner.norm, 1e-6), rt.lm_head, rt.pitch)[:, :rt.V]
    out["fused_lm_head_mismatch"] = float((a != bref).sum())
    # inner cached path vs uncached logits
    with torch.no_grad():
        hid = full[:, -1]
        ids = batch[:, -1, :7]
        lg = model.forward_token(hid, ids)
        c2 = DynamicCache()
        steps = [model.forward_token(hid, None, cache=c2)]
        for i in range(7):
            steps.append(model.forward_token(None, ids[:, i:i + 1], cache=c2))
    out["inner_cached_vs_full_logits"] = rel(torch.cat(steps, 1).float(), lg.float())
    # greedy generate vs oracle generate (bf16 oracle on the same device), teacher-free
    prompt = batch[:, :6].cpu().numpy()
    ids_new = model.generate(prompt=prompt, batch_size=2, max_len=14, top_k=1, generator=torch.Generator(DEV).manual_seed(0))
    ids_ref = O.generate(sd16, ocfg, tok, prompt, batch_size=2, max_len=14, top_k=1,
                         inv_freq_net=model.net.rotary_emb.inv_freq, inv_freq_tok=model.net_token.rotary_emb.inv_freq)
    n = min(ids_new.shape[1], ids_ref.shape[1])
    out["greedy_len_new"], out["greedy_len_ref"] = float(ids_new.shape[1]), float(ids_ref.shape[1])
    out["greedy_token_agree"] = float((ids_new[:, :n] == ids_ref[:, :n]).mean())
    # the CUDA-graph loop and the host-driven loop run the same kernels: identical greedy ids
    os.environ["B200_GENERATE"] = "eager"
    ids_eager = model.generate(prompt=prompt, batch_size=2, max_len=14, top_k=1, generator=torch.Generator(DEV).manual_seed(0))
    os.environ["B200_GENERATE"] = "nograph"
    ids_ng = model.generate(prompt=prompt, batch_size=2, max_len=14, top_k=1, generator=torch.Generator(DEV).manual_seed(0))
    os.environ["B200_GENERATE"] = "graph"
    ids_graph = model.generate(prompt=prompt, batch_size=2, max_len=14, top_k=1, generator=torch.Generator(DEV).manual_seed(0))
    os.environ.pop("B200_GENERATE")               # default again: the persistent kernel (what ids_new was generated with)
    out["greedy_graph_vs_nograph_mismatch"] = float((ids_graph != ids_ng).sum()) if ids_graph.shape == ids_ng.shape else 1e9
    # persistent kernel vs launch-per-phase loop on flat random-init logits: same arithmetic except the attention's
    # summation order, so near-ties may flip -> agreement fraction here, bit-equality on the peaked checkpoints
    out["greedy_persist_vs_graph_agree"] = float((ids_new == ids_graph).mean()) if ids_new.shape == ids_graph.shape else 0.0
    # (graph replay == the same launches issued from the host; the host-driven loop prefills the last prompt event
    #  with the flash kernel instead of the decode kernel, so on these flat random-init logits it may pick other
    #  near-ties -- it is held to bit-equality on the peaked checkpoint instead, see check_model_peaked_greedy)
    out["greedy_eager_vs_graph_agree"] = float((ids_new == ids_eager).mean()) if ids_new.shape == ids_eager.shape else 0.0
    # grammar validity of sampled generation
    ids_s = model.generate(prompt=None, batch_size=4, max_len=24, generator=torch.Generator(DEV).manual_seed(1))
    bad = 0
    for row in ids_s[:, 1:].reshape(-1, 8):          # skip the BOS event of every row
        if row[0] == tok.eos_id or row[0] == tok.pad_id:
            continue
        if tok.tokens2event(row.tolist()) == []:
            bad += 1
    out["sampled_invalid_events"] = float(bad)
    return out


def _song_batch(tok, B, n_events, seed, fixed_step=3):
    """Deterministic grammar-valid 'songs': bos, one patch_change, then
    notes walking up a scale.  Learnable in a few hundred steps => large top-1 margins, no EOS."""
    rng = np.random.default_rng(seed)
    out = np.zeros((B, n_events, 8), dtype=np.int64)
    for b in range(B):
        ch, step, pitch = int(rng.integers(0, 4)), int(rng.integers(1, 6)), int(rng.integers(40, 80))
        if fixed_step:
            step = fixed_step      # continuation is then a deterministic function of the previous event
        rows = [[tok.bos_id] + [0] * 7, tok.event2tokens(["patch_change", 0, 0, 1, ch, int(rng.integers(0, 128))])]
        k = 0
        while len(rows) < n_events:
            rows.append(tok.event2tokens(["note", 1 if k % 4 == 0 else 0, (4 * k) % 16, 1, ch, pitch, 80, 4]))
            pitch = 40 + ((pitch - 40 + step) % 40)
            k += 1
        out[b] = np.asarray(rows)
    return torch.from_numpy(out)


@bounded([
    ("peaked_persist_vs_graph_mismatch", 0.0), ("stream_vs_generate_mismatch", 0.0), ("stream_masked_mismatch", 0.0),
    ("stream_denied_ids_emitted", 0.0), ("stream_mask_leak_mismatch", 0.0), ("stream_concurrent_errors", 0.0),
    ("stream_concurrent_mismatch", 0.0), ("stream_resumed_on_other_thread_mismatch", 0.0), ("peaked_greedy_mismatch", 0.0),
    ("peaked_eager_vs_graph_mismatch", 0.0), ("peaked_invalid_events", 0.0), ("peaked_loss_last", 1.5),
    ("peaked_argmax_mismatch_vs_oracle16", 0.0), ("peaked_logits_vs_fp32", 3e-2),
], info=("peaked_loss_first", "peaked_len_new", "peaked_len_ref", "peaked_first_divergence_event",
         "peaked_first_divergence_margin", "peaked_min_top1_margin_fp32",
         "stream_masked_differs_from_plain", "peaked_argmax_mismatch_vs_fp32",
         "peaked_argmax_oracle16_diff_vs_fp32"))
def check_model_peaked_greedy():
    """Train a 4-layer full-width model with the FUSED sm_90a trainer until it has learnt the token grammar,
    then free-running greedy generate must be bit-identical to the oracle's (bf16, same weights), and the loss
    curve must fall (exercises fwd+bwd+clip+AdamW end to end)."""
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    tok = model.tokenizer
    losses = []
    for step in range(1, 241):
        batch = _song_batch(tok, 16, 66, seed=step).to(DEV)
        loss = model.training_loss(batch)
        model.fused_optimizer_step(lr=3e-4 * min(1.0, step / 20), step=step, weight_decay=0.01)
        if step % 20 == 0 or step == 1:
            losses.append(float(loss))
    print("peaked training losses:", [round(x, 3) for x in losses])
    out["peaked_loss_first"], out["peaked_loss_last"] = losses[0], losses[-1]
    model.eval()
    sd16 = _sd(model, BF)
    prompt = _song_batch(tok, 4, 9, seed=999).numpy()
    ids_new = model.generate(prompt=prompt, batch_size=4, max_len=40, top_k=1)          # default: persistent kernel
    os.environ["B200_GENERATE"] = "eager"
    ids_eager = model.generate(prompt=prompt, batch_size=4, max_len=40, top_k=1)        # host-driven loop
    os.environ["B200_GENERATE"] = "graph"
    ids_graph = model.generate(prompt=prompt, batch_size=4, max_len=40, top_k=1)        # CUDA-graph loop
    os.environ.pop("B200_GENERATE")
    out["peaked_eager_vs_graph_mismatch"] = float((ids_eager != ids_graph).sum()) if ids_eager.shape == ids_graph.shape else 1e9
    out["peaked_persist_vs_graph_mismatch"] = float((ids_new != ids_graph).sum()) if ids_new.shape == ids_graph.shape else 1e9
    ids_ref = O.generate(sd16, ocfg, tok, prompt, batch_size=4, max_len=40, top_k=1,
                         inv_freq_net=model.net.rotary_emb.inv_freq, inv_freq_tok=model.net_token.rotary_emb.inv_freq)
    out["peaked_len_new"], out["peaked_len_ref"] = float(ids_new.shape[1]), float(ids_ref.shape[1])
    n = min(ids_new.shape[1], ids_ref.shape[1])
    neq = ids_new[:, :n] != ids_ref[:, :n]
    out["peaked_greedy_mismatch"] = float(neq.sum()) + abs(ids_new.shape[1] - ids_ref.shape[1])
    # tie / margin audit): if the runs diverge, the first differing token must be one where
    # the fp32 oracle's margin between the two candidates is within the bf16 noise
    sd32a = {k: v.float() for k, v in sd16.items()}
    ref_t = torch.from_numpy(ids_ref).to(DEV)
    with torch.no_grad():
        h32a = O.forward(sd32a, ocfg, ref_t[:, :-1])
        l32a = O.forward_token(sd32a, ocfg, h32a.reshape(-1, 1024), ref_t[:, 1:].reshape(-1, 8)[:, :-1]).view(4, n - 1, 8, -1)
    if neq.any():
        first_e = int(np.argwhere(neq.any(-1).any(0))[0][0])
        bs, ts = np.nonzero(neq[:, first_e])
        b0, t0 = int(bs[0]), int(ts[0])
        row = l32a[b0, first_e - 1, t0]
        out["peaked_first_divergence_event"] = float(first_e)
        out["peaked_first_divergence_margin"] = float((row[ids_ref[b0, first_e, t0]] - row[ids_new[b0, first_e, t0]]).abs())
        print("first divergence at event", first_e, "row", b0, "token", t0, "ref", ids_ref[b0, first_e], "new", ids_new[b0, first_e])
    top2 = l32a[:, 8:].topk(2, -1).values
    out["peaked_min_top1_margin_fp32"] = float((top2[..., 0] - top2[..., 1])[ref_t[:, 9:] != 0].min())
    # app.py's streaming loop: same events as generate() when no option is set, and with the
    # disable_* options the oracle's restatement of app.py:27-120 event for event (greedy), no denied id emitted
    P0 = prompt.shape[1]
    evs = list(model.generate_stream(prompt=prompt, batch_size=4, max_len=40, top_k=1))
    ids_stream = np.stack(evs, axis=1)
    out["stream_vs_generate_mismatch"] = (float((ids_stream != ids_new[:, P0:]).sum())
                                          if ids_stream.shape == ids_new[:, P0:].shape else 1e9)
    chans = [int(c) for c in np.unique([tok.tokens2event(r.tolist())[1 + tok.events["note"].index("channel")]
                                        for r in ids_new[:, P0:].reshape(-1, 8) if r[0] == tok.event_ids["note"]])][:2]
    deny = O.deny_ids(tok, True, True, chans)
    evs = list(model.generate_stream(prompt=prompt, batch_size=4, max_len=40, top_k=1, disable_patch_change=True,
                                     disable_control_change=True, disable_channels=chans))
    ids_masked = np.stack(evs, axis=1)
    ref_masked = O.generate(sd16, ocfg, tok, prompt, batch_size=4, max_len=40, top_k=1, deny=deny, max_context=4096,
                            inv_freq_net=model.net.rotary_emb.inv_freq, inv_freq_tok=model.net_token.rotary_emb.inv_freq)[:, P0:]
    out["stream_masked_mismatch"] = (float((ids_masked != ref_masked).sum()) if ids_masked.shape == ref_masked.shape
                                     else 1e9)
    out["stream_denied_ids_emitted"] = float(np.isin(ids_masked, sorted(deny)).sum())
    out["stream_masked_differs_from_plain"] = float((ids_masked[:, :min(ids_masked.shape[1], ids_stream.shape[1])]
                                                     != ids_stream[:, :min(ids_masked.shape[1], ids_stream.shape[1])]).sum())
    print("stream: disabled channels", chans, "masked events", ids_masked.shape[1], "plain events", ids_stream.shape[1])
    # two generations streaming concurrently from two threads on ONE model (gradio serves app.generate from worker threads,
    # app.py:496): each owns its loop state, so both must reproduce their sequential results; a generator resumed from
    # another thread than the one that created it must work too
    import threading
    prompt_b = _song_batch(tok, 4, 9, seed=321).numpy()
    seq_a = np.stack(list(model.generate_stream(prompt=prompt, batch_size=4, max_len=30, top_k=1)), axis=1)
    seq_b = np.stack(list(model.generate_stream(prompt=prompt_b, batch_size=4, max_len=30, top_k=1)), axis=1)
    got, errs = {}, []

    def drive(name, pr):
        try:
            got[name] = np.stack(list(model.generate_stream(prompt=pr, batch_size=4, max_len=30, top_k=1)), axis=1)
        except Exception as e:     # noqa: BLE001
            errs.append(repr(e))
    th = [threading.Thread(target=drive, args=("a", prompt)), threading.Thread(target=drive, args=("b", prompt_b))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    out["stream_concurrent_errors"] = float(len(errs))
    out["stream_concurrent_mismatch"] = (float((got["a"] != seq_a).sum() + (got["b"] != seq_b).sum())
                                         if not errs and got["a"].shape == seq_a.shape and got["b"].shape == seq_b.shape else 1e9)
    gen = model.generate_stream(prompt=prompt, batch_size=4, max_len=30, top_k=1)
    first = next(gen)
    rest = []
    t2 = threading.Thread(target=lambda: rest.extend(list(gen)))
    t2.start()
    t2.join()
    moved = np.stack([first] + rest, axis=1)
    out["stream_resumed_on_other_thread_mismatch"] = float((moved != seq_a).sum()) if moved.shape == seq_a.shape else 1e9
    if errs:
        print("concurrent stream errors:", errs)
    ids_after = model.generate(prompt=prompt, batch_size=4, max_len=40, top_k=1)      # the mask must not leak into generate()
    out["stream_mask_leak_mismatch"] = float((ids_after != ids_new).sum()) if ids_after.shape == ids_new.shape else 1e9
    # the generated continuation is itself grammar-valid
    bad = sum(1 for row in ids_new[:, 1:].reshape(-1, 8) if row[0] not in (tok.eos_id, tok.pad_id) and tok.tokens2event(row.tolist()) == [])
    out["peaked_invalid_events"] = float(bad)
    # teacher-forced logits on a fresh song vs the oracle bf16 / fp32
    batch = _song_batch(tok, 2, 50, seed=5).to(DEV)
    sd32 = {k: v.float() for k, v in sd16.items()}
    with torch.no_grad():
        h = model.forward(batch[:, :-1])
        lg = model.forward_token(h.reshape(-1, 1024), batch[:, 1:].reshape(-1, 8)[:, :-1])
        h32 = O.forward(sd32, ocfg, batch[:, :-1])
        l32 = O.forward_token(sd32, ocfg, h32.reshape(-1, 1024), batch[:, 1:].reshape(-1, 8)[:, :-1])
        l16 = O.forward_token(sd16, ocfg, O.forward(sd16, ocfg, batch[:, :-1]).reshape(-1, 1024),
                              batch[:, 1:].reshape(-1, 8)[:, :-1])
    tg = batch[:, 1:].reshape(-1, 8)
    live = tg != 0
    am, a32, a16 = lg.float().argmax(-1), l32.argmax(-1), l16.float().argmax(-1)
    # reported, not asserted: bf16 and fp32 may pick differently at fp32 near-ties (every disagreement is printed below
    # with its fp32 margin).  Asserted instead: on the same weights and rounding points, the oracle's own bf16 run picks
    # what this implementation picks.
    out["peaked_argmax_mismatch_vs_fp32"] = float((am[live] != a32[live]).sum())
    out["peaked_argmax_mismatch_vs_oracle16"] = float((am[live] != a16[live]).sum())
    out["peaked_argmax_oracle16_diff_vs_fp32"] = float((a16[live] != a32[live]).sum())
    for r, t in (live & (am != a32)).nonzero().tolist():    # evidence for any disagreement with fp32
        row = l32[r, t]
        print(f"peaked argmax vs fp32: row {r} token {t}: new {int(am[r, t])} fp32 {int(a32[r, t])} oracle-bf16 {int(a16[r, t])}, "
              f"fp32 margin {float(row[a32[r, t]] - row[am[r, t]]):.3e}, bf16-vs-fp32 max deviation "
              f"{float((l16.float() - l32).abs().max()):.3e}")
    out["peaked_logits_vs_fp32"] = rel(lg.float(), l32)
    return out


@bounded([("large_loss_abs", 3e-2), ("large_grad_global_rel", 8e-2), ("min:large_params", 457220096.0)],
         info=("large_generate_events",))
def check_model_large():
    """tv2o-large (24 event-level / 6 token-level layers, BASELINE config 5): fused loss + gradients vs the oracle at a
    small shape, and a short KV-cached generate at the maximum context bookkeeping (max_len 4096 pools)."""
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model(GM.config("tv2o-large"))
    out["large_params"] = float(sum(p.numel() for p in model.parameters()))
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    batch = synth_batch(model.tokenizer, 1, 130, seed=3).to(DEV)
    sd = {k: v.detach().float().requires_grad_(True) for k, v in model.state_dict().items()}
    ref = O.train_loss(sd, ocfg, batch)
    ref.backward()
    loss = model.training_loss(batch)
    out["large_loss_abs"] = float((loss - ref.detach()).abs())
    out["large_grad_global_rel"] = global_rel(grads(model), {n: sd[n].grad for n, _ in model.named_parameters()})
    del sd
    model.eval()
    ids = model.generate(batch_size=2, max_len=4096 if False else 40, generator=torch.Generator(DEV).manual_seed(0))
    out["large_generate_events"] = float(ids.shape[1])
    return out



# ------------------------------------------------------------------------------------------ round-2 additions
def _ordered_bf16(t):
    """bf16 bit patterns mapped to integers that are monotonic in the value (for ulp distances)."""
    i = t.contiguous().view(torch.int16).int()
    return torch.where(i >= 0, i, -(i & 0x7FFF))


def _exact_metrics(y, ref64, name, out):
    """y (bf16) vs an fp64 reference: fraction of elements that are not the correctly-rounded bf16 value, the largest
    distance in bf16 ulps among elements that are not tiny, and the worst |err| / (1 ulp + 1e-3 rms) -- a dropped k-block
    or a wrong split-K slice moves whole tiles by many ulps; fp32 summation order moves isolated elements by one."""
    want = ref64.to(torch.float32).to(BF)
    neq = (y != want)
    out[f"exact_frac_{name}"] = float(neq.float().mean())
    rms = float(ref64.pow(2).mean().sqrt())
    big = ref64.abs() > 0.05 * rms
    ulp = (_ordered_bf16(y) - _ordered_bf16(want)).abs()
    out[f"exact_maxulp_{name}"] = float(ulp[big].max()) if bool(big.any()) else 0.0
    tol = ref64.abs() * 2.0 ** -7 + 1e-3 * rms
    out[f"exact_err_over_tol_{name}"] = float(((y.double() - ref64).abs() / tol).max())


# fraction of non-correctly-rounded elements at benchmark shapes: fp32 summation order alone moves ~1e-3 of them by one
# ulp, long-K split sums a few 1e-3 (measured: 5.6e-4 forward K=1024, 1.7e-3..4.3e-3 dgrad K=3072/8192, 3e-3..2.2e-2
# wgrad over 16 384 / 131 072 rows)
@bounded([("exact_maxulp_", 1.0), ("exact_err_over_tol_", 1.0), ("exact_frac_wgrad_", 3e-2), ("exact_frac_", 6e-3),
          ("wgrad_splits_", 64.0)])
def check_gemm_exact():
    """Tensor-core GEMM at the benchmark's own shapes (M = 131 072 rows, K = 131 072 split-K, the tail-split path)
    against an fp64 reference of the same bf16 operands, as mismatch fraction / ulp distance instead of a norm."""
    out = {}
    # forward (K-major x K-major): token-level projections and the event-level MLP shape of the bench step
    for (M, N, K) in ((131072, 1024, 1024), (16384, 8192, 1024), (4096, 3406, 1024)):
        a, w = randn(M, K, seed=M % 97), randn(N, K, scale=0.05, seed=N % 89)
        pitch = (N + 7) // 8 * 8
        y = ops.linear(a, w, pitch=pitch if pitch != N else None)
        ref = a.double() @ w.double().T
        _exact_metrics(y[:, :N], ref, f"fwd_{M}x{N}x{K}", out)
        del a, w, y, ref
    # dgrad (B operand MN-major); [16384, 8192] @ [8192, 1024] takes the K-split of the last partial wave (tail split)
    for (M, N, K) in ((16384, 8192, 1024), (131072, 3072, 1024)):
        dy, w = randn(M, N, seed=5), randn(N, K, scale=0.05, seed=6)
        dx = ops.linear_dgrad(dy, w)
        ref = dy.double() @ w.double()
        _exact_metrics(dx, ref, f"dgrad_{M}x{N}x{K}", out)
        del dy, w, dx, ref
    # wgrad (both operands MN-major): K = 131 072 rows with split-K 9 / 3, and the 16 384-row event-level shapes
    for (M, N, K) in ((131072, 1024, 1024), (131072, 3072, 1024), (16384, 1024, 4096), (16384, 3072, 1024)):
        dy, x = randn(M, N, seed=7), randn(M, K, seed=8)
        dw = torch.empty(N, K, device=DEV, dtype=BF)
        ops.linear_wgrad(dy, x, dw, accumulate=False)
        bn, sp = ops._plan(N, K, M, True)
        out[f"wgrad_splits_{M}x{N}x{K}"] = float(sp)
        ref = dy.double().T @ x.double()
        _exact_metrics(dw, ref, f"wgrad_{M}x{N}x{K}", out)
        del dy, x, dw, ref
    return out


@bounded([("decode_fused_append_mismatch", 0.0), ("decode_fused_T", 6e-3)])
def check_decode_paged():
    """b200_attn_decode_fused (RoPE + KV append + single-query attention, the kernel inside the CUDA-graph generate loop)
    against dense fp32 SDPA with the context crossing 64-position page boundaries, a permuted block table, n_split in
    {1, 2, 16} and the position read from the device (graph mode) or passed by value."""
    out = {}
    from midi_b200 import decode as dec
    from midi_b200.engine import StackCfg
    nh, D, page, Bn, cap = 16, 64, 64, 3, 4096
    H = nh * D
    inv = O.default_inv_freq(D).to(BF).to(DEV)
    cos, sin = ops.rope_table(inv, cap)
    cfg = StackCfg("net", 1, nh, H, 4 * H, 1e-6)
    g = torch.Generator(device=DEV).manual_seed(11)
    scale = 1.0 / math.sqrt(D)
    for T in (1, 63, 64, 65, 257, 1500, 4095):
        pos = T - 1
        for n_split in (1, 2, 16):
            if (T + n_split - 1) // n_split > 1024:
                continue
            kv = dec.PagedKV(cfg, Bn, cap, page, DEV)
            kv.block_table.copy_(torch.randperm(Bn * kv.max_pages, generator=g, device=DEV).int().view(Bn, kv.max_pages))
            hist = randn(Bn * pos, 3 * H, seed=T) if pos > 0 else None
            if pos > 0:
                lib.call("b200_kv_append", hist.data_ptr(), kv.k[0].data_ptr(), kv.v[0].data_ptr(), kv.block_table.data_ptr(),
                         kv.max_pages, kv.page, nh, D, Bn, pos, 0, None, 3 * H, lib.stream())
            new = randn(Bn, 3 * H, seed=T + 1)
            o = torch.empty(Bn, H, device=DEV, dtype=BF)
            ws = torch.empty(lib.query("b200_attn_decode_workspace_bytes", Bn, nh, D, n_split), dtype=torch.uint8, device=DEV)
            # n_split 16 = what the loop with 4096-event pools runs (position from the device counter, max_T = pool size);
            # n_split 1 / 2 = the host-driven path (position by value, max_T = T)
            graph_mode = n_split == 16
            pos_dev = torch.tensor([pos], dtype=torch.int32, device=DEV) if graph_mode else None
            lib.call("b200_attn_decode_fused", new.data_ptr(), kv.k[0].data_ptr(), kv.v[0].data_ptr(), kv.block_table.data_ptr(),
                     kv.max_pages, kv.page, cos.data_ptr(), sin.data_ptr(), o.data_ptr(), Bn, nh, D, 0 if graph_mode else pos,
                     lib.ptr(pos_dev), cap if graph_mode else T, 3 * H, H, scale, n_split, ws.data_ptr(), ws.numel(), lib.stream())
            rc, rs = O.rope_cos_sin(inv, torch.tensor([pos], device=DEV), BF)
            q = O.apply_rope(new[:, :H].view(Bn, 1, nh, D).transpose(1, 2), rc, rs)             # (Bn, nh, 1, D) bf16
            k_new = O.apply_rope(new[:, H:2 * H].view(Bn, 1, nh, D).transpose(1, 2), rc, rs)
            v_new = new[:, 2 * H:].view(Bn, 1, nh, D).transpose(1, 2)
            if pos > 0:
                hk = hist.view(Bn, pos, 3, nh, D)[:, :, 1].transpose(1, 2)
                hv = hist.view(Bn, pos, 3, nh, D)[:, :, 2].transpose(1, 2)
                k_all, v_all = torch.cat([hk, k_new], 2), torch.cat([hv, v_new], 2)
            else:
                k_all, v_all = k_new, v_new
            ref = _sdpa_ref(q.float(), k_all.float(), v_all.float(), pos)
            out[f"decode_fused_T{T}_s{n_split}"] = rel(o.float().view(Bn, 1, nh, D).transpose(1, 2), ref)
            # the new key / value landed in the right page slot (bit-exact RoPE'd key)
            bad = 0
            for b in range(Bn):
                pg = int(kv.block_table[b, pos // page])
                bad += int((kv.k[0][pg, :, pos % page] != k_new[b, :, 0]).sum()) + int((kv.v[0][pg, :, pos % page] != v_new[b, :, 0]).sum())
            out[f"decode_fused_append_mismatch_T{T}_s{n_split}"] = float(bad)
    return out


# The reference's own GPU path: the HF LlamaModels inside MIDIModel (they are the parameter containers, so they read the
# same weights) run exactly as the reference's midi_model.py:116-150 runs them -- eager bf16, torch SDPA.
def _hf_forward(model, x, cache=None):
    e = model.net.embed_tokens(x).sum(dim=-2)
    return model.net(inputs_embeds=e, past_key_values=cache, use_cache=cache is not None).last_hidden_state


def _hf_forward_token(model, hidden_state=None, x=None, cache=None):
    if hidden_state is not None:
        hidden_state = hidden_state.unsqueeze(1)
    if x is not None:
        x = model.net_token.embed_tokens(x)
        if hidden_state is not None:
            x = torch.cat([hidden_state, x], dim=1)
        hidden_state = x
    h = model.net_token(inputs_embeds=hidden_state, past_key_values=cache, use_cache=cache is not None).last_hidden_state
    return model.lm_head(h)


# event-level layer: <= 1e-3 against the reference's GPU path (the oracle's own attention formulation sits further from
# that path).  Token-level layer: torch routes (N, 4, 8, 256) to another SDPA backend whose internal rounding differs;
# this implementation equals the oracle to 2e-5 there and both sit 2.06e-3 from HF (`inner_sdpa_backend_*` metrics
# record each backend's distance to fp32).  Attention alone: two independent bf16-P implementations are ~1e-3 apart,
# each 2.0e-3 from fp32.  The oracle's teacher-forced layers get the model_layer_tf bound.
@bounded([
    ("hidden_new_vs_hf", 3e-2), ("logits_new_vs_hf", 4e-2), ("logits_tf_new_vs_hf", 2e-2), ("min:argmax_agree_new_hf", 0.9),
    ("outer_layer_tf_new_vs_hf", 1e-3), ("inner_layer_tf_new_vs_hf", 3e-3), ("attn_new_vs_sdpa16", 1.5e-3),
    ("hf_loss_abs", 5e-2), ("hf_grad_global_rel", 8e-2), ("outer_layer_tf", 6e-3), ("inner_layer_tf", 6e-3),
], info=("hidden_oracle16_vs_hf", "logits_oracle16_vs_hf", "attn_oracle16_vs_sdpa16", "attn_new_vs_fp32",
         "attn_sdpa16_vs_fp32", "attn_oracle16_vs_fp32", "inner_attn_new_vs_fp32",
         "inner_attn_sdpa_default_vs_fp32", "inner_attn_new_vs_sdpa_default",
         *[f"inner_sdpa_backend_{b}_{m}" for b in ("flash", "efficient", "math", "cudnn")
           for m in ("vs_fp32", "equals_default")]))
def check_model_vs_hf():
    """This implementation vs the reference's eager-bf16 GPU path (HF LlamaModel + torch SDPA on the same device, same
    weights), and the oracle vs that same path: where the oracle's attention rounds differently from the GPU SDPA
    backend, `*_oracle16_vs_hf` shows the distance the teacher-forced tolerance has to absorb."""
    from midi_b200.synth import synth_batch
    out = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).eval()
    sd16 = _sd(model, BF)
    rt = model._rt()
    batch = synth_batch(model.tokenizer, 2, 130, seed=1234).to(DEV)
    x, y = batch[:, :-1], batch[:, 1:]
    ids = y.reshape(-1, 8)[:, :-1]
    with torch.no_grad():
        h = model.forward(x)
        lg = model.forward_token(h.reshape(-1, 1024), ids)
        h_hf = _hf_forward(model, x)
        lg_hf = _hf_forward_token(model, h_hf.reshape(-1, 1024), ids)
        h16 = O.forward(sd16, ocfg, x, inv_freq=model.net.rotary_emb.inv_freq)
        l16 = O.forward_token(sd16, ocfg, h16.reshape(-1, 1024), ids, inv_freq=model.net_token.rotary_emb.inv_freq)
        lg_tf = model.forward_token(h_hf.reshape(-1, 1024), ids)                 # token-level stack fed HF's hidden
        lg_hf_tf = lg_hf
    out["hidden_new_vs_hf"] = rel(h.float(), h_hf.float())
    out["hidden_oracle16_vs_hf"] = rel(h16.float(), h_hf.float())
    out["logits_new_vs_hf"] = rel(lg.float(), lg_hf.float())
    out["logits_oracle16_vs_hf"] = rel(l16.float(), lg_hf.float())
    out["logits_tf_new_vs_hf"] = rel(lg_tf.float(), lg_hf_tf.float())
    out["argmax_agree_new_hf"] = float((lg.float().argmax(-1) == lg_hf.float().argmax(-1)).float().mean())
    # one decoder layer, teacher-forced with the same bf16 input, event level and token level
    import torch.nn as nn
    for which, eng, hf, inv, (nseq, S) in (("outer", rt.outer, model.net, model.net.rotary_emb.inv_freq, (2, 96)),
                                           ("inner", rt.inner, model.net_token, model.net_token.rotary_emb.inv_freq, (64, 8))):
        x_in = randn(nseq * S, 1024, seed=3 if which == "outer" else 4)
        keep_hf, keep = hf.layers, eng.layers
        hf.layers = nn.ModuleList(list(keep_hf)[:1])
        eng.layers = keep[:1]
        try:
            with torch.no_grad():
                ref = hf(inputs_embeds=x_in.view(nseq, S, 1024), use_cache=False).last_hidden_state
                ours, _ = eng.forward(x_in, nseq, S, inv, save=False)
                one = O.StackCfg(eng.cfg.prefix, 1, eng.cfg.n_head, 1024, eng.cfg.inner)
                sd1 = {k: v for k, v in sd16.items() if k.startswith(f"{eng.cfg.prefix}.layers.0.") or k == f"{eng.cfg.prefix}.norm.weight"}
                orc = O.llama_stack(sd1, one, x_in.view(nseq, S, 1024), inv)
        finally:
            hf.layers, eng.layers = keep_hf, keep
        out[f"{which}_layer_tf_new_vs_hf"] = rel(ours.float().view(nseq, S, 1024), ref.float())
        out[f"{which}_layer_tf_oracle16_vs_hf"] = rel(orc.float(), ref.float())
    # attention alone: torch SDPA bf16 (the reference's backend) vs this kernel vs the oracle's formulation
    B, S, nh, D = 2, 512, 16, 64
    qkv = randn(B * S, 3 * nh * D, seed=21)
    q, k, v = (qkv.view(B, S, 3, nh, D)[:, :, i].transpose(1, 2) for i in range(3))
    o_new, _ = ops.attn_causal_fwd(qkv, B, S, nh, D, want_lse=False)
    o_new = o_new.view(B, S, nh, D).transpose(1, 2)
    o_sdpa = F.scaled_dot_product_attention(q, k, v, is_causal=True)
    o_orc = O.attention(q, k, v, 0)
    o_32 = _sdpa_ref(q.float(), k.float(), v.float(), 0)
    out["attn_new_vs_sdpa16"] = rel(o_new.float(), o_sdpa.float())
    out["attn_oracle16_vs_sdpa16"] = rel(o_orc.float(), o_sdpa.float())
    out["attn_new_vs_fp32"] = rel(o_new.float(), o_32)
    out["attn_sdpa16_vs_fp32"] = rel(o_sdpa.float(), o_32)
    out["attn_oracle16_vs_fp32"] = rel(o_orc.float(), o_32)
    # which SDPA backend does torch pick for the token-level shape, and how far is each from fp32 / from this kernel
    from torch.nn.attention import SDPBackend, sdpa_kernel
    Nn, L, nh2, D2 = 64, 8, 4, 256
    qkv2 = randn(Nn * L, 3 * nh2 * D2, seed=22)
    q2, k2, v2 = (qkv2.view(Nn, L, 3, nh2, D2)[:, :, i].transpose(1, 2) for i in range(3))
    o32 = _sdpa_ref(q2.float(), k2.float(), v2.float(), 0)
    o_tiny = ops.attn_tiny_fwd(qkv2, Nn, L, nh2, D2).view(Nn, L, nh2, D2).transpose(1, 2)
    o_def = F.scaled_dot_product_attention(q2, k2, v2, is_causal=True)
    out["inner_attn_new_vs_fp32"] = rel(o_tiny.float(), o32)
    out["inner_attn_sdpa_default_vs_fp32"] = rel(o_def.float(), o32)
    out["inner_attn_new_vs_sdpa_default"] = rel(o_tiny.float(), o_def.float())
    for name, be in (("flash", SDPBackend.FLASH_ATTENTION), ("efficient", SDPBackend.EFFICIENT_ATTENTION),
                     ("math", SDPBackend.MATH), ("cudnn", SDPBackend.CUDNN_ATTENTION)):
        try:
            with sdpa_kernel(be):
                ob = F.scaled_dot_product_attention(q2, k2, v2, is_causal=True)
            out[f"inner_sdpa_backend_{name}_vs_fp32"] = rel(ob.float(), o32)
            out[f"inner_sdpa_backend_{name}_equals_default"] = float(torch.equal(ob, o_def))
        except Exception:
            out[f"inner_sdpa_backend_{name}_vs_fp32"] = -1.0          # backend not available for this shape
    # train step: loss and gradients vs HF autograd in bf16 (the reference's training arithmetic, train.py:168-185)
    model.train()
    tb = synth_batch(model.tokenizer, 2, 66, seed=77, pad_tail=3).to(DEV)
    loss = model.training_loss(tb)
    mine = grads(model)
    for p in model.parameters():
        p.grad = None
    hx = _hf_forward(model, tb[:, :-1].contiguous())
    yy = tb[:, 1:].reshape(-1, 8)
    lgt = _hf_forward_token(model, hx.reshape(-1, 1024), yy[:, :-1])
    l_hf = F.cross_entropy(lgt.view(-1, model.tokenizer.vocab_size), yy.reshape(-1), reduction="mean", ignore_index=model.tokenizer.pad_id)
    l_hf.backward()
    out["hf_loss_abs"] = float((loss.float() - l_hf.float()).abs())
    out["hf_grad_global_rel"] = global_rel(mine, grads(model))
    return out


def _song_batch_long(tok, B, n_events, seed):
    return _song_batch(tok, B, n_events, seed, fixed_step=3)


@bounded([
    ("medium_peaked_loss_last", 0.1), ("opt_state_roundtrip_mismatch", 0.0), ("long_greedy_mismatch", 0.0),
    ("long_pool_vs_public_mismatch", 0.0), ("long_persist_vs_graph_mismatch", 0.0), ("min:long_page_boundaries_crossed", 8.0),
    ("long_invalid_events", 0.0), ("min:long_len_new", 740.0), ("cached_vs_full_hidden_S4096", 3e-2),
    ("cached_vs_full_hidden_past4096", 3e-2), ("min:generate_past4096_len", 4100.0),
    ("bench_shape_loss_abs_vs_oracle32", 3e-2),
], info=("medium_peaked_steps", "long_n_split", "long_len_ref", "long_first_divergence_event",
         "long_first_divergence_margin", "bench_shape_loss_new", "bench_shape_loss_oracle32",
         "bench_shape_loss_abs_oracle16_vs_oracle32"))
def check_model_medium_long():
    """BASELINE config 3 on the real tv2o-medium architecture (12 event-level / 3 token-level layers): train it peaked
    with the fused trainer on long songs, then (a) the CUDA-graph generate loop with 4096-event pools (n_split 16) runs
    >= 600 events past >= 8 KV page boundaries and must emit the oracle's greedy ids bit for bit, (b) the KV-cached
    forward equals the full forward at S = 4096, (c) contexts beyond max_position_embeddings work (app.py: prompt + 4096),
    (d) the loss at the benchmark shape (8 x 2048 events) equals the oracle's on the same weights and batch."""
    from midi_b200.synth import synth_batch
    from transformers import DynamicCache
    out = {}
    model = GM.cpu_model(GM.config("tv2o-medium"))
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    tok = model.tokenizer
    losses = []
    n_steps = 0
    # curriculum: short songs first (many distinct songs per step: the pitch / time rule is learnt after a plateau near 0.47,
    # as in the 4-layer check), then long songs so that positions up to 768 have been trained
    for step in range(1, 1501):
        batch = _song_batch_long(tok, 16, 66, seed=step).to(DEV)
        loss = model.training_loss(batch)
        model.fused_optimizer_step(lr=3e-4 * min(1.0, step / 20), step=step, weight_decay=0.01)
        n_steps = step
        if step % 20 == 0 or step == 1:
            losses.append(float(loss))
            if step >= 100 and max(losses[-2:]) < 0.04:
                break
    short_steps = n_steps
    for step in range(n_steps + 1, n_steps + 401):
        batch = _song_batch_long(tok, 4, 769, seed=step).to(DEV)
        loss = model.training_loss(batch)
        model.fused_optimizer_step(lr=1e-4, step=step, weight_decay=0.01)
        n_steps = step
        if step % 20 == 0:
            losses.append(float(loss))
            if step - short_steps >= 100 and max(losses[-2:]) < 0.02:
                break
    print("medium peaked training losses:", [round(v, 3) for v in losses], "steps", short_steps, n_steps)
    out["medium_peaked_loss_last"] = losses[-1]
    out["medium_peaked_steps"] = float(n_steps)
    # optimizer state round trip (checkpoint / resume of the fused AdamW)
    osd = model.optimizer_state_dict()
    st = model.__dict__["_b200_opt"]
    m0 = st["m"].clone()
    st["m"].zero_()
    resumed = model.load_optimizer_state_dict(osd)
    out["opt_state_roundtrip_mismatch"] = float((st["m"] != m0).sum()) + abs(resumed - n_steps)
    model.eval()
    sd16 = _sd(model, BF)
    inv_n, inv_t = model.net.rotary_emb.inv_freq, model.net_token.rotary_emb.inv_freq
    # ---- (a) long greedy generation, graph loop with 4096-event pools vs the oracle
    P, n_new, Bg = 100, 640, 4
    prompt = _song_batch_long(tok, Bg, P, seed=999).numpy()
    key, gg = model._checkout_generator(Bg, 4096, 1.0, 0.98, 1, None)
    out["long_n_split"] = float(max(1, min(32, (4096 + 255) // 256)))
    try:
        ids_pool = gg.run(torch.from_numpy(prompt).to(DEV), use_graph="persist", max_new=n_new).cpu().numpy()
        ids_pool_graph = gg.run(torch.from_numpy(prompt).to(DEV), use_graph=True, max_new=n_new).cpu().numpy()
    finally:
        model._return_generator(key, gg)
    out["long_persist_vs_graph_mismatch"] = float((ids_pool != ids_pool_graph).sum()) if ids_pool.shape == ids_pool_graph.shape else 1e9
    ids_pub = model.generate(prompt=prompt, batch_size=Bg, max_len=P + n_new, top_k=1)          # public API, exact-size pools
    ids_ref = O.generate(sd16, ocfg, tok, prompt, batch_size=Bg, max_len=P + n_new, top_k=1, inv_freq_net=inv_n, inv_freq_tok=inv_t)
    out["long_len_new"], out["long_len_ref"] = float(ids_pool.shape[1]), float(ids_ref.shape[1])
    n = min(ids_pool.shape[1], ids_ref.shape[1])
    neq = ids_pool[:, :n] != ids_ref[:, :n]
    out["long_greedy_mismatch"] = float(neq.sum()) + abs(ids_pool.shape[1] - ids_ref.shape[1])
    out["long_pool_vs_public_mismatch"] = float((ids_pool != ids_pub).sum()) if ids_pool.shape == ids_pub.shape else 1e9
    out["long_page_boundaries_crossed"] = float((P + n_new - 1) // 64 - (P - 1) // 64)
    bad = sum(1 for row in ids_pool[:, 1:].reshape(-1, 8) if row[0] not in (tok.eos_id, tok.pad_id) and tok.tokens2event(row.tolist()) == [])
    out["long_invalid_events"] = float(bad)
    if neq.any():       # tie audit: the first divergence must sit on an fp32 near-tie
        first_e = int(np.argwhere(neq.any(-1).any(0))[0][0])
        bs, ts = np.nonzero(neq[:, first_e])
        b0, t0 = int(bs[0]), int(ts[0])
        sd32 = {k_: v_.float() for k_, v_ in sd16.items()}
        ref_t = torch.from_numpy(ids_ref[b0:b0 + 1, :first_e + 1]).to(DEV)
        with torch.no_grad():
            h32 = O.forward(sd32, ocfg, ref_t[:, :-1], inv_freq=inv_n)
            l32 = O.forward_token(sd32, ocfg, h32[:, -1], ref_t[:, -1, :7], inv_freq=inv_t)
        row = l32[0, t0]
        out["long_first_divergence_event"] = float(first_e)
        out["long_first_divergence_margin"] = float((row[ids_ref[b0, first_e, t0]] - row[ids_pool[b0, first_e, t0]]).abs())
        print("long: first divergence at event", first_e, "row", b0, "token", t0, ids_ref[b0, first_e], ids_pool[b0, first_e])
        del sd32
    # ---- (b) KV-cached forward == full forward at S = 4096 (prefill 4000 events, then 96 single-event steps)
    song = _song_batch_long(tok, 1, 4100, seed=31).to(DEV)
    with torch.no_grad():
        full = model.forward(song[:, :4096])
        c = DynamicCache()
        parts = [model.forward(song[:, :4000], cache=c)]
        for t in range(4000, 4096):
            parts.append(model.forward(song[:, t:t + 1], cache=c))
        cached = torch.cat(parts, 1)
    out["cached_vs_full_hidden_S4096"] = rel(cached.float(), full.float())
    out["cached_vs_full_hidden_S4096_tail"] = rel(cached[:, 4000:].float(), full[:, 4000:].float())
    # ---- (c) beyond max_position_embeddings: cached forward to 4100 positions, and generate(max_len=4100)
    with torch.no_grad():
        for t in range(4096, 4100):
            parts.append(model.forward(song[:, t:t + 1], cache=c))
        full2 = model.forward(song[:, :4100])
    out["cached_vs_full_hidden_past4096"] = rel(torch.cat(parts[-4:], 1).float(), full2[:, 4096:].float())
    ids_long = model.generate(prompt=song[:, :4090].cpu().numpy(), batch_size=1, max_len=4100, top_k=1)
    out["generate_past4096_len"] = float(ids_long.shape[1])
    del full, full2, cached, parts, c
    # ---- (d) loss at the benchmark shape vs the oracle (bf16 and fp32 weights, same batch), forward only
    model.train()
    bb = synth_batch(tok, 8, 2049, seed=1234).to(DEV)
    with torch.no_grad():
        def oracle_loss(sd):       # train.py:168-185 with the model's own (bf16-rounded) inv_freq buffers
            yb = bb[:, 1:].reshape(-1, 8)
            hid = O.forward(sd, ocfg, bb[:, :-1].contiguous(), inv_freq=inv_n)
            lgo = O.forward_token(sd, ocfg, hid.reshape(-1, 1024), yb[:, :-1], inv_freq=inv_t)
            return float(F.cross_entropy(lgo.view(-1, ocfg.vocab), yb.reshape(-1), reduction="mean", ignore_index=ocfg.pad_id))
        l_new = float(model.training_loss(bb, backward=False))
        l_16 = oracle_loss(sd16)
        torch.cuda.empty_cache()
        sd32 = {k_: v_.float() for k_, v_ in sd16.items()}
        l_32 = oracle_loss(sd32)
        del sd32
        torch.cuda.empty_cache()
    out["bench_shape_loss_new"], out["bench_shape_loss_oracle32"] = l_new, l_32
    out["bench_shape_loss_abs_vs_oracle32"] = abs(l_new - l_32)
    out["bench_shape_loss_abs_oracle16_vs_oracle32"] = abs(l_16 - l_32)
    return out


# train.py:439-449: rank-64 GEMM shapes, adapter gradients vs the oracle's autograd, frozen base untouched
@bounded([
    ("lora_scale_mismatch", 0.0), ("lora_gemm_up_untouched", 0.0), ("lora_gemm_", 4e-3), ("lora_loss_abs", 3e-2),
    ("lora_grad_global_rel", 6e-2), ("lora_base_grads_present", 0.0), ("lora_frozen_changed", 0.0),
    ("min:lora_adapters_changed", 70.0), ("lora_dropin_vs_fused_grad_rel", 2e-2), ("lora_dropin_base_grads_present", 0.0),
    ("lora_cached_vs_full_hidden", 3e-2), ("lora_hidden_vs_oracle32", 3e-2), ("min:lora_generate_len", 2.0),
], info=("lora_grad_worst_rel_info",))
def check_lora_train():
    """LoRA training (train.py:439-449: r = 64, lora_alpha = 128, all seven projections, frozen base) on the native engine.
    (a) the rank-r GEMM shapes the adapters add, through the C ABI, incl. the in-place strided residual epilogue;
    (b) loss and adapter gradients vs the oracle's autograd over W + scale * B A (= peft's unmerged forward in exact
    arithmetic); the frozen base gets no gradient and is bit-identical after the fused optimizer step; drop-in autograd path
    == fused path; (c) inference with injected adapters (merged decode weights) == the training-path forward."""
    from midi_b200.synth import synth_batch
    from midi_b200 import lora
    from transformers import DynamicCache
    out = {}
    r = 64
    # ---- (a) adapter GEMM shapes (rows not a multiple of 128, N = r and K = r smaller than a tile)
    for i, rows in enumerate((1000, 4096)):
        x, A, Bm = randn(rows, 1024, seed=200 + i), randn(r, 1024, scale=0.05, seed=210 + i), randn(1024, r, scale=0.05, seed=220 + i)
        t = ops.linear(x, A)                                                        # [rows, r]
        out[f"lora_gemm_down_{rows}"] = rel(t.float(), x.float() @ A.float().T)
        ts = ops.scale(t, 2.0)
        out[f"lora_scale_mismatch_{rows}"] = float((ts != (t.float() * 2.0).to(BF)).sum())
        y = randn(rows, 3072, seed=230 + i)
        y0 = y.clone()
        yv = y[:, 1024:2048]
        ops.gemm(ts, Bm, rows, 1024, r, lda=r, ldb=r, out=yv, ldc=3072, residual=yv)    # in place on the k third
        ref = ((ts.float() @ Bm.float().T).to(BF).float() + y0[:, 1024:2048].float())
        out[f"lora_gemm_up_inplace_{rows}"] = rel(y[:, 1024:2048].float(), ref)
        out[f"lora_gemm_up_untouched_{rows}"] = float((y[:, :1024] != y0[:, :1024]).sum() + (y[:, 2048:] != y0[:, 2048:]).sum())
        dy = randn(rows, 3072, seed=240 + i)
        dyv = dy[:, 2048:]
        dts = ops.gemm(dyv, Bm, rows, r, 1024, lda=3072, ldb=r, b_mn=True)          # dy . B  -> [rows, r]
        out[f"lora_gemm_dts_{rows}"] = rel(dts.float(), dyv.float() @ Bm.float())
        gB = torch.empty(1024, r, device=DEV, dtype=BF)
        ops.gemm(dyv, ts, 1024, r, rows, lda=3072, ldb=r, a_mn=True, b_mn=True, out=gB, ldc=r, allow_split=True)
        out[f"lora_gemm_gB_{rows}"] = rel(gB.float(), dyv.float().T @ ts.float())
        gA = torch.empty(r, 1024, device=DEV, dtype=BF)
        ops.gemm(dts, x, r, 1024, rows, lda=r, ldb=1024, a_mn=True, b_mn=True, out=gA, ldc=1024, allow_split=True)
        refA = dts.float().T @ x.float()
        out[f"lora_gemm_gA_{rows}"] = rel(gA.float(), refA)
        ops.gemm(dts, x, r, 1024, rows, lda=r, ldb=1024, a_mn=True, b_mn=True, out=gA, ldc=1024, accumulate=True, allow_split=True)
        out[f"lora_gemm_gA_accumulate_{rows}"] = rel(gA.float(), 2 * refA)
        dx = randn(rows, 1024, seed=250 + i)
        dx0 = dx.clone()
        ops.gemm(dts, A, rows, 1024, r, lda=r, ldb=1024, b_mn=True, out=dx, ldc=1024, residual=dx)
        out[f"lora_gemm_dx_inplace_{rows}"] = rel(dx.float(), (dts.float() @ A.float()).to(BF).float() + dx0.float())
        print(f"lora: adapter GEMM shapes at {rows} rows done", flush=True)
    torch.cuda.synchronize()
    # ---- (b) a 4-layer model of the real width: train.py:439-449
    model = GM.cpu_model()
    model = model.to(DEV, dtype=BF).train()
    model.requires_grad_(False)
    model.add_adapter(lora.LoraAdapterConfig(r=r, lora_alpha=128, target_modules=["q_proj", "o_proj", "k_proj", "v_proj",
                                             "gate_proj", "up_proj", "down_proj"], lora_dropout=0, bias="none", task_type="CAUSAL_LM"))
    g = torch.Generator(device="cpu").manual_seed(5)
    with torch.no_grad():                                     # B = 0 at init would make dA vanish: give it trained-like values
        for n, p in model.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(DEV, BF))
    ocfg = O.cfg_from_hf(model.config)
    batch = synth_batch(model.tokenizer, 2, 66, seed=77, pad_tail=3).to(DEV)
    leaf = {n: p.detach().float().requires_grad_(True) for n, p in model.named_parameters()}
    sd = O.lora_effective_sd(leaf, 2.0)          # scaling = lora_alpha / r = 128 / 64
    ref = O.train_loss(sd, ocfg, batch)
    ref.backward()
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    loss = model.training_loss(batch)
    out["lora_loss_abs"] = float((loss - ref.detach()).abs())
    print("lora: fused training step done, loss", float(loss), "oracle", float(ref.detach()), flush=True)
    fused = grads(model)
    adapters = [n for n, _ in model.named_parameters() if ".lora_" in n]
    out["lora_grad_global_rel"] = global_rel(fused, {n: leaf[n].grad for n in adapters})
    out["lora_grad_worst_rel_info"] = max(rel(fused[n].float(), leaf[n].grad) for n in adapters)
    out["lora_base_grads_present"] = float(sum(".lora_" not in n for n in fused))
    model.fused_optimizer_step(lr=1e-3, step=1)
    torch.cuda.synchronize()
    out["lora_frozen_changed"] = float(sum(int(not torch.equal(p, before[n])) for n, p in model.named_parameters() if ".lora_" not in n))
    out["lora_adapters_changed"] = float(sum(int(not torch.equal(p, before[n])) for n, p in model.named_parameters() if ".lora_" in n))
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(before[n])
    for p in model.parameters():
        p.grad = None
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()
    hidden = model.forward(x)
    yy = y.reshape(-1, y.shape[-1])
    logits = model.forward_token(hidden.reshape(-1, hidden.shape[-1]), yy[:, :-1])
    l2 = F.cross_entropy(logits.view(-1, model.tokenizer.vocab_size), yy.view(-1), reduction="mean", ignore_index=model.tokenizer.pad_id)
    l2.backward()
    out["lora_dropin_vs_fused_grad_rel"] = global_rel(grads(model), fused)
    print("lora: drop-in step done", flush=True)
    out["lora_dropin_base_grads_present"] = float(sum(int(p.grad is not None) for n, p in model.named_parameters() if ".lora_" not in n))
    # ---- (c) inference with injected adapters: KV-cached forward (merged decode weights) vs the training-path forward
    model.eval()
    with torch.no_grad():
        full = model.forward(x[:, :40])
        c = DynamicCache()
        parts = [model.forward(x[:, :30], cache=c)] + [model.forward(x[:, t:t + 1], cache=c) for t in range(30, 40)]
        out["lora_cached_vs_full_hidden"] = rel(torch.cat(parts, 1).float(), full.float())
        href = O.forward({k: v.detach() for k, v in sd.items()}, ocfg, x[:, :40], inv_freq=model.net.rotary_emb.inv_freq)
        out["lora_hidden_vs_oracle32"] = rel(full.float(), href)
    ids = model.generate(batch_size=2, max_len=8, top_k=1)
    out["lora_generate_len"] = float(ids.shape[1])
    return out


# ------------------------------------------------------------------------------------------ conformance groups
# The wgmma GEMM and attention called straight through the C ABI with explicit plans, layouts and strides, scored per
# element / per row against fp64 (tests/parity_metrics.py).  Outputs live inside NaN-filled buffers (extra rows, a wider
# pitch) and every input's padding is NaN, so a store outside its range, a tile left unwritten or a read past an extent
# shows up.  Metrics are aggregated per family (worst case); the worst case of each family is printed.
def _rup8(n):
    return (n + 7) // 8 * 8


class _Worst:
    """Worst value per metric over many cases, and which case it came from (NaN counts as worst)."""

    def __init__(self, prefix):
        self.prefix, self.m, self.where = prefix, {}, {}

    def add(self, family, case, d):
        for k, v in d.items():
            key = f"{self.prefix}{family}_{k}" if family else f"{self.prefix}{k}"
            old = self.m.get(key)
            if old is None or math.isnan(v) or (not math.isnan(old) and v > old):
                self.m[key], self.where[key] = float(v), case

    def report(self):
        for k in sorted(self.m):
            print(f"  {k} = {self.m[k]:.4g}  worst at {self.where[k]}")
        return dict(self.m)


def _gm_operand(vals, mn_major, extra):
    """vals [rows, K] as the kernel reads it: K-major = stored [rows, K] with NaN columns K..ld and NaN rows past rows;
    MN-major = stored [K, rows] with NaN rows past K and NaN columns past rows."""
    t = vals.T if mn_major else vals
    return P.poisoned(t.contiguous(), t.shape[0] + extra, _rup8(t.shape[1]) + 8)


def _gm_call(A, B, C, R, M, N, K, ldc, ldr, a_mn, b_mn, acc, bn, splits, ws):
    lib.call("b200_gemm_bf16", A.data_ptr(), B.data_ptr(), C.data_ptr(), lib.ptr(R), M, N, K, A.stride(0), B.stride(0),
             ldc, ldr, int(a_mn), int(b_mn), int(acc), bn, splits, lib.ptr(ws), 0 if ws is None else ws.numel(), lib.stream())


# per-element exactness against the correctly rounded fp64 result (maxulp / err_over_tol as in gemm_exact), NaN
# sentinels around every output and in every input's padding.  Fraction not correctly rounded, H100 80GB HBM3 at 700 W:
# 1.1e-4 K <= 200, 4.0e-4 split-K, 3.5e-3 at K = 6184 (tail split or not); bounds about 5x.  One rounding point: <= 1 ulp.
# Two (residual, accumulate, RoPE, SwiGLU act): <= 2 ulp, measured 2 (see parity_metrics.exact_metrics).  err_over_tol
# measured <= 0.88.
@bounded([
    ("gm_sentinels_changed", 0.0), ("gm_nan_in_range", 0.0), ("gm_padcols_nonzero", 0.0), ("gm_edge_rejected", 0.0),
    ("min:gm_instantiations_run", 8.0), ("min:gm_tail_cases_engaged", 2.0), ("min:gm_multiwave_waves", 1.01),
    ("gm_store_frac", 1e-3), ("gm_residual_frac", 1e-3), ("gm_inplace_frac", 1e-3), ("gm_split_frac", 2e-3),
    ("gm_accum_frac", 1e-3), ("gm_tail_frac", 1.5e-2), ("gm_notail_frac", 1.5e-2), ("gm_edge_frac", 1e-3),
    *[(f"gm_{f}_maxulp", 1.0) for f in ("store", "split", "tail", "notail", "edge")],
    *[(f"gm_{f}_maxulp", 2.0) for f in ("residual", "inplace", "accum")],
    *[(f"gm_{f}_err_over_tol", 1.0) for f in ("store", "residual", "inplace", "split", "accum", "tail", "notail", "edge")],
])
def check_gemm_matrix():
    """b200_gemm_bf16 with an explicit (block_n, splits) for every instantiation (block_n x operand layouts), each
    epilogue, split-K with uneven slices, accumulate, the tail split and small / ragged edges, against an fp64 product of
    the same bf16 operands rounded at the epilogue's rounding points.  No edge is rejected by argument validation or
    tensor-map encoding (gm_edge_rejected counts them)."""
    W = _Worst("gm_")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    layouts = [(0, 0), (0, 1), (1, 0), (1, 1)]
    ran, rejected, min_waves = set(), 0, float("inf")

    def operands(M, N, K, a_mn, b_mn, seed):
        a, b = randn(M, K, seed=seed), randn(N, K, scale=0.05, seed=seed + 1)
        return a, b, _gm_operand(a, a_mn, 5), _gm_operand(b, b_mn, 5), a.double() @ b.double().T

    def store(fam, M, N, K, bn, a_mn, b_mn, seed, ldc=None, ws=None):
        case = f"{M}x{N}x{K} bn{bn} a{a_mn}b{b_mn}"
        a, b, A, B, ref = operands(M, N, K, a_mn, b_mn, seed)
        N8 = _rup8(N)
        ldc = ldc or N8 + 16
        C = P.nan_buffer((M + 3, ldc), device=DEV)
        _gm_call(A, B, C, None, M, N, K, ldc, 0, a_mn, b_mn, 0, bn, 1, ws)
        W.add(fam, case, P.exact_metrics(C[:M, :N], ref))
        W.add("", case, P.sentinel_report(C, (slice(0, M), slice(0, N)), (slice(0, M), slice(N, N8))))
        ran.add((bn, a_mn, b_mn))
        return ref

    def residuals(M, N, K, bn, a_mn, b_mn, seed):
        a, b, A, B, ref = operands(M, N, K, a_mn, b_mn, seed)
        r = randn(M, N, seed=seed + 2)
        acc = P.round_bf16(ref)
        want = (acc + r.double()).to(torch.float32).to(BF)
        # residual in its own buffer, ldr != ldc
        ldc = N + 16
        R = P.poisoned(r, M + 2, N + 24)
        C = P.nan_buffer((M + 3, ldc), device=DEV)
        _gm_call(A, B, C, R, M, N, K, ldc, R.stride(0), a_mn, b_mn, 0, bn, 1, None)
        case = f"{M}x{N}x{K} bn{bn} a{a_mn}b{b_mn}"
        W.add("residual", case, P.exact_metrics(C[:M, :N], acc + r.double(), want, inter=ref))
        W.add("", case, P.sentinel_report(C, (slice(0, M), slice(0, N))))
        # residual aliasing the output in place, in a column view of a wider buffer (engine._fold, _lora_fwd)
        wide = P.nan_buffer((M + 3, N + 40), device=DEV)
        wide[:M, 16:16 + N] = r
        view = wide[:, 16:]
        _gm_call(A, B, view, view, M, N, K, wide.stride(0), wide.stride(0), a_mn, b_mn, 0, bn, 1, None)
        W.add("inplace", case, P.exact_metrics(wide[:M, 16:16 + N], acc + r.double(), want, inter=ref))
        W.add("", case, P.sentinel_report(wide, (slice(0, M), slice(16, 16 + N))))

    # every instantiation: one ragged shape and one multi-wave shape (more work items than SMs, ragged last wave and
    # ragged last M / N tiles, so some persistent CTA's second item is ragged), each with every bf16 epilogue
    for bn in (128, 256):
        for li, (a_mn, b_mn) in enumerate(layouts):
            for si, (M, N, K) in enumerate(((129, 136, 72), (2200, 2000, 200))):
                seed = 1000 + 100 * si + 10 * li + bn // 128
                if si == 1:
                    min_waves = min(min_waves, (M + 127) // 128 * ((N + bn - 1) // bn) / sms)
                store("store", M, N, K, bn, a_mn, b_mn, seed)
                residuals(M, N, K, bn, a_mn, b_mn, seed)

    # split-K: K = 1050 is 17 k-blocks, so 2 / 3 splits are uneven, 7 re-counts to 6 non-empty splits and 40 clamps to
    # 17; the workspace is sized by b200_gemm_workspace_bytes alone
    M, N, K = 300, 520, 1050
    for bn in (128, 256):
        for i, splits in enumerate((2, 3, 7, 40)):
            a_mn, b_mn = layouts[(i + bn // 128) % 4]
            a, b, A, B, ref = operands(M, N, K, a_mn, b_mn, 2000 + 10 * i + bn)
            ws = torch.empty(lib.query("b200_gemm_workspace_bytes", M, N, splits), dtype=torch.uint8, device=DEV)
            C = P.nan_buffer((M + 3, N), device=DEV)
            _gm_call(A, B, C, None, M, N, K, N, 0, a_mn, b_mn, 0, bn, splits, ws)
            case = f"splits{splits} bn{bn} a{a_mn}b{b_mn}"
            W.add("split", case, P.exact_metrics(C[:M], ref))
            W.add("", case, P.sentinel_report(C, (slice(0, M), slice(0, N))))
            ran.add((bn, a_mn, b_mn))
    # accumulate onto a non-zero C at splits 1 and 3: bf16(bf16(acc) + old)
    for splits in (1, 3):
        for bn, (a_mn, b_mn) in ((128, (1, 1)), (256, (0, 1))):
            a, b, A, B, ref = operands(M, N, K, a_mn, b_mn, 2100 + splits + bn)
            old = randn(M, N, seed=2200 + splits)
            ws = torch.empty(lib.query("b200_gemm_workspace_bytes", M, N, splits), dtype=torch.uint8, device=DEV)
            C = P.nan_buffer((M + 3, N), device=DEV)
            C[:M] = old
            _gm_call(A, B, C, None, M, N, K, N, 0, a_mn, b_mn, 1, bn, splits, ws)
            acc = P.round_bf16(ref)
            case = f"accumulate splits{splits} bn{bn} a{a_mn}b{b_mn}"
            W.add("accum", case, P.exact_metrics(C[:M], acc + old.double(), (acc + old.double()).to(torch.float32).to(BF),
                                                 inter=ref))
            W.add("", case, P.sentinel_report(C, (slice(0, M), slice(0, N))))

    # tail split of the last partial wave: shapes whose tail workspace the library itself asks for on this device are
    # run with it and without it; ragged M, ragged N (2002: not a multiple of 8 either), both block_n
    engaged = 0
    for i, (M, N, K, bn, a_mn, b_mn) in enumerate(((1100, 2000, 6184, 128, 0, 0), (2200, 2002, 6184, 256, 0, 1),
                                                   (1100, 2002, 6184, 128, 0, 1), (2200, 2000, 6184, 256, 0, 0))):
        tb = int(lib.query("b200_gemm_tail_workspace_bytes", M, N, K, bn))
        if tb > 0:
            engaged += 1
            store("tail", M, N, K, bn, a_mn, b_mn, 2300 + i, ws=torch.empty(tb, dtype=torch.uint8, device=DEV))
        store("notail", M, N, K, bn, a_mn, b_mn, 2300 + i)

    # small edges: M = 1 / 63 leave the second consumer warpgroup out of range; N = 8, N = 3406 at pitch 3408; K = 8 /
    # 16 / 200 (below one k-block and ragged); every operand has lda > K
    for M, N, K in ((1, 136, 200), (63, 136, 200), (129, 8, 200), (129, 3406, 200), (129, 136, 8), (129, 136, 16),
                    (1, 8, 8), (63, 3406, 16)):
        for bn in (128, 256):
            for li, (a_mn, b_mn) in enumerate(layouts):
                try:
                    store("edge", M, N, K, bn, a_mn, b_mn, 2400 + li, ldc=3408 if N == 3406 else None)
                except lib.B200Error as e:
                    rejected += 1
                    print(f"  rejected {M}x{N}x{K} bn{bn} a{a_mn}b{b_mn}: {e}")
    out = W.report()
    out["gm_instantiations_run"] = float(len(ran))
    out["gm_tail_cases_engaged"] = float(engaged)
    out["gm_edge_rejected"] = float(rejected)
    out["gm_multiwave_waves"] = min_waves
    return out


# as gemm_matrix, same card
@bounded([
    ("ge_sentinels_changed", 0.0), ("ge_nan_in_range", 0.0), ("ge_rope_vs_unfused_mismatch", 0.0),
    ("ge_swiglu_gu_vs_unfused_mismatch", 0.0), ("ge_swiglu_act_vs_unfused_mismatch", 0.0),
    ("ge_rope_frac", 1e-3), ("ge_swiglu_gu_frac", 1e-3), ("ge_swiglu_act_frac", 1e-3),
    ("ge_swiglu_gu_maxulp", 1.0), ("ge_rope_maxulp", 2.0), ("ge_swiglu_act_maxulp", 2.0),
    *[(f"ge_{f}_err_over_tol", 1.0) for f in ("rope", "swiglu_gu", "swiglu_act")],
])
def check_gemm_epilogues():
    """Fused RoPE (head_dim 64 / 128 / 256, rope_cols < N, S = 37 so sequences straddle 128-row tiles) and fused SwiGLU
    (K = 200, M in {1, 129}, I in {128, 384}) epilogues: bit-identical to the plain GEMM + the stand-alone kernel, and
    within one ulp of an fp64 chain with the same rounding points.  Sentinel outputs, poisoned inputs."""
    W = _Worst("ge_")
    # RoPE: qkv = [q | k | v], H = 256 columns each; columns [0, 512) rotated per head, v stored as is
    S, K, H = 37, 200, 256
    for M in (259, 129):
        for D in (64, 128, 256):
            N, rope_cols = 3 * H, 2 * H
            x, w = randn(M, K, seed=M + D), randn(N, K, scale=0.05, seed=M + D + 1)
            A, B = P.poisoned(x, M + 5, K + 16), P.poisoned(w, N + 5, K + 24)
            inv = O.default_inv_freq(D).to(BF).to(DEV)
            cos, sin = ops.rope_table(inv, S)
            ldc = N + 16
            C = P.nan_buffer((M + 3, ldc), device=DEV)
            lib.call("b200_gemm_bf16_rope", A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, A.stride(0), B.stride(0), ldc,
                     cos.data_ptr(), sin.data_ptr(), S, D, rope_cols, lib.stream())
            plain = torch.empty(M, N, device=DEV, dtype=BF)
            _gm_call(A, B, plain, None, M, N, K, N, 0, 0, 0, 0, 256, 1, None)
            ops.rope_qk_(plain, cos, sin, S, H, D)
            case = f"M{M} D{D}"
            W.add("", case, {f"rope_vs_unfused_mismatch_D{D}": float((C[:M, :N] != plain).sum())})
            # fp64 chain: x = bf16(acc); o1 = bf16(bf16(x1 c) + bf16(-x2 s)), o2 = bf16(bf16(x2 c) + bf16(x1 s))
            acc = x.double() @ w.double().T
            xr = P.round_bf16(acc)
            pos = torch.arange(M, device=DEV) % S
            c, s = cos.double()[pos][:, None], sin.double()[pos][:, None]
            q = xr[:, :rope_cols].view(M, -1, 2, D // 2)
            x1, x2 = q[:, :, 0], q[:, :, 1]
            o1 = P.round_bf16(x1 * c) + P.round_bf16(-x2 * s)
            o2 = P.round_bf16(x2 * c) + P.round_bf16(x1 * s)
            chain = torch.cat([torch.stack([o1, o2], 2).reshape(M, rope_cols), xr[:, rope_cols:]], 1)
            mag = torch.maximum(x1.abs(), x2.abs())
            inter = torch.cat([torch.stack([mag, mag], 2).reshape(M, rope_cols), torch.zeros_like(xr[:, rope_cols:])], 1)
            W.add("rope", case, P.exact_metrics(C[:M, :N], chain, chain.to(torch.float32).to(BF), inter=inter))
            W.add("", case, P.sentinel_report(C, (slice(0, M), slice(0, N))))
    # SwiGLU: gu = [g | u] = x Wgu^T stored, act = bf16(bf16(silu(g)) u)
    K = 200
    for M in (1, 129):
        for I in (128, 384):
            x, w = randn(M, K, seed=M + I), randn(2 * I, K, scale=0.05, seed=M + I + 1)
            A, B = P.poisoned(x, M + 5, K + 16), P.poisoned(w, 2 * I + 5, K + 24)
            gu = P.nan_buffer((M + 3, 2 * I + 16), device=DEV)
            act = P.nan_buffer((M + 3, I + 8), device=DEV)
            lib.call("b200_gemm_bf16_swiglu", A.data_ptr(), B.data_ptr(), gu.data_ptr(), act.data_ptr(), M, I, K, A.stride(0),
                     B.stride(0), gu.stride(0), act.stride(0), lib.stream())
            plain = torch.empty(M, 2 * I, device=DEV, dtype=BF)
            _gm_call(A, B, plain, None, M, 2 * I, K, 2 * I, 0, 0, 0, 0, 256, 1, None)
            act_ref = ops.swiglu(plain)
            case = f"M{M} I{I}"
            W.add("", case, {"swiglu_gu_vs_unfused_mismatch": float((gu[:M, :2 * I] != plain).sum()),
                             "swiglu_act_vs_unfused_mismatch": float((act[:M, :I] != act_ref).sum())})
            acc = x.double() @ w.double().T
            g, u = P.round_bf16(acc[:, :I]), P.round_bf16(acc[:, I:])
            chain = P.round_bf16(g * torch.sigmoid(g)) * u
            W.add("swiglu_gu", case, P.exact_metrics(gu[:M, :2 * I], acc))
            W.add("swiglu_act", case, P.exact_metrics(act[:M, :I], chain))
            W.add("", case, P.sentinel_report(gu, (slice(0, M), slice(0, 2 * I))))
            W.add("", case, P.sentinel_report(act, (slice(0, M), slice(0, I))))
    return W.report()


def _attn_ref64_parts(q, k, v, do, off, scale, o_in=None):
    """P.attn_ref64 of (B, h, S, D) tensors, on the whole tensors when their fp64 [Sq, Sk] score matrices fit in 2^26
    elements (0.5 GB), else one batch row and as many heads as fit at a time: materialised at once, a (8, 2048) or
    (1, 4096) case at 16 heads would take tens of GB of fp64 temporaries."""
    B, nh, Sq, _ = q.shape
    Sk = k.shape[2]
    cap = 1 << 26
    if B * nh * Sq * Sk <= cap:
        return P.attn_ref64(q, k, v, do, off, scale, o_in)
    hg = max(1, cap // (Sq * Sk))
    out = None
    for b in range(B):
        for h0 in range(0, nh, hg):
            i = (slice(b, b + 1), slice(h0, h0 + hg))
            part = P.attn_ref64(q[i], k[i], v[i], do[i], off, scale, None if o_in is None else o_in[i])
            if out is None:
                out = [torch.empty((B, nh) + t.shape[2:], dtype=t.dtype, device=t.device) for t in part]
            for t, r in zip(out, part):
                t[i] = r
    return tuple(out)


def _attn_case(W, case, ins, new_out, B, Sq, Sk, nh, cos, sin, scale=0.125, floor=1e-3):
    """One case of the attention conformance groups: b200_attn_causal_fwd{_wgmma,} and, from each implementation's own
    o and lse, b200_attn_causal_bwd{_wgmma,} plain and with the RoPE backward fused into dq / dk, all through the C ABI.
    Scored per (batch, head, row) against fp64 attention and its fp64 gradient given the o each backward receives, and
    wgmma against mma on the same inputs.  The mma backward needs n_heads % 4 == 0, so other head counts run its
    forward only.

    ins    : {"q", "k", "v", "do"} -> (data pointer, [batch, row, head] element strides, (B, nh, S, D) view)
    new_out: "o" -> fresh NaN output buffers for o, "dqkv" -> for dq, dk, dv, as ([(buffer, region the kernel must
             write)], [(data pointer, strides, (B, nh, S, D) view)] of each output)."""
    D = 64
    off = Sk - Sq
    q, k, v, do = (ins[n][2] for n in ("q", "k", "v", "do"))
    o64, lse64, _, _, _ = _attn_ref64_parts(q, k, v, do, off, scale)
    atol = 1e-3 * float(do.double().norm(dim=-1).median())   # row-norm floor on the scale of the inputs
    st_in = [s for n in ("q", "k", "v") for s in ins[n][1]]
    rows = {}
    for impl, sfx in (("wg", "_wgmma"), ("mma", "")):
        obufs, ((o_ptr, o_st, o),) = new_out("o")
        n_lse = B * nh * Sq
        lse = torch.full((n_lse + 64,), float("nan"), device=DEV)
        stt = torch.tensor(st_in + o_st, dtype=torch.int64)
        lib.call("b200_attn_causal_fwd" + sfx, ins["q"][0], ins["k"][0], ins["v"][0], o_ptr, lse.data_ptr(),
                 stt.data_ptr(), B, nh, Sq, Sk, D, scale, lib.stream())
        rows[(impl, "o")] = P.row_worst(o, o64, atol=atol)
        W.add(impl, case, {"lse_abs": float((lse[:n_lse].view(B, nh, Sq).double() - lse64).abs().max())})
        for buf, region in obufs:
            W.add("", case, P.sentinel_report(buf, region))
        W.add("", case, P.sentinel_report(lse, (slice(0, n_lse),)))
        if impl == "mma" and nh % 4:
            continue
        _, _, dq64, dk64, dv64 = _attn_ref64_parts(q, k, v, do, off, scale, o_in=o)
        dq64r = P.rope_bwd64(dq64, cos, sin, torch.arange(Sq, device=DEV) + off)
        dk64r = P.rope_bwd64(dk64, cos, sin, torch.arange(Sk, device=DEV))
        for rope in (False, True):
            gbufs, parts = new_out("dqkv")
            delta = torch.empty(n_lse, device=DEV)
            stb = torch.tensor(st_in + o_st + ins["do"][1] + [s for p in parts for s in p[1]], dtype=torch.int64)
            lib.call("b200_attn_causal_bwd" + sfx, ins["q"][0], ins["k"][0], ins["v"][0], o_ptr, ins["do"][0],
                     lse.data_ptr(), delta.data_ptr(), parts[0][0], parts[1][0], parts[2][0], stb.data_ptr(), B, nh, Sq,
                     Sk, D, scale, cos.data_ptr() if rope else None, sin.data_ptr() if rope else None, lib.stream())
            g = {n: p[2] for n, p in zip(("dq", "dk", "dv"), parts)}
            if rope:
                W.add(impl, case, {"rope_dq_row": P.row_worst(g["dq"], dq64r, atol=atol),
                                   "rope_dk_row": P.row_worst(g["dk"], dk64r, atol=atol),
                                   "rope_dv_mismatch": float((g["dv"] != dv_plain).sum())})
            else:
                for n, ref in (("dq", dq64), ("dk", dk64), ("dv", dv64)):
                    rows[(impl, n)] = P.row_worst(g[n], ref, atol=atol)
                dv_plain = g["dv"].clone()
            for buf, region in gbufs:
                W.add("", case, P.sentinel_report(buf, region))
    for (impl, n), val in rows.items():
        W.add(impl, case, {f"{n}_row": val})
        if impl == "wg" and ("mma", n) in rows:
            # same semantics, so the wgmma worst row should stay near the mma worst row on the same inputs
            W.add("wg_over_mma", case, {n: val / (1.5 * rows[("mma", n)] + floor)})


def _attn_bounds(p):
    """The bound table of an attention conformance group whose metrics _attn_case names with prefix p."""
    return [(f"{p}sentinels_changed", 0.0), (f"{p}nan_in_range", 0.0), (f"{p}wg_rope_dv_mismatch", 0.0),
            (f"{p}mma_rope_dv_mismatch", 0.0), (f"{p}wg_over_mma_", 1.0), (f"{p}wg_lse_abs", AE_LSE_ABS),
            (f"{p}mma_lse_abs", AE_LSE_ABS),
            *[(f"{p}{i}_{n}_row", AE_ROW) for i in ("wg", "mma") for n in ("o", "dq", "dk", "dv", "rope_dq", "rope_dk")]]


# same card: worst row 3.4e-3 (o), 4.4e-3 / 4.6e-3 / 4.5e-3 (dq / dk / dv, with or without the fused RoPE backward),
# equal for both implementations; wgmma / (1.5 mma + 1e-3) <= 0.58; LSE 4.8e-5 (saturated softmax)
AE_ROW, AE_LSE_ABS = 1e-2, 1e-4


@bounded(_attn_bounds("ae_"))
def check_attn_edges():
    """Both attention implementations through the C ABI with explicit strides (_attn_case): separate q / k / v / dO
    buffers with a batch pitch of S + 3 rows and a row pitch of H + 16 (all padding NaN), outputs inside NaN buffers; S
    from 1 to 320, Sq < Sk, one head, saturated softmax."""
    W = _Worst("ae_")
    D, scale = 64, 0.125
    cases = [(3, S, S, nh, 1.0) for S in (1, 2, 17, 63, 64, 65, 127, 129, 320) for nh in (1, 4)]
    cases += [(3, Sq, Sk, 4, 1.0) for Sq, Sk in ((1, 300), (5, 70), (64, 129), (65, 200))]
    cases += [(2, 129, 129, 4, 8.0)]
    inv = O.default_inv_freq(D).to(BF).to(DEV)
    for ci, (B, Sq, Sk, nh, amp) in enumerate(cases):
        H = nh * D
        ld = H + 16
        case = f"B{B} Sq{Sq} Sk{Sk} h{nh}" + (f" x{amp:g}" if amp != 1.0 else "")

        def st(S):
            return [(S + 3) * ld, ld, D]

        def buf(S):
            t = P.nan_buffer((B, S + 3, ld), device=DEV)
            return t, (t.data_ptr(), st(S), t[:, :S, :H].view(B, S, nh, D).transpose(1, 2))

        def operand(S, seed, a=1.0):
            t, desc = buf(S)
            t[:, :S, :H] = randn(B, S, H, scale=a, seed=seed)
            return desc

        def new_out(kind):
            made = [buf(Sq)] if kind == "o" else [buf(Sq), buf(Sk), buf(Sk)]
            return [(t, (slice(None), slice(0, d[2].shape[2]), slice(0, H))) for t, d in made], [d for _, d in made]

        ins = {"q": operand(Sq, 3000 + 4 * ci, amp), "k": operand(Sk, 3001 + 4 * ci, amp), "v": operand(Sk, 3002 + 4 * ci),
               "do": operand(Sq, 3003 + 4 * ci)}
        cos, sin = ops.rope_table(inv, Sk)
        _attn_case(W, case, ins, new_out, B, Sq, Sk, nh, cos, sin, scale)
    return W.report()


# The score families of the long-context groups, shaped through one "carrier" column of every head: column 31, the
# slowest-rotating RoPE pair, so that the decode kernel's rotation of the new q (cos >= 0.85 up to position 4095) keeps
# each family's shape.  Every value is exact in bf16 (powers of two and small integers).
AL_FAMILIES = ("amp1", "amp4", "sink", "late", "flat")
_CARRIER = 31


def _score_family(fam, q, k, sink_key=64.0):
    """q, k [..., S, n_heads, D] bf16 (the key position is the index along dim -3) shaped into a score family:
    "amp1" as given; "amp4" both x4, saturating rows; "sink" q[c] = 2 and k[c] = sink_key at key 0, 0 elsewhere, so
    key 0 leads every query by about sink_key / 4 - 4 nats; "late" q[c] = 16 and k[c] = (key // 64) / 2, so the scores
    rise by one nat per 64-key tile (over 0.17 nats of noise) and the running max moves in every tile; "flat" q = 0:
    every score is 0, attention is uniform and P is exactly 1.

    "late" keeps q's and k's random parts in disjoint RoPE pairs (q x4 where k = 0, k x8 where q / 32), so the ramp
    carries no noise and neither operand is dominated by the component all rows share.  Both backward kernels round dS
    to bf16 before dS.K and dS^T.Q: with the ramp's magnitude on k alone, the sum over a dq row, whose dS cancel, scaled
    that rounding into a worst dq row of 0.1 at S = 4096; on q alone every dk row lay along the carrier and some were
    near zero (worst 0.48).  Pairs stay within their class under the decode kernel's rotation of q, and the carrier's
    partner column is 0 in both."""
    if fam == "amp1":
        return q, k
    if fam == "amp4":
        return q * 4, k * 4
    if fam == "flat":
        return torch.zeros_like(q), k
    kpos = torch.arange(k.shape[-3], device=k.device).view(-1, 1)
    if fam == "sink":
        q, k = q.clone(), k.clone()
        q[..., _CARRIER] = 2.0
        k[..., _CARRIER] = torch.where(kpos == 0, sink_key, 0.0).to(k.dtype)
        return q, k
    D = q.shape[-1]
    col = torch.arange(D, device=q.device) % (D // 2)
    q_own = col < D // 4                                   # pairs 0 .. 15: q's random part, k = 0
    k_own = ~q_own & (col != _CARRIER)                     # pairs 16 .. 30: k's random part, q / 32
    q = torch.where(q_own, q * 4, q / 32)
    k = torch.where(k_own, k * 8, torch.zeros_like(k))
    q[..., _CARRIER], q[..., _CARRIER + D // 2] = 16.0, 0.0
    k[..., _CARRIER] = (kpos // 64).to(k.dtype) / 2
    return q, k


# Segment layouts the ragged trainer can produce beyond those of tests/test_gpu_ragged.py: 32 one-tile segments; short
# segments before two long ones, which the longest-first order table interleaves; one 4096-row segment (64 key tiles)
AL_SEGMENTS = ([64] * 32, [64] * 8 + [1984, 2048], [4096])


# measured on an NVIDIA H100 80GB HBM3 at 700 W, both implementations alike: worst row 3.7e-3 (o, B8 S2048 amp1),
# 7.7e-3 (dq, B8 S2048 sink), 7.3e-3 (dk, B1 S4096 late), 5.0e-3 (dv, B8 S2048 amp4), RoPE backward within 5 %; LSE
# 2.2e-5 (wgmma) / 2.0e-5 (mma), both at amp4; wgmma / (1.5 mma + 1e-3) <= 0.61; segment mode bit-identical, rows <= 5.0e-3,
# LSE 1.3e-6.  The row error does not grow with S: the attn_edges bounds stand.  30 s, 3.9 GiB peak device memory.
@bounded([
    *_attn_bounds("al_"),
    ("al_seg_seg_mismatch", 0.0), ("al_seg_sentinels_changed", 0.0), ("al_seg_nan_in_range", 0.0),
    ("al_seg_row", AE_ROW), ("al_seg_lse_abs", AE_LSE_ABS),
    ("min:al_key_tiles", 64.0), ("min:al_batched_long_cases", 1.0), ("min:al_families_at_4096", 4.0),
])
def check_attn_long():
    """The attention conformance of attn_edges (_attn_case) at the lengths training runs: the benchmark shape (8, 2048),
    (2, 2047), (2, 2049), (3, 1000) and (1, 4096) at 16 heads, with q / k / v column views of one packed qkv buffer of
    row pitch 3H + 64, o / dO / dqkv at their own padded pitches, as ops.attn_causal_fwd / _bwd lay them out (all
    padding NaN, spare NaN rows under every output); at (8, 2048) and (1, 4096) also the peaked score families of
    _score_family.  Plus the segment kernels on AL_SEGMENTS, bit-identical per segment to the unsegmented kernel and
    scored against fp64 (seg_attention_case)."""
    W = _Worst("al_")
    D, nh, scale = 64, 16, 0.125
    H = nh * D
    ldq, ldo, ldd, lddo = 3 * H + 64, H + 24, 3 * H + 56, H + 40
    cases = [(8, 2048, f) for f in AL_FAMILIES] + [(1, 4096, f) for f in AL_FAMILIES]
    cases += [(2, 2047, "amp1"), (2, 2049, "amp1"), (3, 1000, "amp1")]
    inv = O.default_inv_freq(D).to(BF).to(DEV)
    key_tiles, batched_long, fams_4096 = 0, 0, set()
    for ci, (B, S, fam) in enumerate(cases):
        case = f"B{B} S{S} {fam}"
        R = B * S
        vals = randn(B, S, 3, nh, D, seed=7000 + ci)
        q, k = _score_family(fam, vals[:, :, 0], vals[:, :, 1])
        qkv = P.nan_buffer((R + 64, ldq), device=DEV)
        for c, t in enumerate((q, k, vals[:, :, 2])):
            qkv[:R, c * H:(c + 1) * H] = t.reshape(R, H)
        dob = P.poisoned(randn(R, H, seed=7100 + ci), R + 64, lddo)

        def desc(t, col, ld):
            return t.data_ptr() + 2 * col, [S * ld, ld, D], t[:R, col:col + H].view(B, S, nh, D).transpose(1, 2)

        def new_out(kind):
            if kind == "o":
                t = P.nan_buffer((R + 64, ldo), device=DEV)
                return [(t, (slice(0, R), slice(0, H)))], [desc(t, 0, ldo)]
            t = P.nan_buffer((R + 64, ldd), device=DEV)
            return [(t, (slice(0, R), slice(0, 3 * H)))], [desc(t, c * H, ldd) for c in range(3)]

        ins = {"q": desc(qkv, 0, ldq), "k": desc(qkv, H, ldq), "v": desc(qkv, 2 * H, ldq), "do": desc(dob, 0, lddo)}
        cos, sin = ops.rope_table(inv, S)
        _attn_case(W, case, ins, new_out, B, S, S, nh, cos, sin, scale)
        key_tiles = max(key_tiles, (S + 63) // 64)
        batched_long += int(B > 1 and S >= 2048)
        if S == 4096 and fam != "amp1":
            fams_4096.add(fam)
    for segs in AL_SEGMENTS:
        W.add("seg", f"segments {segs[0]} x{len(segs)}" if len(set(segs)) == 1 else f"segments {segs}",
              seg_attention_case(segs, nh))
        key_tiles = max(key_tiles, max(segs) // 64)
    out = W.report()
    out["al_key_tiles"], out["al_batched_long_cases"] = float(key_tiles), float(batched_long)
    out["al_families_at_4096"] = float(len(fams_4096))
    return out


def seg_attention_case(segs, nh):
    """b200_attn_causal_{fwd,bwd}_seg_wgmma on one packed batch of segments of the given row counts (multiples of 64),
    nh heads, with the fused RoPE backward and without, outputs in NaN-sentinel buffers: every segment must be
    bit-identical to b200_attn_causal_{fwd,bwd}_wgmma run on that segment alone (in segment mode the kernels run the same
    tiles in the same order on the same operands), and is scored per row against fp64.  Returns the metrics without a
    case tag: sentinel counts, seg_mismatch_* (differing elements), row_* (worst row) and lse_abs."""
    import midi_model as mm
    D = 64
    H = nh * D
    N = sum(segs)
    ldq, ldo = 3 * H + 64, H + 64
    g = torch.Generator(device=DEV).manual_seed(7)
    rnd = lambda *s: torch.randn(*s, generator=g, device=DEV).to(BF)
    qkvb = P.poisoned(rnd(N, 3 * H), N + 64, ldq)
    dob = P.poisoned(rnd(N, H), N + 64, ldo)
    seg = mm._ragged_layout(list(segs), 1, torch.device(DEV))[1]
    cos, sin = ops.rope_table(O.default_inv_freq(D).to(BF).to(DEV), max(segs))
    st_f = torch.tensor([ldq, D] * 3 + [ldo, D], dtype=torch.int64)
    st_b = torch.tensor([ldq, D] * 3 + [ldo, D] * 2 + [ldq, D] * 3, dtype=torch.int64)
    nb = lambda r, c: P.nan_buffer((r, c), device=DEV)
    m = {}
    # ---- segment mode
    q, k, v = (qkvb.data_ptr() + 2 * i * H for i in range(3))
    ob = nb(N + 64, ldo)
    lse = torch.full((nh * N + 64,), float("nan"), device=DEV)
    lib.call("b200_attn_causal_fwd_seg_wgmma", q, k, v, ob.data_ptr(), lse.data_ptr(), st_f.data_ptr(), N // 64, nh, D,
             0.125, seg.tiles.data_ptr(), seg.order.data_ptr(), lib.stream())
    m.update({f"{k_}_fwd": v_ for k_, v_ in P.sentinel_report(ob, (slice(0, N), slice(0, H))).items()})
    m.update({f"{k_}_lse": v_ for k_, v_ in P.sentinel_report(lse, (slice(0, nh * N),)).items()})
    grads = {}
    for rope in (False, True):
        dq = nb(N + 64, ldq)
        delta = torch.empty(nh * N, device=DEV)
        lib.call("b200_attn_causal_bwd_seg_wgmma", q, k, v, ob.data_ptr(), dob.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                 dq.data_ptr(), dq.data_ptr() + 2 * H, dq.data_ptr() + 4 * H, st_b.data_ptr(), N // 64, nh, D, 0.125,
                 cos.data_ptr() if rope else None, sin.data_ptr() if rope else None, seg.tiles.data_ptr(),
                 seg.order.data_ptr(), lib.stream())
        m.update({f"{k_}_bwd_rope{int(rope)}": v_
                  for k_, v_ in P.sentinel_report(dq, (slice(0, N), slice(0, 3 * H))).items()})
        grads[rope] = dq
    lse = lse[:nh * N].view(nh, N)
    # ---- each segment alone through the unsegmented kernel, and fp64
    mism = {"o": 0, "lse": 0, "dqkv": 0, "dqkv_rope": 0}
    worst = {}
    r0 = 0
    for R in segs:
        base = qkvb.data_ptr() + r0 * ldq * 2
        st1 = torch.tensor([R * ldq, ldq, D] * 3 + [R * ldo, ldo, D], dtype=torch.int64)
        o1 = nb(R, ldo)
        l1 = torch.empty(nh * R, device=DEV)
        lib.call("b200_attn_causal_fwd_wgmma", base, base + 2 * H, base + 4 * H, o1.data_ptr(), l1.data_ptr(), st1.data_ptr(),
                 1, nh, R, R, D, 0.125, lib.stream())
        mism["o"] += int((o1[:, :H] != ob[r0:r0 + R, :H]).sum())
        mism["lse"] += int((l1.view(nh, R) != lse[:, r0:r0 + R]).sum())
        stb1 = torch.tensor([R * ldq, ldq, D] * 3 + [R * ldo, ldo, D] * 2 + [R * ldq, ldq, D] * 3, dtype=torch.int64)
        for rope in (False, True):
            d1 = nb(R, ldq)
            delta = torch.empty(nh * R, device=DEV)
            lib.call("b200_attn_causal_bwd_wgmma", base, base + 2 * H, base + 4 * H, o1.data_ptr(),
                     dob.data_ptr() + r0 * ldo * 2, l1.data_ptr(), delta.data_ptr(), d1.data_ptr(), d1.data_ptr() + 2 * H,
                     d1.data_ptr() + 4 * H, stb1.data_ptr(), 1, nh, R, R, D, 0.125, cos.data_ptr() if rope else None,
                     sin.data_ptr() if rope else None, lib.stream())
            mism["dqkv_rope" if rope else "dqkv"] += int((d1[:, :3 * H] != grads[rope][r0:r0 + R, :3 * H]).sum())
        heads = lambda t, c0: t[r0:r0 + R, c0:c0 + H].view(R, nh, D).transpose(0, 1)
        qs, ks, vs, dos, os_ = heads(qkvb, 0), heads(qkvb, H), heads(qkvb, 2 * H), heads(dob, 0), heads(ob, 0)
        o64, lse64, dq64, dk64, dv64 = (t[0] for t in _attn_ref64_parts(qs[None], ks[None], vs[None], dos[None], 0, 0.125,
                                                                         o_in=os_[None]))
        atol = 1e-3 * float(dos.double().norm(dim=-1).median())
        sc = {"o": P.row_worst(os_, o64, atol=atol), "lse_abs": float((lse[:, r0:r0 + R].double() - lse64).abs().max())}
        for rope in (False, True):
            gq, gk, gv = (heads(grads[rope], c) for c in (0, H, 2 * H))
            rq = P.rope_bwd64(dq64, cos, sin, slice(0, R)) if rope else dq64
            rk = P.rope_bwd64(dk64, cos, sin, slice(0, R)) if rope else dk64
            sfx = "_rope" if rope else ""
            sc["dq" + sfx] = P.row_worst(gq, rq, atol=atol)
            sc["dk" + sfx] = P.row_worst(gk, rk, atol=atol)
            sc["dv" + sfx] = P.row_worst(gv, dv64, atol=atol)
        for n, val in sc.items():
            worst[n] = max(worst.get(n, 0.0), val)
        r0 += R
    m.update({f"seg_mismatch_{n}": float(c) for n, c in mism.items()})
    m.update({(n if n == "lse_abs" else f"row_{n}"): val for n, val in worst.items()})
    return m


# ------------------------------------------------------------------------------------------ decode conformance groups
# The kernels behind generate() through the C ABI, as the groups above treat the training GEMM and attention: outputs and
# KV pools in NaN buffers, NaN (or, where NaN would read as "no candidate", a large value) in every operand's padding,
# projections scored per element against fp64 chains with the kernels' rounding points, attention per (row, head)
# against fp64 over the pools read through the block table, samplers / RNG / commit against exact restatements
# (tests/decode_reference.py).
GV_KS = (8, 200, 1024, 1032, 4096)


def _rope_chain64(x, cos, sin, pos):
    """The three-rounding RoPE of rope_kernel / decode_attn_fused_kernel in fp64: x (..., D) bf16 at position pos ->
    (rotated values as fp64, |x| magnitude of the pre-rotation pair for exact_metrics' inter)."""
    D = x.shape[-1]
    c, s = cos[pos].double(), sin[pos].double()
    x1, x2 = x[..., :D // 2].double(), x[..., D // 2:].double()
    o1 = P.round_bf16(P.round_bf16(x1 * c) + P.round_bf16(-x2 * s))
    o2 = P.round_bf16(P.round_bf16(x2 * c) + P.round_bf16(x1 * s))
    mag = torch.maximum(x1.abs(), x2.abs())
    return torch.cat([o1, o2], -1), torch.cat([mag, mag], -1)


def _rms_chain64(x, w, eps):
    """bf16(w * bf16(x * rstd)) in fp64 (rstd exact): the RMSNorm rounding points of the decode projections."""
    x = x.double()
    rstd = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    return P.round_bf16(w.double() * P.round_bf16(x * rstd))


# measured on an H100 80GB HBM3 at 700 W.  Fraction not correctly rounded 8.2e-4 (plain, residual), 7.4e-4 (fused),
# 3.8e-4 (SwiGLU), bounds about 5x; <= 1 ulp for one rounding point, 2 with the residual (measured 2 plain + residual, 1
# elsewhere); err_over_tol <= 0.71.  The three bit-identity claims of gemv_fused_kernel hold (0 mismatches), the norm one
# at every K including those where b200_rmsnorm_fwd uses its block kernel.
@bounded([
    ("gv_sentinels_changed", 0.0), ("gv_nan_in_range", 0.0), ("gv_fused_vs_gemv_mismatch", 0.0),
    ("gv_norm_vs_unfused_mismatch", 0.0), ("gv_swiglu_vs_unfused_mismatch", 0.0),
    ("min:gv_fused_cases", 80.0), ("min:gv_fused_batches", 16.0), ("min:gv_loop_columns_per_warp", 2.0),
    *[(f"gv_{f}_frac", 4e-3) for f in ("plain", "res", "fused")],
    *[(f"gv_{f}_frac", 2e-3) for f in ("fusedres", "fusedsw", "fusedswres")],
    *[(f"gv_{f}_maxulp", 1.0) for f in ("plain", "fused")],
    *[(f"gv_{f}_maxulp", 2.0) for f in ("res", "fusedres", "fusedsw", "fusedswres")],
    *[(f"gv_{f}_err_over_tol", 1.0) for f in ("plain", "res", "fused", "fusedres", "fusedsw", "fusedswres")],
])
def check_gemv_conformance():
    """b200_gemv_bf16 at every batch instantiation B = 1..16 and b200_gemv_fused over its option matrix (x by pointer or
    gathered by ids with a stride and out-of-range ids, RMSNorm, SwiGLU, residual), K across the 4-vector prefetch
    boundary (1024 / 1032) and N past 8 warps x 4 CTAs x SMs (warps take a second column, the `!first` branch), with
    padded leading dimensions; plus the bit-identity claims of the fused kernel against the unfused launches."""
    W = _Worst("gv_")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_loop = 32 * sms + 40
    Ns = (1, 7, 8, 136, 3406, n_loop)
    eps, Vt = 1e-6, 50
    combos = [(ids, nrm, sw, res) for ids in (0, 1) for nrm in (0, 1) for sw in (0, 1) for res in (0, 1)]
    n_fused, bs_fused = 0, set()

    def gemv(X, Wp, R, y, B, N, K):
        lib.call("b200_gemv_bf16", X.data_ptr(), Wp.data_ptr(), lib.ptr(R), y.data_ptr(), B, N, K, X.stride(0),
                 Wp.stride(0), R.stride(0) if R is not None else 0, y.stride(0), lib.stream())

    def fused(X, ids, table, nw, Wp, R, y, B, N, K, sw):
        lib.call("b200_gemv_fused", lib.ptr(X), lib.ptr(ids), ids.stride(0) if ids is not None else 0, lib.ptr(table),
                 Vt if ids is not None else 0, lib.ptr(nw), eps, Wp.data_ptr(), lib.ptr(R), y.data_ptr(), B, N, K,
                 X.stride(0) if X is not None else 0, Wp.stride(0), R.stride(0) if R is not None else 0, y.stride(0),
                 int(sw), lib.stream())

    for ki, K in enumerate(GV_KS):
        wv = {N: randn(2 * N, K, scale=0.05, seed=5000 + N + K) for N in Ns}
        wp = {N: P.poisoned(wv[N], 2 * N + 1, K + 16) for N in Ns}        # [gate | up] rows; plain uses the first N
        # ---- b200_gemv_bf16, every B, with and without residual; the fused kernel without options on the same inputs
        for B in range(1, 17):
            x = randn(B, K, seed=B * 31 + K)
            X = P.poisoned(x, B + 1, K + 8)
            for N in Ns:
                case = f"B{B} N{N} K{K}"
                ref = x.double() @ wv[N][:N].double().T
                for res in (False, True):
                    r = randn(B, N, seed=B + N + K) if res else None
                    R = P.poisoned(r, B + 1, N + 3) if res else None
                    y = P.nan_buffer((B + 2, N + 5), device=DEV)
                    gemv(X, wp[N], R, y, B, N, K)
                    if res:
                        acc = P.round_bf16(ref)
                        W.add("res", case, P.exact_metrics(y[:B, :N], acc + r.double(),
                                                           (acc + r.double()).to(torch.float32).to(BF), inter=ref))
                    else:
                        W.add("plain", case, P.exact_metrics(y[:B, :N], ref))
                    W.add("", case, P.sentinel_report(y, (slice(0, B), slice(0, N))))
                    y2 = P.nan_buffer((B + 2, N + 5), device=DEV)
                    fused(X, None, None, None, wp[N], R, y2, B, N, K, 0)
                    W.add("", case, {"fused_vs_gemv_mismatch": float((y2[:B, :N] != y[:B, :N]).sum())})
        # ---- b200_gemv_fused option matrix: each combination at every K, B and N rotating so that all are reached
        table = P.nan_buffer((Vt + 2, K), device=DEV)                  # rows Vt, Vt + 1 NaN: an unclamped id reads them
        table[:Vt] = randn(Vt, K, seed=77 + K)
        nw = P.nan_buffer((K + 8,), device=DEV)
        nw[:K] = (1 + 0.1 * randn(K, seed=78 + K).float()).to(BF)
        for ci, (use_ids, nrm, sw, res) in enumerate(combos):
            B = (ci * 7 + ki * 3) % 16 + 1
            N = Ns[(ci + ki) % len(Ns)]
            case = f"B{B} N{N} K{K} ids{use_ids} norm{nrm} swiglu{sw} res{res}"
            g = torch.Generator(device=DEV).manual_seed(ci + 10 * K)
            if use_ids:
                ids = torch.randint(0, Vt, (B, 3), generator=g, device=DEV)
                for b, bad in zip(range(B), (-3, Vt, 10 ** 12, Vt + 1)):
                    ids[b, 0] = bad                                        # out of range: the kernel reads row 0
                rows = ids[:, 0].clone()
                rows[(rows < 0) | (rows >= Vt)] = 0
                xrows, X = table[rows], None
            else:
                ids = None
                xrows = randn(B, K, seed=ci + K)
                X = P.poisoned(xrows, B + 1, K + 8)
            xin = _rms_chain64(xrows, nw[:K], eps) if nrm else xrows.double()
            acc = xin @ wv[N][:N].double().T
            if sw:
                g_, u_ = P.round_bf16(acc), P.round_bf16(xin @ wv[N][N:].double().T)
                pre = P.round_bf16(g_ * torch.sigmoid(g_)) * u_
            else:
                pre = acc
            r = randn(B, N, seed=ci + N + K + 1) if res else None
            R = P.poisoned(r, B + 1, N + 3) if res else None
            y = P.nan_buffer((B + 2, N + 5), device=DEV)
            fused(X, ids, table if use_ids else None, nw if nrm else None, wp[N], R, y, B, N, K, sw)
            fam = "fused" + ("sw" if sw else "") + ("res" if res else "")
            if res:
                base = P.round_bf16(pre)
                W.add(fam, case, P.exact_metrics(y[:B, :N], base + r.double(),
                                                 (base + r.double()).to(torch.float32).to(BF), inter=pre))
            else:
                W.add(fam, case, P.exact_metrics(y[:B, :N], pre))
            W.add("", case, P.sentinel_report(y, (slice(0, B), slice(0, N))))
            n_fused += 1
            bs_fused.add(B)
        # ---- bit identity: fused RMSNorm + projection == b200_rmsnorm_fwd + b200_gemv_bf16; fused SwiGLU == b200_gemv_bf16
        # (2 N rows) + b200_swiglu_fwd
        for B in (1, 5, 16):
            x = randn(B, K, scale=3.0, seed=900 + B + K)
            N = 136
            y = P.nan_buffer((B + 2, N + 5), device=DEV)
            fused(x, None, None, nw, wp[N], None, y, B, N, K, 0)
            n1 = torch.empty(B, K, device=DEV, dtype=BF)
            lib.call("b200_rmsnorm_fwd", x.data_ptr(), nw.data_ptr(), n1.data_ptr(), None, B, K, eps, lib.stream())
            y2 = P.nan_buffer((B + 2, N + 5), device=DEV)
            gemv(n1, wp[N], None, y2, B, N, K)
            W.add("", f"B{B} K{K}", {"norm_vs_unfused_mismatch": float((y[:B, :N] != y2[:B, :N]).sum())})
            for N in (8, 136, n_loop):
                y = P.nan_buffer((B + 2, N + 5), device=DEV)
                fused(x, None, None, None, wp[N], None, y, B, N, K, 1)
                gu = torch.empty(B, 2 * N, device=DEV, dtype=BF)
                gemv(x, wp[N], None, gu, B, 2 * N, K)
                act = torch.empty(B, N, device=DEV, dtype=BF)
                lib.call("b200_swiglu_fwd", gu.data_ptr(), act.data_ptr(), B, N, lib.stream())
                W.add("", f"B{B} N{N} K{K}", {"swiglu_vs_unfused_mismatch": float((y[:B, :N] != act).sum())})
        del wv, wp
    out = W.report()
    out["gv_fused_cases"], out["gv_fused_batches"] = float(n_fused), float(len(bs_fused))
    out["gv_loop_columns_per_warp"] = math.ceil(n_loop / (4 * sms * 8))
    return out


def _paged_pools(nh, D, page, Bn, cap, seed):
    """NaN K / V pools with spare pages and a permuted block table."""
    mp = (cap + page - 1) // page
    n_pages = Bn * mp + 3
    g = torch.Generator(device=DEV).manual_seed(seed)
    bt = torch.randperm(n_pages, generator=g, device=DEV)[:Bn * mp].int().view(Bn, mp).contiguous()
    return P.nan_buffer((n_pages, nh, page, D), device=DEV), P.nan_buffer((n_pages, nh, page, D), device=DEV), bt, mp


def _same(a, b):
    """Element-wise bit equality that counts two NaNs as equal (pool slots nobody may write stay NaN)."""
    return (a == b) | (torch.isnan(a.float()) & torch.isnan(b.float()))


def _kv_append(qkv, kp, vp, bt, mp, page, nh, D, Bn, s_new, pos0, dev):
    """b200_kv_append of s_new rows per batch row at pos0, passed by value or (dev) from the device."""
    pd = torch.tensor([pos0], dtype=torch.int32, device=DEV) if dev else None
    lib.call("b200_kv_append", qkv.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), mp, page, nh, D, Bn, s_new,
             0 if dev else pos0, lib.ptr(pd), qkv.stride(0), lib.stream())


def _fused_decode_case(W, kern, case, qkv, pools, pools0, expect, bt, mp, page, cos, sin, Bn, nh, D, pos, dev, max_T,
                       n_split, ref, atol):
    """b200_attn_decode_fused of the new token rows qkv at position pos (by value or from the device) on the pools
    reset to pools0: the pools must equal `expect` (the appended slots, no other slot touched) and the output must
    match ref per (row, head); the CTA kernels must also be bit-identical to b200_rope_qk + b200_kv_append +
    b200_attn_decode on the same inputs."""
    kp, vp = pools
    k0, v0 = pools0
    kexp, vexp = expect
    H, scale = nh * D, 1.0 / math.sqrt(D)
    kp.copy_(k0)
    vp.copy_(v0)
    pdv = torch.tensor([pos], dtype=torch.int32, device=DEV) if dev else None
    o = P.nan_buffer((Bn + 1, H + 8), device=DEV)
    nbytes = lib.query("b200_attn_decode_workspace_bytes", Bn, nh, D, n_split)
    ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
    lib.call("b200_attn_decode_fused", qkv.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), mp, page,
             cos.data_ptr(), sin.data_ptr(), o.data_ptr(), Bn, nh, D, 0 if dev else pos, lib.ptr(pdv), max_T,
             qkv.stride(0), o.stride(0), scale, n_split, ws.data_ptr(), nbytes, lib.stream())
    W.add(kern, case, {"append_mismatch": float((~_same(kp, kexp)).sum() + (~_same(vp, vexp)).sum()),
                       "o_row": P.row_worst(o[:Bn, :H].view(Bn, nh, 1, D), ref, atol=atol)})
    W.add(kern, case, P.sentinel_report(o, (slice(0, Bn), slice(0, H))))
    if kern == "warp256":
        return
    # the unfused launches on the same inputs: b200_rope_qk + b200_kv_append + b200_attn_decode
    q2 = qkv.clone()
    lib.call("b200_rope_qk", q2.data_ptr(), cos.data_ptr(), sin.data_ptr(), Bn, 1, H, D, q2.stride(0), 0,
             pos, None, lib.stream())
    k2, v2 = k0.clone(), v0.clone()
    _kv_append(q2, k2, v2, bt, mp, page, nh, D, Bn, 1, pos, False)
    o2 = P.nan_buffer((Bn + 1, H + 8), device=DEV)
    lib.call("b200_attn_decode", q2.data_ptr(), k2.data_ptr(), v2.data_ptr(), bt.data_ptr(), mp, page,
             o2.data_ptr(), Bn, 1, nh, D, pos, None, max_T, q2.stride(0), o2.stride(0), scale, n_split,
             ws.data_ptr(), nbytes, lib.stream())
    W.add(kern, case, {"vs_unfused_mismatch": float((~_same(o, o2)).sum() + (~_same(kp, k2)).sum()
                                                    + (~_same(vp, v2)).sum())})


# same card: appends bit-exact, nothing else written; worst (row, head) against fp64 attention 3.3e-3 (b200_attn_decode,
# head_dim 64), 2.7e-3 (256), 2.8e-3 / 2.4e-3 / 2.7e-3 (fused: 64-dim CTA, 256-dim CTA, warp kernel); fused CTA kernels
# bit-identical to RoPE + append + b200_attn_decode; 302 splits without keys ran
@bounded([
    ("da_append_mismatch", 0.0), ("da_append_sentinels_changed", 0.0), ("da_append_nan_in_range", 0.0),
    ("da_attn_sentinels_changed", 0.0), ("da_attn_nan_in_range", 0.0), ("da_attn_pool_changed", 0.0),
    ("da_attn_d64_o_row", 1.5e-2), ("da_attn_d256_o_row", 1.5e-2), ("min:da_empty_splits_run", 1.0),
    *[(f"da_{k}_{m}", 0.0) for k in ("cta64", "cta256", "warp256")
      for m in ("append_mismatch", "sentinels_changed", "nan_in_range", "vs_unfused_mismatch")],
    *[(f"da_{k}_o_row", 1.5e-2) for k in ("cta64", "cta256", "warp256")],
])
def check_decode_attn_conformance():
    """b200_kv_append, b200_attn_decode and b200_attn_decode_fused (its 64-dim and 256-dim CTA kernels and the warp kernel
    of the token-level stack) on NaN pools behind a permuted block table: appended slots bit-exact and no other slot
    touched, contexts across page boundaries, splits with no keys, positions by value and from the device, padded
    leading dimensions; outputs per (row, head) against fp64 attention over the pools."""
    import decode_reference as DR
    W = _Worst("da_")
    n_empty_splits = 0

    # ---- b200_kv_append
    for nh, D, page, cap in ((16, 64, 64, 192), (4, 256, 8, 24)):
        H, Bn = nh * D, 3
        for s_new in (1, 5):
            for pos0 in (0, page - 2):
                for dev in (False, True):
                    case = f"D{D} s_new{s_new} pos0 {pos0}" + (" dev" if dev else "")
                    kp, vp, bt, mp = _paged_pools(nh, D, page, Bn, cap, seed=pos0 + s_new)
                    vals = randn(Bn * s_new, 3 * H, seed=D + s_new + pos0)
                    qkv = P.poisoned(vals, Bn * s_new + 1, 3 * H + 24)
                    _kv_append(qkv, kp, vp, bt, mp, page, nh, D, Bn, s_new, pos0, dev)
                    v4 = vals.view(Bn, s_new, 3, nh, D)
                    bad = 0
                    for b in range(Bn):
                        bad += int((DR.gather_kv(kp, bt, page, b, pos0 + s_new)[:, pos0:] != v4[b, :, 1].transpose(0, 1)).sum())
                        bad += int((DR.gather_kv(vp, bt, page, b, pos0 + s_new)[:, pos0:] != v4[b, :, 2].transpose(0, 1)).sum())
                    m = DR.slot_mask(kp.shape, bt, page, [(b, pos0 + i) for b in range(Bn) for i in range(s_new)])
                    W.add("append", case, {"mismatch": float(bad)})
                    W.add("append", case, P.sentinel_report(kp, m))
                    W.add("append", case, P.sentinel_report(vp, m))

    # ---- b200_attn_decode: s_q query rows per batch row, row i sees keys 0 .. past + i
    for nh, D, page in ((16, 64, 64), (4, 256, 8)):
        H, Bn, scale = nh * D, 2, 1.0 / math.sqrt(D)
        for T in (1, 31, 32, 33, 63, 64, 65, 1500, 2048):
            max_T = T if T == 2048 else T + 17               # 2048 / 2 splits: a chunk of exactly 1024 keys
            kp, vp, bt, mp = _paged_pools(nh, D, page, Bn, max_T, seed=T + D)
            hist = randn(Bn * T, 3 * H, seed=T * 3 + D)
            _kv_append(hist, kp, vp, bt, mp, page, nh, D, Bn, T, 0, False)
            k0, v0 = kp.clone(), vp.clone()
            atol = 1e-3 * float(hist[:, 2 * H:].double().view(-1, D).norm(dim=-1).median())
            for s_q in (1, 5, 8):
                if s_q > T:
                    continue
                past = T - s_q
                qv = randn(Bn * s_q, H, seed=T + s_q + D)
                Q = P.poisoned(qv, Bn * s_q + 1, H + 24)
                q4 = qv.view(Bn, s_q, nh, D).transpose(1, 2)
                ref = torch.stack([DR.paged_attention64(q4[b], kp, vp, bt, page, b, T, scale) for b in range(Bn)])
                for n_split in (1, 2, 3, 16, 32):
                    if (max_T + n_split - 1) // n_split > 1024:
                        continue
                    chunk = (T + n_split - 1) // n_split
                    n_empty_splits += sum(1 for s in range(n_split) if s * chunk >= T)
                    for dev in (False, True):
                        case = f"D{D} T{T} s_q{s_q} n_split{n_split}" + (" past_dev" if dev else "")
                        pdv = torch.tensor([past], dtype=torch.int32, device=DEV) if dev else None
                        rows = Bn * s_q
                        o = P.nan_buffer((rows + 2, H + 16), device=DEV)
                        nbytes = lib.query("b200_attn_decode_workspace_bytes", rows, nh, D, n_split)
                        ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
                        lib.call("b200_attn_decode", Q.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), mp, page,
                                 o.data_ptr(), Bn, s_q, nh, D, 0 if dev else past, lib.ptr(pdv), max_T, Q.stride(0),
                                 o.stride(0), scale, n_split, ws.data_ptr(), nbytes, lib.stream())
                        got = o[:rows, :H].view(Bn, s_q, nh, D).transpose(1, 2)
                        W.add(f"attn_d{D}", case, {"o_row": P.row_worst(got, ref, atol=atol)})
                        W.add("attn", case, P.sentinel_report(o, (slice(0, rows), slice(0, H))))
            W.add("attn", f"D{D} T{T}", {"pool_changed": float((~_same(kp, k0)).sum() + (~_same(vp, v0)).sum())})

    # ---- b200_attn_decode_fused: RoPE + append + attention of one new token per batch row
    for kern, nh, D, page, cap, Ts, splits in (("cta64", 16, 64, 64, 1600, (1, 33, 64, 65, 1500), (1, 2, 3, 16)),
                                                ("cta256", 4, 256, 8, 128, (1, 9, 33, 100), (1, 2, 3)),
                                                ("warp256", 4, 256, 8, 32, (1, 8, 9, 32), (1,))):
        H, Bn, scale = nh * D, 3, 1.0 / math.sqrt(D)
        inv = O.default_inv_freq(D).to(BF).to(DEV)
        cos, sin = ops.rope_table(inv, cap)
        for T in Ts:
            pos = T - 1
            max_T = cap if kern != "cta64" else T + 7
            kp, vp, bt, mp = _paged_pools(nh, D, page, Bn, cap, seed=T + D + 1)
            if pos:
                _kv_append(randn(Bn * pos, 3 * H, seed=T + D + 2), kp, vp, bt, mp, page, nh, D, Bn, pos, 0, False)
            k0, v0 = kp.clone(), vp.clone()
            vals = randn(Bn, 3 * H, seed=T + D + 3)
            qkv = P.poisoned(vals, Bn + 1, 3 * H + 8)
            v4 = vals.view(Bn, 3, nh, D)
            q64, _ = _rope_chain64(v4[:, 0], cos, sin, pos)
            k64, _ = _rope_chain64(v4[:, 1], cos, sin, pos)
            kexp, vexp = k0.clone(), v0.clone()
            for b in range(Bn):
                pg = int(bt[b, pos // page])
                kexp[pg, :, pos % page] = k64[b].to(BF)
                vexp[pg, :, pos % page] = v4[b, 2]
            ref = torch.stack([DR.paged_attention64(q64[b][:, None], kexp, vexp, bt, page, b, T, scale) for b in range(Bn)])
            atol = 1e-3 * float(v4[:, 2].double().norm(dim=-1).median())
            for n_split in splits:
                if (max_T + n_split - 1) // n_split > 1024:
                    continue
                for dev in (False, True):
                    _fused_decode_case(W, kern, f"{kern} T{T} n_split{n_split}" + (" pos_dev" if dev else ""), qkv,
                                       (kp, vp), (k0, v0), (kexp, vexp), bt, mp, page, cos, sin, Bn, nh, D, pos, dev, max_T,
                                       n_split, ref, atol)
    out = W.report()
    out["da_empty_splits_run"] = float(n_empty_splits)
    return out

# Generation's longest contexts: 4096-event pools read in n_split chunks and combined.  Measured on an NVIDIA H100 80GB
# HBM3 at 700 W: worst (row, head) 3.7e-3 (b200_attn_decode, late T2049 B16 s_q8 n_split8), 3.1e-3 (fused, amp1 T2049
# B16 n_split4); appends bit-exact, no other pool slot or sentinel written, fused bit-identical to the unfused launches;
# 156672 combines with split maxima more than 20 nats apart.  3 s, 2.6 GiB peak device memory.
DL_TS = (2049, 3000, 4095, 4096)
DL_SPLITS = (4, 8, 16, 32)      # 4: the fewest that keep a chunk of 4096 keys at <= 1024; 16: what generate runs
DL_FAMILIES = ("amp1", "sink", "late", "flat")


@bounded([
    ("dl_attn_sentinels_changed", 0.0), ("dl_attn_nan_in_range", 0.0), ("dl_attn_pool_changed", 0.0),
    ("dl_attn_o_row", 1.5e-2), ("dl_cta64_o_row", 1.5e-2),
    *[(f"dl_cta64_{m}", 0.0) for m in ("append_mismatch", "sentinels_changed", "nan_in_range", "vs_unfused_mismatch")],
    ("min:dl_splits_at_4096", 4.0), ("min:dl_combines_over_20_nats", 1.0),
])
def check_decode_attn_long():
    """b200_attn_decode (s_q 1 and 8) and b200_attn_decode_fused (64-dim CTA kernel) as decode_attn_edges runs them, at
    max_T 4096 with T from 2049 to 4096, n_split 4 to 32, 1 and 16 batch rows and the score families of _score_family
    (the sink 28 to 32 nats above every other key, so the combine scales the other splits' partials down by more than
    20 nats).  Positions by value and from the device; outputs per (row, head) against fp64 over the pools, no pool slot
    but the appended ones written, the fused kernel bit-identical to RoPE + append + b200_attn_decode."""
    import decode_reference as DR
    W = _Worst("dl_")
    nh, D, page, max_T = 16, 64, 64, 4096
    H, scale = nh * D, 1.0 / math.sqrt(D)
    cos, sin = ops.rope_table(O.default_inv_freq(D).to(BF).to(DEV), max_T)
    splits_4096, wide = set(), 0
    for fi, fam in enumerate(DL_FAMILIES):
        for ti, T in enumerate(DL_TS):
            for Bn in (1, 16):
                seed = 8000 + 100 * fi + 10 * ti + Bn
                vals = randn(Bn, T, 3, nh, D, seed=seed)
                q, k = _score_family(fam, vals[:, :, 0], vals[:, :, 1], sink_key=128.0)
                qkv_t = torch.stack([q, k, vals[:, :, 2]], 2)          # [Bn, T, 3, nh, D]: the qkv row of position t
                atol = 1e-3 * float(vals[:, :, 2].double().norm(dim=-1).median())
                # ---- b200_attn_decode: the queries of the last s_q positions over all T keys
                kp, vp, bt, mp = _paged_pools(nh, D, page, Bn, max_T, seed=seed)
                _kv_append(qkv_t.reshape(Bn * T, 3 * H), kp, vp, bt, mp, page, nh, D, Bn, T, 0, False)
                k0, v0 = kp.clone(), vp.clone()
                for s_q in (1, 8):
                    past, rows = T - s_q, Bn * s_q
                    qv = q[:, past:]
                    Q = P.poisoned(qv.reshape(rows, H), rows + 1, H + 24)
                    ref = torch.stack([DR.paged_attention64(qv[b].transpose(0, 1), kp, vp, bt, page, b, T, scale)
                                       for b in range(Bn)])
                    for n_split in DL_SPLITS:
                        for dev in (False, True):
                            case = f"{fam} T{T} B{Bn} s_q{s_q} n_split{n_split}" + (" past_dev" if dev else "")
                            pdv = torch.tensor([past], dtype=torch.int32, device=DEV) if dev else None
                            o = P.nan_buffer((rows + 2, H + 16), device=DEV)
                            nbytes = lib.query("b200_attn_decode_workspace_bytes", rows, nh, D, n_split)
                            ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
                            lib.call("b200_attn_decode", Q.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), mp,
                                     page, o.data_ptr(), Bn, s_q, nh, D, 0 if dev else past, lib.ptr(pdv), max_T,
                                     Q.stride(0), o.stride(0), scale, n_split, ws.data_ptr(), nbytes, lib.stream())
                            got = o[:rows, :H].view(Bn, s_q, nh, D).transpose(1, 2)
                            W.add("attn", case, {"o_row": P.row_worst(got, ref, atol=atol)})
                            W.add("attn", case, P.sentinel_report(o, (slice(0, rows), slice(0, H))))
                            # the split maxima the combine pass rescaled by: (m, l, o[D]) records per (row, head, split)
                            m = ws[:rows * nh * n_split * (D + 2)].view(rows * nh, n_split, D + 2)[:, :, 0]
                            wide += int((m.amax(1) - m.amin(1) > 20).sum())
                            if T == max_T:
                                splits_4096.add(n_split)
                W.add("attn", f"{fam} T{T} B{Bn}", {"pool_changed": float((~_same(kp, k0)).sum() + (~_same(vp, v0)).sum())})
                # ---- b200_attn_decode_fused: the token at position T - 1 over the T - 1 before it
                pos = T - 1
                kp, vp, bt, mp = _paged_pools(nh, D, page, Bn, max_T, seed=seed + 1)
                _kv_append(qkv_t[:, :pos].reshape(Bn * pos, 3 * H), kp, vp, bt, mp, page, nh, D, Bn, pos, 0, False)
                k0, v0 = kp.clone(), vp.clone()
                v4 = qkv_t[:, pos]
                qkv = P.poisoned(v4.reshape(Bn, 3 * H), Bn + 1, 3 * H + 8)
                q64, _ = _rope_chain64(v4[:, 0], cos, sin, pos)
                k64, _ = _rope_chain64(v4[:, 1], cos, sin, pos)
                kexp, vexp = k0.clone(), v0.clone()
                for b in range(Bn):
                    pg = int(bt[b, pos // page])
                    kexp[pg, :, pos % page] = k64[b].to(BF)
                    vexp[pg, :, pos % page] = v4[b, 2]
                ref = torch.stack([DR.paged_attention64(q64[b][:, None], kexp, vexp, bt, page, b, T, scale)
                                   for b in range(Bn)])
                for n_split in DL_SPLITS:
                    for dev in (False, True):
                        _fused_decode_case(W, "cta64", f"{fam} T{T} B{Bn} n_split{n_split}" + (" pos_dev" if dev else ""),
                                           qkv, (kp, vp), (k0, v0), (kexp, vexp), bt, mp, page, cos, sin, Bn, nh, D, pos,
                                           dev, max_T, n_split, ref, atol)
    out = W.report()
    out["dl_splits_at_4096"], out["dl_combines_over_20_nats"] = float(len(splits_4096)), float(wide)
    return out


SM_VOCABS = (1, 37, 3406, 4096)
SM_TOP_PS = (1.0, 0.9, 0.75, 0.5)


def sm_top_ks(V):
    return sorted({1, 20, 64, 65, V})


# every id and value exact; 5.3 % of the logits-sampler rows are ambiguous (a candidate's fp64 p within 2^-17 of a bf16
# rounding midpoint), bound about 5x
@bounded([
    ("sm_topp_fp32_mismatch", 0.0), ("sm_topp_bf16_mismatch", 0.0), ("min:sm_topp_fp32_rows", 2000.0),
    ("min:sm_topp_bf16_rows", 2000.0), ("sm_logits_mismatch", 0.0), ("sm_logits_ambiguous_frac", 0.25),
    ("sm_logits_stride_untouched_changed", 0.0), ("sm_fast_vs_general_mismatch", 0.0), ("sm_uniform_mismatch", 0.0),
    ("sm_uniform_counter_error", 0.0), ("sm_commit_mismatch", 0.0),
])
def check_sampler_conformance():
    """b200_sample_topp_topk and b200_sample_from_logits against the exact restatements of tests/decode_reference.py
    (every row's id), the fast top_k <= 64 path against the general one, b200_uniform_fill and b200_event_commit."""
    import decode_reference as DR
    from midi_b200 import decode as dec
    from midi_b200.tokenizer_tables import TokenizerTables
    out = {}
    # ---- b200_sample_topp_topk: fp32 and bf16 probabilities, padding columns hold 1.0 (a read past V would win)
    for is_bf16 in (0, 1):
        bad = rows = 0
        for V in SM_VOCABS:
            probs = DR.sampler_cases(V, seed=V)
            t = torch.from_numpy(probs).to(DEV)
            if is_bf16:
                t = t.to(BF)
                probs = t.float().cpu().numpy()
            R_ = t.shape[0]
            buf = torch.ones(R_ + 1, V + 3, device=DEV, dtype=t.dtype)
            buf[:R_, :V] = t
            u = DR.uniforms(R_, seed=V + 1)
            ud = torch.from_numpy(u).to(DEV)
            for top_k in sm_top_ks(V):
                for top_p in SM_TOP_PS:
                    o = torch.full((R_ + 1,), -7, dtype=torch.long, device=DEV)
                    lib.call("b200_sample_topp_topk", buf.data_ptr(), is_bf16, R_, V, buf.stride(0), top_p, top_k,
                             ud.data_ptr(), o.data_ptr(), lib.stream())
                    want = DR.sample_rows(probs, top_p, top_k, u, bool(is_bf16))
                    got = o.cpu().numpy()
                    bad += int((got[:R_] != want).sum()) + int(got[R_] != -7)
                    rows += R_
        out[f"sm_topp_{'bf16' if is_bf16 else 'fp32'}_mismatch"] = float(bad)
        out[f"sm_topp_{'bf16' if is_bf16 else 'fp32'}_rows"] = float(rows)
    # ---- b200_sample_from_logits: grammar ranges, temperature, masks, out_stride
    tokz = TokenizerTables("v2")
    glut = dec.GrammarLUT(tokz, DEV)
    lut = glut.lut.cpu().numpy()
    V, ld, Rn = 3406, 3408, 64
    g = torch.Generator(device=DEV).manual_seed(21)
    logits = torch.full((Rn, ld), 30.0, device=DEV, dtype=BF)
    logits[:, :V] = (torch.randn(Rn, V, generator=g, device=DEV) * 2.5).to(BF)
    logits[8:16, :V] = logits[8:16, :V].float().clamp(max=2.0).to(BF)             # many exact ties at the top
    logits[16:20, :V] = 0.5                                                           # a whole row tied
    lg_np = logits[:, :V].float().cpu().numpy()
    ev_types = sorted(tokz.event_ids.values())
    ev = [ev_types[r % len(ev_types)] for r in range(Rn)]
    ev[5], ev[6], ev[7] = glut.eos, glut.pad, glut.eos + 1 + glut.n_event_types + 5  # eos / pad / a parameter id: pad only
    ev_d = torch.tensor(ev, dtype=torch.long, device=DEV)
    gm = torch.Generator(device=DEV).manual_seed(22)
    mask = (torch.rand(Rn, V, generator=gm, device=DEV) > 0.1).to(torch.uint8)
    mask[3] = 0                                                                       # empties every range: id lo
    mask_np = mask.cpu().numpy()
    u = DR.uniforms(Rn, seed=23)
    ud = torch.from_numpy(u).to(DEV)

    def row_range(step, r):
        if step == 0:
            return glut.eos, glut.eos + 1 + glut.n_event_types
        e = ev[r] - (glut.eos + 1)
        if ev[r] == glut.eos or e < 0 or e >= glut.n_event_types:
            return glut.pad, glut.pad + 1
        lo, hi = (int(v) for v in lut[e, step - 1])
        return (lo, hi) if hi > lo else (glut.pad, glut.pad + 1)

    bad = amb = n = stride_bad = 0
    for step in range(8):
        for temp in (1.0, 0.7):
            for top_k in (1, 20, 64, 65, 4096):
                for top_p, use_mask in ((0.98, False), (1.0, True), (0.5, step % 2 == 0)):
                    o = torch.full((Rn, 8), -7, dtype=torch.long, device=DEV)
                    lib.call("b200_sample_from_logits", logits.data_ptr(), Rn, V, ld, temp, top_p, top_k, step,
                             ev_d.data_ptr(), glut.lut.data_ptr(), glut.n_event_types, glut.eos, glut.pad,
                             mask.data_ptr() if use_mask else None, ud.data_ptr(), o.data_ptr() + 8 * step, 8, lib.stream())
                    oc = o.cpu().numpy()
                    stride_bad += int((np.delete(oc, step, axis=1) != -7).sum())
                    for r in range(Rn):
                        lo, hi = row_range(step, r)
                        want, a = DR.logits_sample(lg_np[r], temp, top_p, top_k, lo, hi, mask_np[r] if use_mask else None,
                                                   float(u[r]))
                        n += 1
                        amb += int(a)
                        bad += int((not a) and oc[r, step] != want)
    out["sm_logits_mismatch"] = float(bad)
    out["sm_logits_ambiguous_frac"] = amb / n
    out["sm_logits_stride_untouched_changed"] = float(stride_bad)
    # ---- fast path (top_k <= 64) vs general path (top_k > 64) where the allowed set has <= 64 candidates
    small = torch.zeros(Rn, V, dtype=torch.uint8, device=DEV)
    for r in range(Rn):
        small[r, torch.randperm(V, generator=gm, device=DEV)[:40]] = 1
    small[16:20, :] = 0
    small[16:20, 100:160] = 1                                                         # 60 exactly tied candidates
    # step 0 (7 ids) and step 2 (time2, 16 ids) also run without a mask; the other parameters have up to 2048 ids
    diff = 0
    for step in range(8):
        for temp in (1.0, 0.7):
            for top_p in (1.0, 0.98, 0.5):
                for us in range(3):
                    uu = torch.from_numpy(DR.uniforms(Rn, seed=100 + us)).to(DEV)
                    ids = []
                    for top_k in (64, 4096):
                        o = torch.full((Rn,), -7, dtype=torch.long, device=DEV)
                        lib.call("b200_sample_from_logits", logits.data_ptr(), Rn, V, ld, temp, top_p, top_k, step,
                                 ev_d.data_ptr(), glut.lut.data_ptr(), glut.n_event_types, glut.eos, glut.pad,
                                 None if step in (0, 2) else small.data_ptr(), uu.data_ptr(), o.data_ptr(), 1, lib.stream())
                        ids.append(o)
                    diff += int((ids[0] != ids[1]).sum())
    out["sm_fast_vs_general_mismatch"] = float(diff)
    # ---- b200_uniform_fill: the counter-based hash, bit for bit; counter[0] + 1, counter[1] (device seed) kept
    c0, dev_seed, seed = 5, 0x1234567890ABCDE, 987654321
    for n_ in (1, 1024):
        cnt = torch.tensor([c0, dev_seed], dtype=torch.int64, device=DEV)
        ub = torch.full((n_ + 8,), float("nan"), device=DEV)
        lib.call("b200_uniform_fill", ub.data_ptr(), n_, seed, cnt.data_ptr(), lib.stream())
        want = DR.uniform_fill(n_, seed, c0, dev_seed)
        got = ub.cpu().numpy()
        out[f"sm_uniform_mismatch_n{n_}"] = float((got[:n_] != want).sum() + (~np.isnan(got[n_:])).sum())
        out[f"sm_uniform_counter_error_n{n_}"] = float(abs(int(cnt[0]) - (c0 + 1)) + abs(int(cnt[1]) - dev_seed))
    # ---- b200_event_commit, including pos + 1 == max_len (seq is not written)
    B, T, L = 3, 8, 6
    bad = 0
    for p in (2, L - 2, L - 1):
        ev_t = torch.randint(0, 3000, (T, B), device=DEV)
        seq = torch.full((B, L, T), -5, dtype=torch.long, device=DEV)
        nxt = torch.zeros(B, T, dtype=torch.long, device=DEV)
        pos = torch.tensor([p], dtype=torch.int32, device=DEV)
        lib.call("b200_event_commit", ev_t.data_ptr(), seq.data_ptr(), nxt.data_ptr(), pos.data_ptr(), B, T, L, lib.stream())
        ws, wn, wp = DR.event_commit(ev_t.cpu().numpy(), np.full((B, L, T), -5), np.zeros((B, T), np.int64), p, L)
        bad += int((seq.cpu().numpy() != ws).sum() + (nxt.cpu().numpy() != wn).sum()) + abs(int(pos) - wp)
    out["sm_commit_mismatch"] = float(bad)
    for k_ in sorted(out):
        print(f"  {k_} = {out[k_]:.4g}")
    return out


def _event_step64(eng, e, k_pools, v_pools, bt, page, pos, cos, sin, want_x=False):
    """The event-level stack's step for a new event at position `pos` (one for every row, or one per row) in fp64 (no
    rounding), over the cached keys / values 0 .. pos-1 of each layer's pools.  Returns each layer's new (k, v) as
    [B, n_heads, D]; with `want_x` also the stack's output x [B, H] (before the final norm)."""
    c = eng.cfg
    nh, D, H = c.n_head, c.head_dim, c.hidden
    B = e.shape[0]
    rows_pos = [int(pos)] * B if np.ndim(pos) == 0 else [int(p) for p in pos]
    pidx = torch.tensor(rows_pos, device=e.device)

    def rms(x, w):
        return w.double() * x / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + c.eps)

    def rope(x):
        cs, sn = cos[pidx].double()[:, None], sin[pidx].double()[:, None]
        x1, x2 = x[..., :D // 2], x[..., D // 2:]
        return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1)

    x = e.double()
    kv = []
    for li, w in enumerate(eng.layers):
        qkv = rms(x, w.ln1) @ w.qkv.double().T
        q, k, v = (qkv[:, i * H:(i + 1) * H].view(B, nh, D) for i in range(3))
        q, k = rope(q), rope(k)
        kv.append((k, v))
        o = torch.empty(B, nh, D, dtype=torch.float64, device=e.device)
        for b in range(B):
            t = torch.arange(rows_pos[b], device=e.device)
            pg = bt[b].long()[t // page]
            kc = torch.cat([k_pools[li][pg, :, t % page].transpose(0, 1).double(), k[b][:, None]], 1)
            vc = torch.cat([v_pools[li][pg, :, t % page].transpose(0, 1).double(), v[b][:, None]], 1)
            p = torch.softmax((kc @ q[b][:, :, None])[..., 0] / math.sqrt(D), -1)
            o[b] = (p[:, None, :] @ vc)[:, 0]
        h = x + o.reshape(B, H) @ w.o.double().T
        gu = rms(h, w.ln2) @ w.gu.double().T
        I = gu.shape[1] // 2
        x = h + (F.silu(gu[:, :I]) * gu[:, I:]) @ w.down.double().T
    return (kv, x) if want_x else kv


def _token_steps64(eng, lm_head, outer_norm, x, tokens, n, cos, sin, *, rope_lag=0):
    """The token-level half of one event in fp64 (no rounding), from the event-level output x [B, H] and the event's
    tokens [>= n - 1, B] (teacher-forced): hidden = RMSNorm(x) with the event-level stack's final norm, step i's input is
    hidden (i = 0) or the token-level embedding of tokens[i - 1] (an id outside [0, V) reads row 0, as the kernel does),
    causal attention over steps 0 .. i with RoPE at position i (cos / sin: [positions, D / 2]), final norm, lm_head.
    Returns (k, v) [n_layers, B, n, n_heads, D] and logits [B, n, V].  `rope_lag` rotates step i at position i - 1."""
    c = eng.cfg
    nh, D, H = c.n_head, c.head_dim, c.hidden
    B, V = x.shape[0], lm_head.shape[0]

    def rms(z, w):
        return w.double() * z / torch.sqrt(z.pow(2).mean(-1, keepdim=True) + c.eps)

    ids = tokens[:n - 1].long().clone()
    ids[(ids < 0) | (ids >= V)] = 0
    z = torch.cat([rms(x.double(), outer_norm)[:, None], eng.embed.double()[ids.T]], 1)       # [B, n, H]
    t = (torch.arange(n, device=x.device) - rope_lag).clamp_min(0)
    cs, sn = cos[t].double(), sin[t].double()

    def rope(q):                                                                            # [B, nh, n, D]
        q1, q2 = q[..., :D // 2], q[..., D // 2:]
        return torch.cat([q1 * cs - q2 * sn, q2 * cs + q1 * sn], -1)

    future = torch.triu(torch.ones(n, n, dtype=torch.bool, device=x.device), 1)
    ks, vs = [], []
    for w in eng.layers:
        qkv = rms(z, w.ln1) @ w.qkv.double().T
        q, k, v = (qkv[..., i * H:(i + 1) * H].view(B, n, nh, D).transpose(1, 2) for i in range(3))
        q, k = rope(q), rope(k)
        ks.append(k.transpose(1, 2))
        vs.append(v.transpose(1, 2))
        p = torch.softmax((q @ k.transpose(-1, -2) / math.sqrt(D)).masked_fill(future, float("-inf")), -1)
        h = z + (p @ v).transpose(1, 2).reshape(B, n, H) @ w.o.double().T
        gu = rms(h, w.ln2) @ w.gu.double().T
        I = gu.shape[-1] // 2
        z = h + (F.silu(gu[..., :I]) * gu[..., I:]) @ w.down.double().T
    return torch.stack(ks), torch.stack(vs), rms(z, eng.norm) @ lm_head.double().T


# same card: layer-0 k / v bit-identical and within 1 ulp of the fp64 chain (frac 1.2e-4); worst (row, head) of any
# layer's new k / v against the unrounded fp64 event step 1.06e-2 (persistent) and 1.05e-2 (loop); persistent / (1.5
# loop + 1e-3) <= 0.72
@bounded([
    ("pd_l0_kv_persist_vs_phase_mismatch", 0.0), ("pd_l0_k_frac", 1e-3), ("pd_l0_v_frac", 1e-3), ("pd_l0_k_maxulp", 2.0),
    ("pd_l0_v_maxulp", 1.0), ("pd_l0_k_err_over_tol", 1.0), ("pd_l0_v_err_over_tol", 1.0),
    ("pd_persist_over_phase_", 1.0), ("min:pd_one_chunk_batches", 2.0), ("min:pd_multi_chunk_batches", 2.0),
    *[(f"pd_{r}_{m}", 0.0) for r in ("persist", "phase") for m in ("other_slots_changed", "counter_advance_error",
                                                                   "pos_advance_error")],
    *[(f"pd_{r}_{m}_row", 5e-2) for r in ("persist", "phase") for m in ("k", "v")],
])
def check_persist_vs_phase():
    """One event of the persistent generate kernel (b200_decode_events) against one event of the launch-per-phase loop
    (GraphGenerator._event) from the same device state, on a seeded random model of the real widths (2 event-level
    layers, 1 token-level layer).  Layer 0's new k / v are bit-identical (same projection arithmetic) and within an ulp
    of an fp64 chain; deeper layers differ only by the attention's chunking, so each layer's new k / v is scored per
    (row, head) against an fp64 event step over the snapshot's cache and the persistent kernel's error is held to the
    loop's.  Every pool slot but the new one stays as it was (slots past the context are NaN); the RNG counter advances
    by 8 per event."""
    W = _Worst("pd_")
    cfg = GM.config()
    cfg.net_config.num_hidden_layers = 2
    model = GM.cpu_model(cfg).to(DEV, dtype=BF).eval()
    V = model.tokenizer.vocab_size
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    one_chunk, multi_chunk = set(), set()
    floor, max_len = 1e-3, 4097
    for B in (1, 16):
        key, gg = model._checkout_generator(B, max_len, 1.0, 0.98, 20, None)
        try:
            assert gg.persistent_ok()
            eng, kv = gg.outer.eng, gg.kv1
            nh, D, H, page = eng.cfg.n_head, eng.cfg.head_dim, eng.cfg.hidden, kv.page
            for pos in (31, 32, 33, 63, 64, 65, 4095):
                case = f"B{B} pos{pos}"
                T = pos + 1
                target = min(160, max(1, sms * 16 // (B * nh)))          # decode_persist.cu: chunks of 32-key blocks
                chunk = ((T + target - 1) // target + 31) // 32 * 32
                (one_chunk if (T + chunk - 1) // chunk == 1 else multi_chunk).add(B)
                g = torch.Generator(device=DEV).manual_seed(pos + B)
                prompt = torch.randint(0, V, (B, pos + 1, 8), generator=g, device=DEV)
                gg._set_state(prompt)                                  # events 0 .. pos-1 cached, event pos fed next
                past = (torch.arange(kv.max_pages * page, device=DEV) >= pos).view(1, kv.max_pages, 1, page, 1)
                for pool in kv.k + kv.v:
                    pool.view(B, kv.max_pages, nh, page, D).masked_fill_(past, float("nan"))
                snap = [t.clone() for t in kv.k + kv.v + [gg.pos, gg.ev_in, gg.counter, gg.seq]]
                slot = (torch.arange(kv.max_pages * page, device=DEV) == pos).view(1, kv.max_pages, 1, page, 1)
                slot = slot.expand(B, kv.max_pages, nh, page, D).reshape(kv.k[0].shape)
                runs = {}
                for name in ("persist", "phase"):
                    for t, s in zip(kv.k + kv.v + [gg.pos, gg.ev_in, gg.counter, gg.seq], snap):
                        t.copy_(s)
                    if name == "persist":
                        gg._events_persistent(1)
                    else:
                        gg._event()
                    torch.cuda.synchronize()
                    pools = kv.k + kv.v
                    changed = sum(float((~_same(p_, s_) & ~slot).sum()) for p_, s_ in zip(pools, snap))
                    new = [p_.view(B, kv.max_pages, nh, page, D)[:, pos // page, :, pos % page].clone() for p_ in pools]
                    W.add(name, case, {"other_slots_changed": changed,
                                       "counter_advance_error": abs(int(gg.counter[0]) - int(snap[-2][0]) - 8),
                                       "pos_advance_error": abs(int(gg.pos) - pos - 1)})
                    runs[name] = new
                L = len(eng.layers)
                e = ops.embed_sum(snap[-3], eng.embed)
                ref = _event_step64(eng, e, snap[:L], snap[L:2 * L], kv.block_table, page, pos, gg.outer.cos, gg.outer.sin)
                # layer 0: bit-identical, and within an ulp of the fp64 chain with the kernels' rounding points
                l0 = float(sum((runs["persist"][i] != runs["phase"][i]).sum() for i in (0, L)))
                W.add("", case, {"l0_kv_persist_vs_phase_mismatch": l0})
                w0 = eng.layers[0]
                acc = _rms_chain64(e, w0.ln1, eng.cfg.eps) @ w0.qkv.double().T
                kpre = P.round_bf16(acc[:, H:2 * H]).view(B, nh, D).to(BF)
                kch, mag = _rope_chain64(kpre, gg.outer.cos, gg.outer.sin, pos)
                W.add("l0_k", case, P.exact_metrics(runs["persist"][0], kch, kch.to(torch.float32).to(BF), inter=mag))
                W.add("l0_v", case, P.exact_metrics(runs["persist"][L], acc[:, 2 * H:].view(B, nh, D)))
                # every layer against the fp64 event step
                for li in range(L):
                    atol = 1e-3 * float(ref[li][1].norm(dim=-1).median())
                    err = {n_: (P.row_worst(runs[n_][li], ref[li][0], atol=atol),
                                P.row_worst(runs[n_][L + li], ref[li][1], atol=atol)) for n_ in runs}
                    for n_ in runs:
                        W.add(n_, case, {"k_row": err[n_][0], "v_row": err[n_][1]})
                    W.add("persist_over_phase", case, {"k": err["persist"][0] / (1.5 * err["phase"][0] + floor),
                                                       "v": err["persist"][1] / (1.5 * err["phase"][1] + floor)})
        finally:
            model._return_generator(key, gg)
    out = W.report()
    out["pd_one_chunk_batches"], out["pd_multi_chunk_batches"] = float(len(one_chunk)), float(len(multi_chunk))
    return out


# ------------------------------------------------------------------------------------------ persistent kernel, token level
PT_SIZES = (1, 2, 3, 4, 5, 8, 9, 16)         # every batch tile BM (1, 2, 4, 8, 16), full and partly filled
PT_POS = (31, 64, 65, 4095)
PT_MAX_LEN = 4097
PT_PLAIN = ((1.0, 0.98, 20), (1.7, 1.0, 64), (0.5, 0.5, 2))      # (temp, top_p, top_k) of b200_decode_events
PT_RAGGED, PT_QUEUE = (1.0, 0.98, 20), (1.7, 0.5, 64)
PT_ROW_TEMP, PT_ROW_TOP_P, PT_ROW_TOP_K = (0.5, 1.0, 1.7), (1.0, 0.98, 0.5, 0.1), (1, 2, 20, 64)


def _pt_models(names=("base", "peaked")):
    """persist_vs_phase's seeded random model of the real widths with 2 event-level and 2 token-level layers ("base"), and
    the same model with an 8x lm_head ("peaked": its peaked logits make top-p cut, EOS and short events occur and the
    temperature matter)."""
    cfg = GM.config()
    cfg.net_config.num_hidden_layers = 2
    cfg.net_token_config.num_hidden_layers = 2
    out = {}
    for name in names:
        m = GM.cpu_model(cfg)
        if name == "peaked":
            with torch.no_grad():
                m.lm_head.weight.mul_(8.0)
        out[name] = m.to(DEV, dtype=BF).eval()
    return out


def _ragged_offsets(B, pos):
    """Row offsets of the ragged / queue tests: 0, -1, -31, -32, -33 and the largest spread (a row at position 0),
    clipped to positions >= 0."""
    cyc = [0, -1, -31, -32, -33, -pos]
    return [max(cyc[b % len(cyc)], -pos) for b in range(B)]


def _pt_launch(gg, kind, n):
    """n events of the persistent kernel's entry `kind` (plain / ragged / queue / rows) on gg's state, without an exit on a
    finished row."""
    import ctypes
    d, ws, _ = gg._persistent()
    dp, w = ctypes.byref(d), (ws.data_ptr(), ws.numel())
    if kind == "plain":
        lib.call("b200_decode_events", dp, n, *w, lib.stream())
    elif kind == "ragged":
        lib.call("b200_decode_events_ragged", dp, gg.row_off.data_ptr(), n, *w, lib.stream())
    elif kind == "queue":
        lib.call("b200_decode_events_queue", dp, gg.row_off.data_ptr(), gg.row_end.data_ptr(), gg.row_last.data_ptr(), 0, n,
                 *w, lib.stream())
    else:
        lib.call("b200_decode_events_queue_rows", dp, gg.row_off.data_ptr(), gg.row_end.data_ptr(), gg.row_last.data_ptr(),
                 0, n, *w, gg.row_temp.data_ptr(), gg.row_top_p.data_ptr(), gg.row_top_k.data_ptr(), gg.row_seed.data_ptr(),
                 gg.row_first.data_ptr(), lib.stream())


def _pt_masks(gg, kinds, seed):
    """gg.mask rows by kind: 0 every id allowed; 1 a random 40 % of the parameter ids denied; 2 every event type denied
    but EOS (an all-pad event); 3 EOS and every event type but the 7-parameter note denied (8 steps)."""
    g = gg.g
    ev = torch.arange(g.eos + 1, g.eos + 1 + g.n_event_types, device=DEV)
    note = next(e for e, n_ in g.n_params.items() if n_ == 7)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    gg.mask.fill_(1)
    for b, k in enumerate(kinds):
        if k == 1:
            deny = torch.rand(gg.V, generator=gen, device=DEV) < 0.4
            deny[:g.eos + 1 + g.n_event_types] = False
            gg.mask[b, deny] = 0
        elif k == 2:
            gg.mask[b, ev] = 0
        elif k == 3:
            gg.mask[b, ev[ev != note]] = 0
            gg.mask[b, g.eos] = 0


def _pt_state(gg, pools0, prompt, pos, offs, live, c0):
    """Device state of one event: the prefilled pools with every slot from row b's new position on (and every slot of a
    row that is not live) NaN, row b at pos + offs[b] fed its prompt event there, seq all -5.  Returns the pools as set."""
    kv, B = gg.kv1, gg.B
    nh, D, page, mp = kv.cfg.n_head, kv.cfg.head_dim, kv.page, kv.max_pages
    ctx = torch.tensor([pos + o for o in offs], device=DEV)
    past = (torch.arange(mp * page, device=DEV)[None] >= ctx[:, None]) | ~torch.tensor(live, device=DEV)[:, None]
    pre = []
    for pool, s in zip(kv.k + kv.v, pools0):
        pool.copy_(s)
        pool.view(B, mp, nh, page, D).masked_fill_(past.view(B, mp, 1, page, 1), float("nan"))
        pre.append(pool.clone())
    gg.pos.fill_(pos)
    gg.ev_in.copy_(prompt[torch.arange(B, device=DEV), ctx])
    gg.counter.copy_(torch.tensor([c0, gg.seed], dtype=torch.int64))
    gg.seq.fill_(-5)
    gg.row_off.copy_(torch.tensor(offs, dtype=torch.int32))
    return pre


def _pt_loop(gg, x, ev_t, n):
    """The launch-per-phase loop's token-level half (GraphGenerator._event) from the event-level output x, teacher-forced
    with the tokens ev_t [8, B] (ids outside [0, V) read row 0, as the persistent kernel does): returns the token-level
    cache (a fresh PagedKV of page 8) and each step's logits [n, B, V]."""
    from midi_b200 import decode as dec
    eng, B, V = gg.inner.eng, gg.B, gg.V
    hidden = ops.rmsnorm(x, gg.outer.eng.norm, gg.outer.eng.cfg.eps)
    kv2 = dec.PagedKV(eng.cfg, B, 8, 8, DEV)
    logits = []
    for i in range(n):
        if i == 0:
            xin = ops.inner_input(hidden, None, eng.embed)
        else:
            ids = ev_t[i - 1].clone()
            ids[(ids < 0) | (ids >= V)] = 0
            xin = ops.inner_input(None, ids.view(B, 1), eng.embed)
        hs = gg.inner.step(xin, kv2, 1, final_norm=False)
        logits.append(dec._gemv_fused(hs, gg.lm_head, V, norm_w=eng.norm, eps=eng.cfg.eps, ldy=gg.pitch)[:, :V])
    return kv2, torch.stack(logits)


def _pt_ws(ws, L, name, dtype, shape):
    n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
    return ws[L[name]:L[name] + n].clone().view(dtype).view(shape)


# H100 80GB HBM3, 700 W: the token-level half was bit-identical to the launch-per-phase kernels (k / v of every step and
# layer, last logits) and all 15912 unambiguous draws were the restated ones; 3.1 % of the draws were ambiguous (a
# candidate's fp64 p within 2^-17 of a bf16 midpoint), bound about 5x.  Worst row against fp64: x 9.1e-3, k2 9.1e-3,
# v2 8.7e-3, last logits 7.6e-3, bounds about 5x.  The counters' minimums are about 80 % of the counts measured there
# (unambiguous 15912, top-p cuts 89, top_k 1 / 2 / 20 / 64: 644 / 3404 / 6325 / 5539, ties 3998, EOS rows 665, 8-step
# events 316, 2-step events 25); the masked, not-live and fp64 counts follow from the case set alone.
@bounded([
    ("pt_ws_layout_error", 0.0), ("pt_k_loop_mismatch", 0.0), ("pt_v_loop_mismatch", 0.0), ("pt_logits_loop_mismatch", 0.0),
    ("pt_nan_read", 0.0), ("pt_draw_mismatch", 0.0), ("pt_ambiguous_frac", 0.15), ("pt_n_steps_error", 0.0),
    ("pt_not_live_token_not_pad", 0.0), ("pt_seq_mismatch", 0.0), ("pt_ev_in_mismatch", 0.0), ("pt_pos_advance_error", 0.0),
    ("pt_counter_advance_error", 0.0), ("pt_row_last_error", 0.0), ("pt_other_slots_changed", 0.0),
    ("pt_f64_x_row", 4.5e-2), ("pt_f64_k_row", 4.5e-2), ("pt_f64_v_row", 4.5e-2), ("pt_f64_logits_row", 4e-2),
    ("min:pt_count_bm", 5.0), ("min:pt_count_unambiguous", 12000.0), ("min:pt_count_topp_cut", 60.0),
    ("min:pt_count_topk1_draws", 500.0), ("min:pt_count_topk2_draws", 2500.0), ("min:pt_count_topk20_draws", 5000.0),
    ("min:pt_count_topk64_draws", 4000.0), ("min:pt_count_tie", 3000.0), ("min:pt_count_eos_rows", 500.0),
    ("min:pt_count_8_step_events", 250.0), ("min:pt_count_2_step_events", 15.0), ("min:pt_count_masked_rows", 1554.0),
    ("min:pt_count_not_live_rows", 208.0), ("min:pt_count_f64_cases", 128.0),
])
def check_persist_token_exact():
    """One event of the persistent generate kernel per launch -- b200_decode_events at several settings, _ragged, _queue
    with rows that are not live, _queue_rows with per-row settings, seeds and row_first -- at every batch tile, scored step
    by step.  The workspace is 0xFF-filled (NaN in bf16) before the launch; afterwards its x, logits, ev_t, k2 and v2
    (decode_reference.decode_ws_layout) are read.  From the kernel's own x and tokens, the launch-per-phase loop's calls
    (RMSNorm, inner_input, the token-level step, the fused lm_head) must reproduce every token-level k / v and the last
    logits bit for bit; every sampling decision must be decode_reference.logits_sample of the loop's logits in the
    restated grammar range with the restated uniform; the step count, commit, positions, counter, row_last and pool
    slots must be the restated ones; x, k2 / v2 and the logits are anchored to an fp64 event step and token steps."""
    import ctypes
    import decode_reference as DR
    W = _Worst("pt_")
    cnt = {k: 0 for k in ("unambiguous", "topp_cut", "topk1_draws", "topk2_draws", "topk20_draws", "topk64_draws", "tie",
                          "eos_rows", "8_step_events", "2_step_events", "masked_rows", "not_live_rows", "f64_cases")}
    bms, n_dec, n_amb = set(), 0, 0
    for mname, model in _pt_models().items():
        V = model.tokenizer.vocab_size
        for B in PT_SIZES:
            key, gg = model._checkout_generator(B, PT_MAX_LEN, 1.0, 0.98, 20, None)
            d, ws, _ = gg._persistent()
            scalar = (d.temp, d.top_p, d.top_k)
            try:
                assert gg.persistent_ok()
                gg.alloc_rows()
                bms.add(1 if B <= 1 else 2 if B <= 2 else 4 if B <= 4 else 8 if B <= 8 else 16)
                L = DR.decode_ws_layout(d.batch, d.H, d.I_outer, d.I_inner, d.pitch, d.nh_outer, d.n_inner)
                W.add("", f"B{B}", {"ws_layout_error": abs(L["total"] - lib.load().b200_decode_events_workspace_bytes(
                    ctypes.byref(d)))})
                kv, g = gg.kv1, gg.g
                lut, eos, pad, n_ty = g.lut.cpu().numpy(), g.eos, g.pad, g.n_event_types
                H, n_in = d.H, d.n_inner
                nh2, D2 = gg.inner.eng.cfg.n_head, gg.inner.eng.cfg.head_dim
                nl = len(kv.k)
                for pos in PT_POS:
                    gen = torch.Generator(device=DEV).manual_seed(pos * 17 + B)
                    prompt = torch.randint(0, V, (B, pos + 1, 8), generator=gen, device=DEV)
                    gg._set_lengths(prompt, None)
                    gg._set_state(prompt)
                    pools0 = [t.clone() for t in kv.k + kv.v]
                    variants = [("plain", s) for s in PT_PLAIN] + [("ragged", PT_RAGGED), ("queue", PT_QUEUE), ("rows", None)]
                    for vi, (kind, sc) in enumerate(variants):
                        case = f"{mname} B{B} pos{pos} {kind}{vi}"
                        offs = [0] * B if kind == "plain" else _ragged_offsets(B, pos)
                        queue = kind in ("queue", "rows")
                        live = [not (queue and b % 3 == 2) for b in range(B)]
                        ctx = [pos + o for o in offs]
                        c0 = 3 + pos + vi
                        pre = _pt_state(gg, pools0, prompt, pos, offs, live, c0)
                        kinds = [(b + vi + pos) % 4 for b in range(B)]
                        _pt_masks(gg, kinds, seed=pos + 31 * vi + B)
                        if kind == "rows":
                            settings = [(PT_ROW_TEMP[(b + vi) % 3], PT_ROW_TOP_P[(b + pos) % 4], PT_ROW_TOP_K[(b + pos // 2) % 4])
                                        for b in range(B)]
                            first = [max(0, ctx[b] - (3 * b + pos) % 11) for b in range(B)]
                            seeds = [(1000003 * (b + 1) + 7919 * pos + vi) & ((1 << 62) - 1) for b in range(B)]
                            gg.row_temp.copy_(torch.tensor([s[0] for s in settings]))
                            gg.row_top_p.copy_(torch.tensor([s[1] for s in settings]))
                            gg.row_top_k.copy_(torch.tensor([s[2] for s in settings], dtype=torch.int32))
                            gg.row_seed.copy_(torch.tensor(seeds, dtype=torch.int64))
                            gg.row_first.copy_(torch.tensor(first, dtype=torch.int32))
                        else:
                            settings = [sc] * B
                            d.temp, d.top_p, d.top_k = sc
                        row_end = [ctx[b] + 1 if b % 4 == 1 else PT_MAX_LEN - 1 for b in range(B)]
                        row_last = [-1 if live[b] else (-2 if b % 2 else ctx[b]) for b in range(B)]
                        gg.row_end.copy_(torch.tensor(row_end, dtype=torch.int32))
                        gg.row_last.copy_(torch.tensor(row_last, dtype=torch.int32))
                        ev_in0, mask_np = gg.ev_in.clone(), gg.mask.cpu().numpy()
                        ws.fill_(255)
                        _pt_launch(gg, kind, 1)
                        torch.cuda.synchronize()
                        x = _pt_ws(ws, L, "x", BF, (B, H))
                        lg = _pt_ws(ws, L, "logits", BF, (B, d.pitch))[:, :V]
                        evt = _pt_ws(ws, L, "ev_t", torch.int64, (8, B))
                        k2 = _pt_ws(ws, L, "k2", BF, (n_in, B, 8, H))
                        v2 = _pt_ws(ws, L, "v2", BF, (n_in, B, 8, H))
                        evt_np = evt.cpu().numpy()
                        n = 0
                        while n < 8 and (evt_np[n] != -1).all():
                            n += 1
                        n_want = DR.event_n_steps(evt_np[0], live, lut, eos, n_ty)
                        lv = torch.tensor(live, device=DEV)
                        m = {"n_steps_error": abs(n - n_want),
                             "nan_read": float(torch.isnan(x[lv]).sum() + torch.isnan(lg[lv]).sum()
                                               + torch.isnan(k2[:, lv, :n]).sum() + torch.isnan(v2[:, lv, :n]).sum()),
                             "not_live_token_not_pad": float((evt_np[:n][:, ~np.array(live)] != pad).sum())}
                        # ---- 1. the token-level half against the launch-per-phase kernels, bit for bit
                        kv2, llog = _pt_loop(gg, x, evt, max(n, 1))
                        for nm, pools, kern in (("k", kv2.k, k2), ("v", kv2.v, v2)):
                            bad = 0.0
                            for li in range(n_in):
                                lp = pools[li].view(B, nh2, 8, D2).permute(0, 2, 1, 3).reshape(B, 8, H)
                                bad += _ne(kern[li][lv, :n], lp[lv, :n])
                            m[f"{nm}_loop_mismatch"] = bad
                        m["logits_loop_mismatch"] = _ne(lg[lv], llog[max(n, 1) - 1][lv])
                        # ---- 2. every sampling decision
                        if kind == "rows":
                            u = DR.event_uniforms("rows", B, max(n, 1), pos=pos, row_off=offs, row_first=first, row_seed=seeds)
                        else:
                            u = DR.event_uniforms(kind, B, max(n, 1), c0=c0, seed=gg.seed)
                        dec_ = DR.event_decisions(llog.float().cpu().numpy(), evt_np, n, live, settings, mask_np, u, lut,
                                                  eos, pad, n_ty)
                        isdec = dec_["id"] >= 0
                        clear = isdec & ~dec_["amb"]
                        m["draw_mismatch"] = float((clear & (dec_["id"] != evt_np[:n])).sum())
                        n_dec += int(isdec.sum())
                        n_amb += int((isdec & dec_["amb"]).sum())
                        cnt["unambiguous"] += int(clear.sum())
                        cnt["topp_cut"] += int((clear & dec_["cut"]).sum())
                        cnt["tie"] += int((clear & dec_["tie"]).sum())
                        for k_ in PT_ROW_TOP_K:
                            cnt[f"topk{k_}_draws"] += int(clear[:, [s[2] == k_ for s in settings]].sum())
                        # ---- 3. event bookkeeping
                        _, seq_w, ev_w = DR.event_commit_rows(evt_np, n_want, live, np.full((B, PT_MAX_LEN, 8), -5),
                                                              ev_in0.cpu().numpy(), pos, offs, pad)
                        m["seq_mismatch"] = float((gg.seq.cpu().numpy() != seq_w).sum())
                        m["ev_in_mismatch"] = float((gg.ev_in.cpu().numpy() != ev_w).sum())
                        m["pos_advance_error"] = abs(int(gg.pos) - pos - 1)
                        m["counter_advance_error"] = abs(int(gg.counter[0]) - c0 - 8) + abs(int(gg.counter[1]) - gg.seed)
                        if queue:
                            want_last = [(ctx[b] + 1 if evt_np[0, b] == eos or ctx[b] + 1 >= row_end[b] else -1)
                                         if live[b] else row_last[b] for b in range(B)]
                            m["row_last_error"] = float(sum(a != w_ for a, w_ in zip(gg.row_last.tolist(), want_last)))
                        slot = DR.slot_mask(pre[0].shape, kv.block_table, kv.page, [(b, ctx[b]) for b in range(B) if live[b]])
                        m["other_slots_changed"] = sum(float((~_same(p_, s_) & ~slot).sum()) for p_, s_ in zip(kv.k + kv.v, pre))
                        W.add("", case, m)
                        cnt["eos_rows"] += sum(1 for b in range(B) if live[b] and evt_np[0, b] == eos)
                        cnt["8_step_events"] += int(n == 8)
                        cnt["2_step_events"] += int(n == 2)
                        cnt["masked_rows"] += sum(1 for b in range(B) if live[b] and kinds[b] != 0)
                        cnt["not_live_rows"] += B - sum(live)
                        # ---- 4. fp64 anchors (the first plain setting and the per-row kernel)
                        if vi == 0 or kind == "rows":
                            cnt["f64_cases"] += 1
                            e = ops.embed_sum(ev_in0, gg.outer.eng.embed)
                            _, x64 = _event_step64(gg.outer.eng, e, pre[:nl], pre[nl:], kv.block_table, kv.page, ctx,
                                                   gg.outer.cos, gg.outer.sin, want_x=True)
                            k64, v64, lg64 = _token_steps64(gg.inner.eng, gg.lm_head, gg.outer.eng.norm, x, evt, max(n, 1),
                                                            gg.inner.cos, gg.inner.sin)
                            f = {"x_row": P.row_worst(x[lv], x64[lv]),
                                 "logits_row": P.row_worst(lg[lv], lg64[lv, max(n, 1) - 1])}
                            for nm, kern, ref in (("k", k2, k64), ("v", v2, v64)):
                                got = kern[:, lv, :n].reshape(n_in, -1, n, nh2, D2)
                                f[f"{nm}_row"] = P.row_worst(got, ref[:, lv, :n])
                            W.add("f64", case, f)
            finally:
                d.temp, d.top_p, d.top_k = scalar
                gg.set_deny(())
                model._return_generator(key, gg)
    out = W.report()
    out["pt_ambiguous_frac"] = n_amb / max(n_dec, 1)
    out["pt_count_bm"] = float(len(bms))
    for k_, v_ in cnt.items():
        out[f"pt_count_{k_}"] = float(v_)
    for k_ in sorted(out):
        if k_.startswith("pt_count") or k_ == "pt_ambiguous_frac":
            print(f"  {k_} = {out[k_]:.4g}")
    return out


@bounded([("min:pm_count_cases", 12.0), ("min:pm_count_in_kernel_exits", 6.0), ("pm_", 0.0)])
def check_persist_multi_event():
    """One launch of 3 events of the persistent kernel against three launches of one, from the same state, for the plain,
    ragged and per-row kernels: seq, ev_in, every pool, pos, the RNG counter and row_last must agree bit for bit.  This is
    the in-kernel hand-over between events (cur_ev, pos++, the counter with events_done, rows that finish); a snapshot at
    pos = max_len - 3 runs the in-kernel `pos + 1 >= max_len` exit inside the launch."""
    W = _Worst("pm_")
    model = _pt_models(("peaked",))["peaked"]
    V = model.tokenizer.vocab_size
    n_cases = n_exits = 0
    for B in (3, 16):
        key, gg = model._checkout_generator(B, PT_MAX_LEN, 1.0, 0.98, 20, None)
        try:
            gg.alloc_rows()
            kv = gg.kv1
            for pos in (65, PT_MAX_LEN - 3):
                gen = torch.Generator(device=DEV).manual_seed(pos + 5 * B)
                prompt = torch.randint(0, V, (B, pos + 1, 8), generator=gen, device=DEV)
                gg._set_lengths(prompt, None)
                gg._set_state(prompt)
                pools0 = [t.clone() for t in kv.k + kv.v]
                for kind in ("plain", "ragged", "rows"):
                    offs = [0] * B if kind == "plain" else _ragged_offsets(B, pos)
                    live = [not (kind == "rows" and b % 3 == 2) for b in range(B)]
                    ctx = [pos + o for o in offs]
                    _pt_state(gg, pools0, prompt, pos, offs, live, c0=11 + pos)
                    # row 0 never finishes (no EOS, no budget), so every launch has a live row
                    _pt_masks(gg, [0] + [b % 4 for b in range(1, B)], seed=pos + B)
                    gg.mask[0, gg.g.eos] = 0
                    if kind == "rows":
                        gg.row_temp.copy_(torch.tensor([PT_ROW_TEMP[b % 3] for b in range(B)]))
                        gg.row_top_p.copy_(torch.tensor([PT_ROW_TOP_P[b % 4] for b in range(B)]))
                        gg.row_top_k.copy_(torch.tensor([PT_ROW_TOP_K[(b + 2) % 4] for b in range(B)], dtype=torch.int32))
                        gg.row_seed.copy_(torch.tensor([977 * b + pos for b in range(B)], dtype=torch.int64))
                        gg.row_first.copy_(torch.tensor([max(0, c - b % 5) for b, c in enumerate(ctx)], dtype=torch.int32))
                        gg.row_end.copy_(torch.tensor([c + 2 if b % 4 == 1 else PT_MAX_LEN - 1 for b, c in enumerate(ctx)],
                                                      dtype=torch.int32))
                        gg.row_last.copy_(torch.tensor([-1 if live[b] else -2 for b in range(B)], dtype=torch.int32))
                    state = kv.k + kv.v + [gg.seq, gg.ev_in, gg.pos, gg.counter, gg.row_last]
                    snap = [t.clone() for t in state]
                    runs = []
                    for split in (False, True):
                        for t, s in zip(state, snap):
                            t.copy_(s)
                        for _ in range(3 if split else 1):
                            _pt_launch(gg, kind, 1 if split else 3)
                        torch.cuda.synchronize()
                        runs.append([t.clone() for t in state])
                    one, three = runs
                    n_run = int(one[-3]) - pos
                    W.add("", f"B{B} pos{pos} {kind}", {
                        "one_vs_three_mismatch": sum(float((~_same(a, b_)).sum()) for a, b_ in zip(one, three)),
                        "events_run_error": abs(n_run - min(3, PT_MAX_LEN - 1 - pos))})
                    n_cases += 1
                    n_exits += int(n_run < 3)
        finally:
            gg.set_deny(())
            model._return_generator(key, gg)
    out = W.report()
    out["pm_count_cases"], out["pm_count_in_kernel_exits"] = float(n_cases), float(n_exits)
    return out


# ------------------------------------------------------------------------------------------ train-step conformance groups
# The rest of the train step -- embeddings, RMSNorm, RoPE, SwiGLU, token-level attention, cross-entropy, grad clip and
# AdamW (elementwise.cu, attn_tiny.cu, train_misc.cu) -- through the C ABI, as the groups above treat the GEMM, attention
# and decode kernels: every dispatch variant, operands in NaN-poisoned buffers, outputs in NaN buffers, scored per
# element (or per attention row) against the fp64 restatements of tests/parity_metrics.py rounded at the kernels' own
# rounding points (DESIGN.md 3.3).
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ne(a, b):
    """Number of elements that differ (a NaN differs from everything)."""
    return float((a != b).sum())


# all copies and the fp32 gather-sum in the kernel's order are exact claims.  Against fp64, H100 80GB HBM3 at 700 W: the
# gather-sum and the backward (fp32 segment sums in an order the atomics choose, one rounding; accumulate one more)
# were correctly rounded in every element (frac 0, err_over_tol <= 0.50); the bounds allow a rare fp32 rounding to
# reach the bf16 result (frac 1e-3 / 2e-3, one ulp, two with accumulate's second rounding)
@bounded([
    ("em_sentinels_changed", 0.0), ("em_nan_in_range", 0.0), ("em_sum_vs_seq32_mismatch", 0.0),
    ("em_inner_mismatch", 0.0), ("em_rows_mismatch", 0.0), ("em_rows_ysel_mismatch", 0.0),
    ("em_rows_bwd_mismatch", 0.0), ("em_bwd_padrow_changed", 0.0), ("em_bwd_empty_mismatch", 0.0),
    ("min:em_bwd_cases", 16.0), ("min:em_bwd_capped_ids", 4.0), ("min:em_bwd_multislice_ids", 8.0),
    ("em_sum_frac", 1e-3), ("em_sum_maxulp", 1.0), ("em_bwd_frac", 2e-3), ("em_bwd_maxulp", 1.0),
    ("em_bwdacc_frac", 2e-3), ("em_bwdacc_maxulp", 2.0),
    *[(f"em_{f}_err_over_tol", 1.0) for f in ("sum", "bwd", "bwdacc")],
])
def check_embed_conformance():
    """b200_embed_sum_fwd (T = 1 / 8, ids -1 / V / 1e12 skipped, NaN table rows past V), b200_inner_input_fwd with and
    without hidden (out-of-range ids read row 0), b200_inner_input_rows_fwd / _rows_bwd_hidden (rows outside [0, n_rows)
    and inv = -1 give zero rows), and b200_embed_bwd in the model's two layouts (outer: 8 ids per gradient row; inner: 7
    ids per event at rows e*8 + 1 + j, the never-read rows e*8 NaN) with one id in one slice (40 occurrences), one in
    many (500: red.add) and one past the 32-slice cap (5000), V = 3406 / 5000 (4 / 5 scan items per thread), pad_id 0 /
    17, accumulate 0 / 1, skipped ids -1 / V and n_ids = 0."""
    W = _Worst("em_")
    H = 1032                    # 129 vectors of 8: the 128-thread CTAs take a second vector
    V = 3406
    table = P.nan_buffer((V + 2, H), device=DEV)     # rows V, V + 1 NaN: an unclamped id reads them
    table[:V] = randn(V, H, scale=0.02, seed=6000)
    bad = torch.tensor([-1, V, 10 ** 12, V + 1], device=DEV)
    # ---- gather-sum: one fp32 sum in t order, one rounding
    for T in (1, 8):
        M = 301
        ids = torch.randint(0, V, (M, T), generator=_gen(6001 + T), device=DEV)
        flat = ids.view(-1)
        flat[::7] = bad[torch.arange(flat[::7].numel(), device=DEV) % 4]
        out = P.nan_buffer((M + 2, H), device=DEV)
        lib.call("b200_embed_sum_fwd", ids.data_ptr(), table.data_ptr(), out.data_ptr(), M, T, H, V, lib.stream())
        ok = ((ids >= 0) & (ids < V))[..., None]
        rows = table[ids.clamp(0, V - 1)]
        seq = torch.zeros(M, H, device=DEV)
        for t in range(T):
            seq = seq + torch.where(ok[:, t], rows[:, t].float(), torch.zeros_like(seq))
        case = f"sum T{T}"
        W.add("sum", case, P.exact_metrics(out[:M], torch.where(ok, rows.double(), 0.0).sum(1)))
        W.add("", case, {"sum_vs_seq32_mismatch": _ne(out[:M], seq.to(BF))})
        W.add("", case, P.sentinel_report(out, (slice(0, M),)))
    # ---- inner input builder: copies, out-of-range ids read row 0
    E, n_ids = 57, 7
    ids = torch.randint(0, V, (E, n_ids), generator=_gen(6010), device=DEV)
    ids[::5, 2] = bad[torch.arange(ids[::5].shape[0], device=DEV) % 4]
    hid = randn(E, H, seed=6011)
    emb = table[torch.where((ids >= 0) & (ids < V), ids, 0)]
    for has_hidden in (0, 1):
        Tin = n_ids + has_hidden
        out = P.nan_buffer((E * Tin + 2, H), device=DEV)
        lib.call("b200_inner_input_fwd", hid.data_ptr() if has_hidden else None, ids.data_ptr(), table.data_ptr(),
                 out.data_ptr(), E, n_ids, H, V, lib.stream())
        ref = (torch.cat([hid[:, None], emb], 1) if has_hidden else emb).reshape(-1, H)
        case = f"inner hidden{has_hidden}"
        W.add("", case, {"inner_mismatch": _ne(out[:E * Tin], ref)})
        W.add("", case, P.sentinel_report(out, (slice(0, E * Tin),)))
    # ---- --sample-seq rows: unique selected rows, rows -1 / n_rows read nothing
    n_rows, T = 90, 8
    hid = randn(n_rows, H, seed=6020)
    y = torch.randint(0, V, (n_rows, T), generator=_gen(6021), device=DEV)
    y[::4, 3] = bad[torch.arange(y[::4].shape[0], device=DEV) % 4]
    sel = torch.randperm(n_rows, generator=_gen(6022), device=DEV)[:40].int()
    sel[5], sel[17] = -1, n_rows
    n = sel.numel()
    out = P.nan_buffer((n * T + 2, H), device=DEV)
    y_sel = torch.full((n * T + 5,), -777, dtype=torch.long, device=DEV)
    lib.call("b200_inner_input_rows_fwd", hid.data_ptr(), y.data_ptr(), sel.data_ptr(), table.data_ptr(), out.data_ptr(),
             y_sel.data_ptr(), n, n_rows, T, H, V, lib.stream())
    live = (sel >= 0) & (sel < n_rows)
    r = sel.long().clamp(0, n_rows - 1)
    yr = y[r]
    ref = torch.cat([hid[r][:, None], table[torch.where((yr[:, :-1] >= 0) & (yr[:, :-1] < V), yr[:, :-1], 0)]], 1)
    ref = torch.where(live[:, None, None], ref, torch.zeros_like(ref)).reshape(n * T, H)
    ysel_ref = torch.where(live[:, None], yr, torch.full_like(yr, -1)).reshape(-1)
    W.add("", "rows fwd", {"rows_mismatch": _ne(out[:n * T], ref),
                           "rows_ysel_mismatch": _ne(y_sel[:n * T], ysel_ref) + _ne(y_sel[n * T:], -777)})
    W.add("", "rows fwd", P.sentinel_report(out, (slice(0, n * T),)))
    # backward for hidden: only rows e * Tin of dx are read (the rest NaN)
    Tin = T
    dx = P.nan_buffer((n * Tin + 3, H), device=DEV)
    dx[0:n * Tin:Tin] = randn(n, H, seed=6023)
    inv = torch.full((n_rows,), -1, dtype=torch.int32, device=DEV)
    inv[sel[live].long()] = torch.arange(n, device=DEV, dtype=torch.int32)[live]
    dh = P.nan_buffer((n_rows + 2, H), device=DEV)
    lib.call("b200_inner_input_rows_bwd_hidden", dx.data_ptr(), inv.data_ptr(), dh.data_ptr(), n_rows, n, Tin, H,
             lib.stream())
    ref = torch.where((inv >= 0)[:, None], dx[inv.long().clamp(0) * Tin], torch.zeros(n_rows, H, dtype=BF, device=DEV))
    W.add("", "rows bwd", {"rows_bwd_mismatch": _ne(dh[:n_rows], ref)})
    W.add("", "rows bwd", P.sentinel_report(dh, (slice(0, n_rows),)))
    # ---- embedding backward
    n_cases = capped = multi = 0
    hot = {40: 123, 500: 2001, 5000: 3}             # occurrences -> id
    for V in (3406, 5000):
        for layout in ("outer", "inner"):
            per_row, row_stride, row_inner, row_off = (8, 1, 0, 0) if layout == "outer" else (7, 8, 1, 1)
            n_ev = 1000 if layout == "outer" else 1100
            n = n_ev * per_row
            g = _gen(6100 + V + per_row)
            ids = torch.randint(0, V, (n,), generator=g, device=DEV)
            pos = torch.randperm(n, generator=g, device=DEV)
            k = 0
            for occ, vid in hot.items():
                ids[pos[k:k + occ]] = vid
                k += occ
            ids[pos[k:k + 30]] = torch.tensor([-1, V], device=DEV).repeat(15)
            n_dout = n_ev * row_stride if layout == "inner" else n_ev
            dvals = randn(n_dout, H, seed=6200 + V + per_row)
            if layout == "outer":                        # gradient rows whose ids are all skipped are never read
                for rr in (4, n_ev - 1):
                    ids[rr * 8:rr * 8 + 8] = torch.tensor([-1, V] * 4, device=DEV)
                    dvals[rr] = float("nan")
            else:                                        # rows e*8 (the hidden position) are never read
                dvals[0::8] = float("nan")
            dout = P.poisoned(dvals, n_dout + 3, H)
            for pad_id in (0, 17):
                ids_p = ids.clone()
                ids_p[pos[k + 30:k + 60]] = pad_id
                ref = P.embed_bwd64(ids_p, dout, V, per_row, row_stride, row_inner, row_off, pad_id)
                nbytes = int(lib.query("b200_embed_bwd_workspace_bytes", n, V, H))
                for acc in (0, 1):
                    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)     # NaN floats, -1 ints
                    dt = P.nan_buffer((V + 2, H), device=DEV)
                    old = randn(V, H, seed=6300 + V + pad_id) if acc else None
                    if acc:
                        dt[:V] = old
                    lib.call("b200_embed_bwd", ids_p.data_ptr(), n, dout.data_ptr(), dt.data_ptr(), V, H, per_row,
                             row_stride, row_inner, row_off, pad_id, acc, ws.data_ptr(), nbytes, lib.stream())
                    case = f"V{V} {layout} pad{pad_id} acc{acc}"
                    if acc:
                        base = P.round_bf16(ref)
                        W.add("bwdacc", case, P.exact_metrics(dt[:V], base + old.double(),
                                                              (base + old.double()).to(torch.float32).to(BF), inter=ref))
                        W.add("", case, {"bwd_padrow_changed": _ne(dt[pad_id], old[pad_id])})
                    else:
                        W.add("bwd", case, P.exact_metrics(dt[:V], ref))
                        W.add("", case, {"bwd_padrow_changed": float((dt[pad_id] != 0).sum())})
                    W.add("", case, P.sentinel_report(dt, (slice(0, V),)))
                    n_cases += 1
            cnt = torch.bincount(ids[(ids >= 0) & (ids < V)], minlength=V)
            capped += int((cnt > 32 * 48).sum())
            multi += int((cnt > 48).sum())
    # n_ids = 0: zeros, or the old table when accumulating
    V = 3406
    nbytes = int(lib.query("b200_embed_bwd_workspace_bytes", 0, V, H))
    for acc in (0, 1):
        ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)
        dt = P.nan_buffer((V + 2, H), device=DEV)
        old = randn(V, H, seed=6400)
        if acc:
            dt[:V] = old
        lib.call("b200_embed_bwd", None, 0, None, dt.data_ptr(), V, H, 8, 1, 0, 0, 0, acc, ws.data_ptr(), nbytes,
                 lib.stream())
        W.add("", f"empty acc{acc}", {"bwd_empty_mismatch": _ne(dt[:V], old if acc else torch.zeros_like(old))})
        W.add("", f"empty acc{acc}", P.sentinel_report(dt, (slice(0, V),)))
    out = W.report()
    out["em_bwd_cases"], out["em_bwd_capped_ids"], out["em_bwd_multislice_ids"] = float(n_cases), float(capped), float(multi)
    return out


RN_WARP_HS = (256, 512, 1024, 2048)     # forward warp kernels (add_rmsnorm's sizes); the backward's are 256 / 512 / 1024
RN_BLOCK_HS = (200, 768, 1032, 4096)


# forward: one fp32 rstd, two roundings (bf16(x rstd), then w * that); add_rmsnorm's h_out = bf16(x + res) is exact.
# backward: dx one rounding, dw an fp32 column sum in an order the atomics choose, one rounding (two when accumulating).
# The workspace is shared by every call, as ops.rmsnorm_bwd shares it, and must be all zero after each.  H100 80GB HBM3
# at 700 W: rstd 1.6e-7 relative; y not correctly rounded 8.6e-6 (warp) / 6.3e-6 (block) / 7.1e-6 (add), <= 2 ulp, and
# err_over_tol 1.30: a flipped inner rounding (<= 2^-7 relative) plus the final half ulp can reach 1.5, the bound.  dx
# 1.6e-4, 1 ulp, 0.48; dw one element of 512 (2.0e-3), 1 ulp, 0.47.  Bounds about 5x.  Before the block path cleared its
# partials, the alternating sequence left dw unwritten (wsseq_dw_frac 1, nan_in_range 1024) and M = 0 left dw unwritten
@bounded([
    ("rn_sentinels_changed", 0.0), ("rn_nan_in_range", 0.0), ("rn_add_h_mismatch", 0.0), ("rn_ws_nonzero_after", 0.0),
    ("rn_m0_dw_mismatch", 0.0),
    ("min:rn_fwd_cases", 36.0), ("min:rn_bwd_cases", 150.0), ("min:rn_bwd_block_cases", 92.0),
    ("rn_rstd_rel", 8e-7),
    *[(f"rn_{f}_frac", 5e-5) for f in ("fwd_warp", "fwd_block", "add")],
    ("rn_dx_frac", 8e-4), *[(f"rn_{f}_frac", 1e-2) for f in ("dw", "dwacc", "wsseq_dw")],
    *[(f"rn_{f}_maxulp", 1.0) for f in ("dx", "dw", "wsseq_dw")],
    *[(f"rn_{f}_maxulp", 2.0) for f in ("fwd_warp", "fwd_block", "add", "dwacc")],
    *[(f"rn_{f}_err_over_tol", 1.5) for f in ("fwd_warp", "fwd_block", "add")],
    *[(f"rn_{f}_err_over_tol", 1.0) for f in ("dx", "dw", "dwacc", "wsseq_dw")],
])
def check_rmsnorm_conformance():
    """b200_rmsnorm_fwd at H in {256, 512, 1024, 2048} (warp kernels) and {200, 768, 1032, 4096} (block kernel),
    M in {1, 3, 5000} (5000 rows is past the grid cap: rows loop), b200_add_rmsnorm_fwd at its four sizes, and
    b200_rmsnorm_bwd at every H with dres null / set, dw null / set, accumulate_dw 0 / 1 and M = 0, all on ONE
    workspace; plus an H order that alternates the block and warp backward paths (1024, 768, 1024, 2048, 256, 1024)
    with dw in a NaN buffer, so a warp call that starts from a dirty accumulator or ticket leaves dw unwritten."""
    W = _Worst("rn_")
    eps = 1e-6
    parts = int(lib.query("b200_rmsnorm_bwd_parts"))
    ws = torch.zeros(parts * max(RN_BLOCK_HS) + 64, dtype=torch.float32, device=DEV)
    n_fwd = n_bwd = n_block = 0

    def weight(H, seed):
        w = P.nan_buffer((H + 8,), device=DEV)
        w[:H] = (1 + 0.1 * randn(H, seed=seed).float()).to(BF)
        return w

    def fwd(x, w, M, H, res=None):
        X = P.poisoned(x, M + 2, H)
        y = P.nan_buffer((M + 2, H), device=DEV)
        rstd = torch.full((M + 4,), float("nan"), device=DEV)
        if res is None:
            lib.call("b200_rmsnorm_fwd", X.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), M, H, eps, lib.stream())
            return y, rstd, None
        R = P.poisoned(res, M + 2, H)
        h = P.nan_buffer((M + 2, H), device=DEV)
        lib.call("b200_add_rmsnorm_fwd", X.data_ptr(), R.data_ptr(), w.data_ptr(), h.data_ptr(), y.data_ptr(),
                 rstd.data_ptr(), M, H, eps, lib.stream())
        return y, rstd, h

    def score_fwd(fam, case, y, rstd, x, w, M, H):
        x64 = x.double()
        r64 = 1.0 / torch.sqrt(x64.pow(2).mean(-1) + eps)
        W.add(fam, case, P.exact_metrics(y[:M], w[:H].double() * P.round_bf16(x64 * r64[:, None])))
        W.add("", case, {"rstd_rel": float(((rstd[:M].double() - r64) / r64).abs().max())})
        W.add("", case, P.sentinel_report(y, (slice(0, M),)))
        W.add("", case, P.sentinel_report(rstd, (slice(0, M),)))

    def bwd(case, dy, x, w, rstd, dres, dw, M, H, acc, fam_dw="dw"):
        nonlocal n_bwd, n_block
        DY, X = P.poisoned(dy, M + 2, H), P.poisoned(x, M + 2, H)
        DR = P.poisoned(dres, M + 2, H) if dres is not None else None
        dx = P.nan_buffer((M + 2, H), device=DEV)
        old = dw[:H].clone() if dw is not None else None
        lib.call("b200_rmsnorm_bwd", DY.data_ptr(), X.data_ptr(), w.data_ptr(), rstd.data_ptr(), lib.ptr(DR), dx.data_ptr(),
                 lib.ptr(dw), M, H, acc, ws.data_ptr(), ws.numel() * 4, lib.stream())
        dx64, dw64 = P.rmsnorm_bwd64(dy, x, w[:H], rstd[:M], dres)
        W.add("dx", case, P.exact_metrics(dx[:M], dx64))
        W.add("", case, P.sentinel_report(dx, (slice(0, M),)))
        if dw is not None:
            if acc:
                base = P.round_bf16(dw64)
                W.add(fam_dw + "acc", case, P.exact_metrics(dw[:H], base + old.double(),
                                                            (base + old.double()).to(torch.float32).to(BF), inter=dw64))
            else:
                W.add(fam_dw, case, P.exact_metrics(dw[:H], dw64))
            W.add("", case, P.sentinel_report(dw, (slice(0, H),)))
        W.add("", case, {"ws_nonzero_after": float((ws.view(torch.int32) != 0).sum())})
        n_bwd += 1
        n_block += H not in (256, 512, 1024)

    for hi, H in enumerate(RN_WARP_HS + RN_BLOCK_HS):
        w = weight(H, 7000 + H)
        fam = "fwd_warp" if H in RN_WARP_HS else "fwd_block"
        for M in (1, 3, 5000):
            x = randn(M, H, scale=3.0 if M == 3 else 1.0, seed=7100 + H + M)
            y, rstd, _ = fwd(x, w, M, H)
            score_fwd(fam, f"fwd H{H} M{M}", y, rstd, x, w, M, H)
            n_fwd += 1
            if H in RN_WARP_HS:
                res = randn(M, H, seed=7200 + H + M)
                ya, rstda, h = fwd(x, w, M, H, res)
                href = (x.float() + res.float()).to(BF)
                case = f"add H{H} M{M}"
                W.add("", case, {"add_h_mismatch": _ne(h[:M], href)})
                W.add("", case, P.sentinel_report(h, (slice(0, M),)))
                score_fwd("add", case, ya, rstda, href, w, M, H)
                n_fwd += 1
            # backward from the forward kernel's rstd: every dres / dw / accumulate combination
            dy = randn(M, H, seed=7300 + H + M)
            dres = randn(M, H, seed=7400 + H + M)
            for use_res in (0, 1):
                for mode in ("none", "acc0", "acc1"):
                    dw = None
                    if mode != "none":
                        dw = P.nan_buffer((H + 8,), device=DEV)
                        if mode == "acc1":
                            dw[:H] = randn(H, seed=7500 + H)
                    bwd(f"bwd H{H} M{M} dres{use_res} dw_{mode}", dy, x, w, rstd, dres if use_res else None, dw, M, H,
                        int(mode == "acc1"))
    # M = 0: dw = 0 (accumulate 0) or unchanged (accumulate 1); nothing else written
    for H in (1024, 768):
        w = weight(H, 7600 + H)
        for acc in (0, 1):
            old = randn(H, seed=7700 + H)
            dw = P.nan_buffer((H + 8,), device=DEV)
            dw[:H] = old
            e = torch.empty(0, dtype=BF, device=DEV)
            lib.call("b200_rmsnorm_bwd", e.data_ptr(), e.data_ptr(), w.data_ptr(), None, None, e.data_ptr(), dw.data_ptr(),
                     0, H, acc, ws.data_ptr(), ws.numel() * 4, lib.stream())
            case = f"M0 H{H} acc{acc}"
            W.add("", case, {"m0_dw_mismatch": _ne(dw[:H], old if acc else torch.zeros_like(old))})
            W.add("", case, P.sentinel_report(dw, (slice(0, H),)))
    # block and warp paths alternating on the one workspace
    for i, H in enumerate((1024, 768, 1024, 2048, 256, 1024)):
        M = 300
        w = weight(H, 7800 + i)
        x = randn(M, H, seed=7900 + i)
        _, rstd, _ = fwd(x, w, M, H)
        dw = P.nan_buffer((H + 8,), device=DEV)
        bwd(f"ws-seq #{i} H{H}", randn(M, H, seed=8000 + i), x, w, rstd, None, dw, M, H, 0, fam_dw="wsseq_dw")
    out = W.report()
    out["rn_fwd_cases"], out["rn_bwd_cases"], out["rn_bwd_block_cases"] = float(n_fwd), float(n_bwd), float(n_block)
    return out


RO_NPOS = 4096 + 64


# forward and backward are exact claims: bf16 x bf16 products are exact in fp32, so each sum rounds once to fp32 and
# then to bf16, as P.round_bf16 rounds the fp64 value (the forward at each of its three rounding points).  H100 80GB HBM3
# at 700 W: 0 mismatches both ways.  Tables (cosf / sinf of the kernel's fp32 argument, one rounding): 7.5e-6 not
# correctly rounded, 1 ulp, err_over_tol 0.42; bound about 5x
@bounded([
    ("ro_sentinels_changed", 0.0), ("ro_nan_in_range", 0.0), ("ro_fwd_mismatch", 0.0), ("ro_ragged_mismatch", 0.0),
    ("ro_v_changed", 0.0), ("min:ro_cases", 20.0),
    ("ro_table_frac", 4e-5), ("ro_table_maxulp", 1.0), ("ro_bwd_frac", 0.0), ("ro_bwd_maxulp", 0.0),
    ("ro_table_err_over_tol", 1.0), ("ro_bwd_err_over_tol", 1.0),
])
def check_rope_conformance():
    """b200_rope_table (4096 + 64 positions from pos0 = 0, pos0 > 0 and pos0_dev) against cos / sin in fp64 of the kernel's fp32
    argument; b200_rope_qk forward (0 mismatches against the three-rounding fp64 chain) and backward (the fp64 transpose
    rounded once: also exact) at head_dim 64 / 256 on rows of ld > 3H with NaN pad columns, with pos0 and pos0_dev; and
    b200_rope_qk_ragged with mixed row_off.  The v third and the pad columns are never written."""
    W = _Worst("ro_")
    n_cases = 0
    for D in (64, 256):
        half, nh = D // 2, 1024 // D
        H = nh * D
        inv = O.default_inv_freq(D).to(BF).to(DEV).float()
        for pos0, dev in ((0, None), (1000, None), (7, 4000)):
            n_pos = RO_NPOS
            c = P.nan_buffer((n_pos + 2, half), device=DEV)
            s = P.nan_buffer((n_pos + 2, half), device=DEV)
            pd = torch.tensor([dev], dtype=torch.int32, device=DEV) if dev is not None else None
            lib.call("b200_rope_table", inv.data_ptr(), half, n_pos, pos0, lib.ptr(pd), c.data_ptr(), s.data_ptr(),
                     lib.stream())
            base = pos0 if dev is None else dev                          # *pos0_dev replaces pos0
            arg = (torch.arange(n_pos, device=DEV) + base).float()[:, None] * inv[None]   # the kernel's fp32 argument
            case = f"table D{D} pos0 {pos0} dev {dev}"
            W.add("table", case, P.exact_metrics(c[:n_pos], torch.cos(arg.double())))
            W.add("table", case, P.exact_metrics(s[:n_pos], torch.sin(arg.double())))
            W.add("", case, P.sentinel_report(c, (slice(0, n_pos),)))
            W.add("", case, P.sentinel_report(s, (slice(0, n_pos),)))
            n_cases += 1
        cos, sin = ops.rope_table(O.default_inv_freq(D).to(BF).to(DEV), RO_NPOS)
        S, ld = 37, 3 * H + 24
        rows = 3 * S

        def run(vals, pos, call):
            buf = P.poisoned(vals, vals.shape[0] + 2, ld)
            call(buf)
            R = vals.shape[0]
            qk = buf[:R, :2 * H].view(R, 2, nh, D)
            W.add("", case, {"v_changed": _ne(buf[:R, 2 * H:3 * H], vals[:, 2 * H:])})
            W.add("", case, P.sentinel_report(buf, (slice(0, R), slice(0, 3 * H))))
            return qk, vals[:, :2 * H].view(R, 2, nh, D), pos.view(R, 1, 1)

        for pos0, dev in ((0, None), (RO_NPOS - S, None), (17, RO_NPOS - S - 40)):
            pd = torch.tensor([dev], dtype=torch.int32, device=DEV) if dev is not None else None
            pos = pos0 + (dev or 0) + torch.arange(rows, device=DEV) % S
            case = f"qk D{D} pos0 {pos0} dev {dev}"
            for bwd in (0, 1):
                vals = randn(rows, 3 * H, seed=8100 + D + pos0 + bwd)
                qk, x, p = run(vals, pos, lambda b: lib.call(
                    "b200_rope_qk", b.data_ptr(), cos.data_ptr(), sin.data_ptr(), rows, S, H, D, ld, bwd, pos0,
                    lib.ptr(pd), lib.stream()))
                if bwd:
                    W.add("bwd", case, P.exact_metrics(qk, P.rope_bwd64(x, cos, sin, p)))
                else:
                    W.add("", case, {"fwd_mismatch": _ne(qk, _rope_chain64(x, cos, sin, p)[0].to(torch.float32).to(BF))})
                n_cases += 1
        # ragged: sequence b at pos0 + *pos0_dev + row_off[b]
        Sg, row_off = 5, torch.tensor([0, -3, -100, 0, -4000, -1, -4090], dtype=torch.int32, device=DEV)
        R = Sg * row_off.numel()
        pos0, dev = 4000, 90
        pd = torch.tensor([dev], dtype=torch.int32, device=DEV)
        pos = pos0 + dev + row_off.long().repeat_interleave(Sg) + torch.arange(R, device=DEV) % Sg
        case = f"ragged D{D}"
        vals = randn(R, 3 * H, seed=8200 + D)
        qk, x, p = run(vals, pos, lambda b: lib.call(
            "b200_rope_qk_ragged", b.data_ptr(), cos.data_ptr(), sin.data_ptr(), R, Sg, H, D, ld, pos0, pd.data_ptr(),
            row_off.data_ptr(), lib.stream()))
        W.add("", case, {"ragged_mismatch": _ne(qk, _rope_chain64(x, cos, sin, p)[0].to(torch.float32).to(BF))})
        n_cases += 1
    out = W.report()
    out["ro_cases"] = float(n_cases)
    return out


# forward: bf16(bf16(silu(g)) u) with the SFU sigmoid (relative error ~2^-22): two roundings; backward one.  scale_bf16
# is one fp32 product and one rounding, restated exactly.  H100 80GB HBM3 at 700 W: forward correctly rounded in every
# element of 9.1M (the bound leaves room for a flipped inner rounding: 1e-4, 2 ulp); backward 3.2e-5 not correctly
# rounded, 1 ulp (bound about 5x); err_over_tol <= 0.49
@bounded([
    ("sw_sentinels_changed", 0.0), ("sw_nan_in_range", 0.0), ("sw_scale_mismatch", 0.0),
    ("min:sw_grid_sweeps", 2.0), ("min:sw_scale_tails", 7.0),
    ("sw_fwd_frac", 1e-4), ("sw_fwd_maxulp", 2.0), ("sw_bwd_frac", 2e-4), ("sw_bwd_maxulp", 1.0),
    ("sw_fwd_err_over_tol", 1.0), ("sw_bwd_err_over_tol", 1.0),
])
def check_swiglu_conformance():
    """b200_swiglu_fwd / _bwd at I in {8, 1024, 4096}, row counts that are not a multiple of the grid (and exceed one
    grid-stride sweep), gates out to +-20 where the sigmoid saturates; b200_scale_bf16 with every n % 8 (the scalar
    tail) and n past one grid-stride sweep."""
    W = _Worst("sw_")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sweep = sms * 16 * 256                         # 16-byte vectors per grid-stride sweep (grid_for's cap)
    sweeps = 0
    for I, rows in ((8, sweep + 4099), (1024, 777), (4096, 1501)):
        g = randn(rows, I, scale=6.0, seed=8300 + I).float().clamp(-20, 20)
        g[0, :4] = torch.tensor([20.0, -20.0, 19.5, -19.5])
        g = g.to(BF)
        u = randn(rows, I, seed=8301 + I)
        gu = torch.cat([g, u], 1)
        GU = P.poisoned(gu, rows + 3, 2 * I)
        act = P.nan_buffer((rows + 2, I), device=DEV)
        lib.call("b200_swiglu_fwd", GU.data_ptr(), act.data_ptr(), rows, I, lib.stream())
        g64, u64 = g.double(), u.double()
        case = f"I{I} rows{rows}"
        W.add("fwd", case, P.exact_metrics(act[:rows], P.round_bf16(g64 * torch.sigmoid(g64)) * u64))
        W.add("", case, P.sentinel_report(act, (slice(0, rows),)))
        dact = randn(rows, I, seed=8302 + I)
        DA = P.poisoned(dact, rows + 3, I)
        dgu = P.nan_buffer((rows + 2, 2 * I), device=DEV)
        lib.call("b200_swiglu_bwd", GU.data_ptr(), DA.data_ptr(), dgu.data_ptr(), rows, I, lib.stream())
        W.add("bwd", case, P.exact_metrics(dgu[:rows], P.swiglu_bwd64(gu, dact)))
        W.add("", case, P.sentinel_report(dgu, (slice(0, rows),)))
        sweeps = max(sweeps, math.ceil(rows * I // 8 / sweep))
    tails = set()
    for n in (*range(1, 9), 8 * 1000 + 3, 8 * sweep + 8 * 1000 + 5):
        x = P.nan_buffer((n + 16,), device=DEV)
        x[:n] = randn(n, seed=8400 + n)
        y = P.nan_buffer((n + 16,), device=DEV)
        lib.call("b200_scale_bf16", x.data_ptr(), y.data_ptr(), n, 0.37, lib.stream())
        case = f"scale n{n}"
        W.add("", case, {"scale_mismatch": _ne(y[:n], (x[:n].float() * 0.37).to(BF))})
        W.add("", case, P.sentinel_report(y, (slice(0, n),)))
        tails.add(n % 8)
    out = W.report()
    out["sw_grid_sweeps"], out["sw_scale_tails"] = float(sweeps), float(len(tails - {0}))
    return out


# H100 80GB HBM3 at 700 W: worst row 4.1e-3 (o), 4.2e-3 / 4.4e-3 / 4.5e-3 (dq / dk / dv), 4.1e-3 / 4.3e-3 with the RoPE
# backward fused: the bf16 rounding of P dominates, as in attn_edges, whose row bound this shares.  The fused RoPE
# forward writes the rotated q / k exactly (the stand-alone chain)
AT_ROW = 1e-2


@bounded([
    ("at_sentinels_changed", 0.0), ("at_nan_in_range", 0.0), ("at_rope_qk_mismatch", 0.0), ("at_qkv_changed", 0.0),
    ("min:at_lengths", 8.0), ("min:at_cases", 48.0),
    *[(f"at_{n}_row", AT_ROW) for n in ("o", "dq", "dk", "dv", "rope_dq", "rope_dk")],
])
def check_attn_tiny_conformance():
    """b200_attn_tiny_fwd / _bwd at every L = 1..8 (a template instantiation each), n_heads 1 / 4 / 5 (partial CTAs of
    the warp grid), ld_qkv > 3H and ld_out > H with NaN padding, with and without the fused RoPE (forward rotates q and
    k in place: checked exactly; backward returns the gradient of the pre-RoPE projections), scored per (event, head,
    row) against fp64 attention with scale 1/16.  The backward recomputes P in fp32 and forms delta = sum_j P dP from
    it, i.e. from the exact o, so the reference's delta uses the exact o too."""
    W = _Worst("at_")
    D, scale = 256, 1.0 / 16
    cos, sin = ops.rope_table(O.default_inv_freq(D).to(BF).to(DEV), 8)
    lengths, n_cases = set(), 0
    for L in range(1, 9):
        for nh, N in ((1, 13), (4, 9), (5, 7)):
            for rope in (False, True):
                H = nh * D
                ldq, ldo = 3 * H + 40, H + 24
                R = N * L
                case = f"L{L} h{nh} N{N}" + (" rope" if rope else "")
                seed = 8500 + 10 * L + nh + 100 * rope
                vals = randn(R, 3 * H, seed=seed)
                QKV = P.poisoned(vals, R + 2, ldq)
                dov = randn(R, H, seed=seed + 1)
                DO = P.poisoned(dov, R + 2, ldo)
                ob = P.nan_buffer((R + 2, ldo), device=DEV)
                rc, rs = (cos.data_ptr(), sin.data_ptr()) if rope else (None, None)
                lib.call("b200_attn_tiny_fwd", QKV.data_ptr(), ob.data_ptr(), N, L, nh, D, ldq, ldo, scale, rc, rs,
                         lib.stream())
                post = QKV[:R, :3 * H]
                if rope:
                    x = vals[:, :2 * H].view(N, L, 2, nh, D)
                    chain = _rope_chain64(x, cos, sin, torch.arange(L, device=DEV).view(1, L, 1, 1))[0]
                    W.add("", case, {"rope_qk_mismatch": _ne(post[:, :2 * H].view(N, L, 2, nh, D),
                                                             chain.to(torch.float32).to(BF)),
                                     "qkv_changed": _ne(post[:, 2 * H:], vals[:, 2 * H:])})
                else:
                    W.add("", case, {"qkv_changed": _ne(post, vals)})
                W.add("", case, P.sentinel_report(QKV, (slice(0, R), slice(0, 3 * H))))
                q, k, v = post.reshape(N, L, 3, nh, D).permute(2, 0, 3, 1, 4)
                do = dov.view(N, L, nh, D).transpose(1, 2)
                o64, _, dq64, dk64, dv64 = P.attn_ref64(q, k, v, do, 0, scale)
                atol = 1e-3 * float(do.double().norm(dim=-1).median())
                o = ob[:R, :H].view(N, L, nh, D).transpose(1, 2)
                W.add("", case, {"o_row": P.row_worst(o, o64, atol=atol)})
                W.add("", case, P.sentinel_report(ob, (slice(0, R), slice(0, H))))
                dq = P.nan_buffer((R + 2, ldq), device=DEV)
                lib.call("b200_attn_tiny_bwd", QKV.data_ptr(), DO.data_ptr(), dq.data_ptr(), N, L, nh, D, ldq, ldo, scale,
                         rc, rs, lib.stream())
                g = dq[:R, :3 * H].reshape(N, L, 3, nh, D).permute(2, 0, 3, 1, 4)
                pos = torch.arange(L, device=DEV)
                if rope:
                    dq64, dk64 = P.rope_bwd64(dq64, cos, sin, pos), P.rope_bwd64(dk64, cos, sin, pos)
                pre = "rope_" if rope else ""
                W.add("", case, {f"{pre}dq_row": P.row_worst(g[0], dq64, atol=atol),
                                 f"{pre}dk_row": P.row_worst(g[1], dk64, atol=atol),
                                 "dv_row": P.row_worst(g[2], dv64, atol=atol)})
                W.add("", case, P.sentinel_report(dq, (slice(0, R), slice(0, 3 * H))))
                lengths.add(L)
                n_cases += 1
    out = W.report()
    out["at_lengths"], out["at_cases"] = float(len(lengths)), float(n_cases)
    return out


LO_VOCABS = (1001, 2041, 3406, 4090, 5003)    # ce_fwd: warp kernels of 4 / 8 / 14 / 16 vectors per lane, CTA kernel
LO_TV2O_MEDIUM_PARAMS = 233842688


# lse / row loss: fp32 with __expf; the mean an fp32 sum; the count exact.  dlogits: one rounding.  Clip: fp32 sums of
# squares.  AdamW: p one rounding of the fp32 update, m / v fp32.  H100 80GB HBM3 at 700 W: lse and row loss 4.0e-6
# absolute, mean 1.2e-7 relative; dlogits 6.6e-5 not correctly rounded, 1 ulp, err_over_tol 0.49; norm 5.9e-7 and
# coefficient 5.4e-7 relative (at 234M elements); p 1.6e-4, 1 ulp, 0.47; m / v 1.2e-7 / 1.9e-7 relative to the terms
# they add.  Bounds about 5x
@bounded([
    ("lo_sentinels_changed", 0.0), ("lo_nan_in_range", 0.0), ("lo_padcols_nonzero", 0.0), ("lo_ce_count_abs", 0.0),
    ("lo_ce_all_ignored_", 0.0), ("min:lo_ce_variants", 5.0), ("min:lo_adamw_steps", 4.0), ("min:lo_clip_cases", 12.0),
    ("lo_ce_lse_abs", 2e-5), ("lo_ce_rowloss_abs", 2e-5), ("lo_ce_mean_rel", 6e-7),
    ("lo_ce_bwd_frac", 3e-4), ("lo_ce_bwd_maxulp", 1.0), ("lo_ce_bwd_err_over_tol", 1.0),
    ("lo_clip_norm_rel", 3e-6), ("lo_clip_coef_rel", 3e-6),
    ("lo_adamw_p_frac", 8e-4), ("lo_adamw_p_maxulp", 1.0), ("lo_adamw_p_err_over_tol", 1.0),
    ("lo_adamw_m_rel", 1e-6), ("lo_adamw_v_rel", 1e-6),
])
def check_loss_optim_conformance():
    """b200_ce_fwd / _bwd at every row kernel (V in LO_VOCABS, none a multiple of 8) with NaN pad columns, targets that
    are ignore_index / -1 / V, an all-ignored batch, logits out to +-60 and grad_scale_dev in fp32 and bf16;
    b200_grad_clip_coef at n = 0, 5, 8k + 3 and the tv2o-medium parameter count, norm below and above max_norm and
    max_norm = 0; b200_adamw_step element by element at steps 1, 2, 3 and 1000, with and without an active clip, with
    lr wd large enough that decay moves p by several bf16 ulps and zero-gradient blocks on both sides of no-decay
    boundaries."""
    W = _Worst("lo_")
    variants = set()
    # ---- cross-entropy
    for vi, V in enumerate(LO_VOCABS):
        V8 = _rup8(V)
        ld, R = V8 + 16, 9001 if V == 2041 else 1000
        ign = 0 if vi % 2 else 17
        z = randn(R, V, scale=3.0, seed=8700 + V).float()
        z[1] = -60.0
        z[1, 7] = 60.0                               # saturated row
        z[2] = (z[2] * 20).clamp(-60, 60)
        z = z.to(BF)
        t = torch.randint(0, V, (R,), generator=_gen(8701 + V), device=DEV)
        t[1], t[4], t[R - 1] = 7, V - 1, V - 2       # targets in the masked last vector
        t[::7], t[3::11], t[5::13] = ign, -1, V
        buf = P.poisoned(z, R + 2, ld)
        lse = torch.full((R + 4,), float("nan"), device=DEV)
        rl = torch.full((R + 4,), float("nan"), device=DEV)
        lac = torch.full((4,), float("nan"), device=DEV)
        lib.call("b200_ce_fwd", buf.data_ptr(), t.data_ptr(), lse.data_ptr(), rl.data_ptr(), lac.data_ptr(), R, V, ld, ign,
                 lib.stream())
        lse64, rl64, mean64, cnt64, d64 = P.ce64(z, t, V, ign)
        case = f"V{V} R{R}"
        W.add("ce", case, {"lse_abs": float((lse[:R].double() - lse64).abs().max()),
                           "rowloss_abs": float((rl[:R].double() - rl64).abs().max()),
                           "mean_rel": abs(float(lac[0]) - mean64) / abs(mean64), "count_abs": abs(float(lac[1]) - cnt64)})
        for b_ in (lse, rl, lac):
            W.add("", case, P.sentinel_report(b_, (slice(0, b_.numel() - (2 if b_ is lac else 4)),)))
        vpl = (V8 // 8 + 31) // 32
        variants.add(next((b for b in (4, 8, 14, 16) if vpl <= b), "cta"))
        for gs, dev in ((1.0, None), (0.5, torch.tensor(3.0, device=DEV)), (2.0, torch.tensor(0.75, dtype=BF, device=DEV))):
            b = buf.clone()
            lib.call("b200_ce_bwd", b.data_ptr(), t.data_ptr(), lse.data_ptr(), lac.data_ptr(), R, V, ld, ign, gs,
                     lib.ptr(dev), int(dev is not None and dev.dtype == BF), lib.stream())
            scale = gs * (float(dev) if dev is not None else 1.0)
            c = case + f" gscale {gs} x {None if dev is None else dev.dtype}"
            W.add("ce_bwd", c, P.exact_metrics(b[:R, :V], d64 * scale))
            W.add("", c, P.sentinel_report(b, (slice(0, R), slice(0, V)), (slice(0, R), slice(V, V8))))
    # every target ignored: loss 0, count 0, zero gradient
    V, R = 3406, 64
    buf = P.poisoned(randn(R, V, scale=3.0, seed=8800), R, _rup8(V) + 16)
    t = torch.full((R,), 0, dtype=torch.long, device=DEV)
    t[::3] = -1
    lse = torch.empty(R, device=DEV)
    rl = torch.empty(R, device=DEV)
    lac = torch.full((2,), float("nan"), device=DEV)
    lib.call("b200_ce_fwd", buf.data_ptr(), t.data_ptr(), lse.data_ptr(), rl.data_ptr(), lac.data_ptr(), R, V,
             buf.stride(0), 0, lib.stream())
    lib.call("b200_ce_bwd", buf.data_ptr(), t.data_ptr(), lse.data_ptr(), lac.data_ptr(), R, V, buf.stride(0), 0, 1.0, None,
             0, lib.stream())
    W.add("", "all ignored", {"ce_all_ignored_loss": abs(float(lac[0])), "ce_all_ignored_count": abs(float(lac[1])),
                              "ce_all_ignored_grad_nonzero": float((buf[:, :_rup8(V)] != 0).sum())})
    # ---- grad-norm clip
    parts = int(lib.query("b200_gradnorm_parts"))
    ws = torch.full((parts + 8,), float("nan"), device=DEV)
    n_clip = 0
    for n in (0, 5, 8 * 1234 + 3, LO_TV2O_MEDIUM_PARAMS):
        g = P.nan_buffer((n + 16,), device=DEV)
        if n:
            g[:n] = randn(n, scale=1e-3, seed=8900 + n % 1000)
        norm64 = float(torch.linalg.vector_norm(g[:n], dtype=torch.float64)) if n else 0.0
        for max_norm in (0.0, norm64 / 3, norm64 * 3 + 1.0):
            nc = torch.full((4,), float("nan"), device=DEV)
            lib.call("b200_grad_clip_coef", g.data_ptr(), n, max_norm, nc.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                     lib.stream())
            coef64 = min(1.0, max_norm / (norm64 + 1e-6)) if max_norm > 0 else 1.0
            case = f"clip n{n} max_norm {max_norm:.3g}"
            W.add("clip", case, {"norm_rel": abs(float(nc[0]) - norm64) / max(norm64, 1e-30),
                                 "coef_rel": abs(float(nc[1]) - coef64) / coef64})
            W.add("", case, P.sentinel_report(nc, (slice(0, 2),)))
            n_clip += 1
        del g
    # ---- AdamW
    n = 256 * 9000                                 # past one grid-stride sweep of 8 x SMs CTAs x 256 threads x 8
    blocks = torch.arange(n // 256, device=DEV)
    nodecay = ((blocks // 3) % 2).to(torch.uint8)  # no-decay runs of 3 blocks
    gz = (blocks % 5 == 1).repeat_interleave(256)   # zero-gradient blocks on both sides of the boundaries
    g = torch.where(gz, 0.0, randn(n, scale=0.5, seed=9000).float()).to(BF)
    nc = torch.zeros(2, device=DEV)
    cws = torch.empty(parts, device=DEV)
    lib.call("b200_grad_clip_coef", g.data_ptr(), n, 1.0, nc.data_ptr(), cws.data_ptr(), cws.numel() * 4, lib.stream())
    steps_run = set()
    b1, b2, eps = 0.9, 0.99, 1e-8

    def f32(*a):                                   # the kernel's fp32 hyperparameters (1 - b2 is 1.2e-6 off 0.01)
        return [float(np.float32(x)) for x in a]
    for lr, wd, clip in ((1e-3, 0.01, False), (1e-2, 5.0, True)):
        p = P.nan_buffer((n + 8,), device=DEV)
        p[:n] = randn(n, scale=0.05, seed=9001)
        m = torch.zeros(n, device=DEV)
        v = torch.zeros(n, device=DEV)
        coef = float(nc[1]) if clip else 1.0
        for step in (1, 2, 3, 1000):
            if step == 1000:                       # a late step from a moment state of that age
                m = randn(n, scale=0.05, seed=9002).float()
                v = randn(n, scale=0.05, seed=9003).float().pow(2)
            p0, m0, v0 = p[:n].clone(), m.clone(), v.clone()
            lib.call("b200_adamw_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), nodecay.data_ptr(), n, lr,
                     b1, b2, eps, wd, step, nc.data_ptr() if clip else None, lib.stream())
            p64, m64, v64 = P.adamw64(p0, g, m0, v0, nodecay, *f32(lr, b1, b2, eps, wd), step, coef)
            case = f"adamw lr {lr} wd {wd} clip {coef:.3g} step {step}"
            W.add("adamw_p", case, P.exact_metrics(p[:n], p64))
            # relative to the terms the fp32 update adds (the moments cancel where the gradient turns)
            gc = g.double() * coef
            m_scale = b1 * m0.double().abs() + (1 - b1) * gc.abs() + 1e-30
            v_scale = b2 * v0.double() + (1 - b2) * gc * gc + 1e-30
            W.add("adamw", case, {"m_rel": float(((m.double() - m64).abs() / m_scale).max()),
                                  "v_rel": float(((v.double() - v64).abs() / v_scale).max())})
            W.add("", case, P.sentinel_report(p, (slice(0, n),)))
            steps_run.add(step)
    out = W.report()
    out["lo_ce_variants"], out["lo_adamw_steps"], out["lo_clip_cases"] = float(len(variants)), float(len(steps_run)), float(n_clip)
    return out


# in the order tests/test_gpu_parity.py runs them
GROUPS = {
    "gemm_fwd": check_gemm_fwd, "gemm_swiglu": check_gemm_swiglu, "gemm_dgrad": check_gemm_dgrad, "gemm_wgrad": check_gemm_wgrad,
    "elementwise": check_elementwise, "fused_rope": check_fused_rope, "attn_flash": check_attn_flash,
    "attn_wgmma": check_attn_wgmma, "attn_tiny": check_attn_tiny, "loss_optim": check_loss_optim, "decode": check_decode,
    "model_forward": check_model_forward, "model_layer_tf": check_model_layer_teacher_forced, "model_train": check_model_train,
    "model_generate": check_model_generate, "model_peaked_greedy": check_model_peaked_greedy, "model_large": check_model_large,
    "gemm_exact": check_gemm_exact, "decode_paged": check_decode_paged, "lora_train": check_lora_train,
    "model_vs_hf": check_model_vs_hf, "model_medium_long": check_model_medium_long,
    "gemm_matrix": check_gemm_matrix, "gemm_epilogues": check_gemm_epilogues, "attn_edges": check_attn_edges,
    "attn_long": check_attn_long, "gemv_matrix": check_gemv_conformance, "decode_attn_edges": check_decode_attn_conformance,
    "decode_attn_long": check_decode_attn_long,
    "sampler_exact": check_sampler_conformance, "persist_vs_phase": check_persist_vs_phase,
    "persist_token_exact": check_persist_token_exact, "persist_multi_event": check_persist_multi_event,
    "embed_exact": check_embed_conformance, "rmsnorm_exact": check_rmsnorm_conformance, "rope_exact": check_rope_conformance,
    "swiglu_exact": check_swiglu_conformance, "attn_tiny_exact": check_attn_tiny_conformance,
    "loss_optim_exact": check_loss_optim_conformance,
}
