"""Per-shape A/B of the wgmma GEMM against cuBLAS (torch.matmul, bf16) on the 24 GEMM shapes of one tv2o-medium
train step (the per-shape table of bench.py's roofline object), each timed alone: CUDA events, 3 warm-up + 20 launches,
operands rotated through enough copies to exceed the 50 MB L2.  Prints a table and writes
$MIDI_TOOLS_OUT/gemm_vs_cublas.json.  `ratio` > 1 means this repo's kernel is faster.

    python tools/gemm_vs_cublas.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from midi_b200 import ops  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
# (kind, rows M, out features N, in features K, launches per step): forward y = x W^T, dgrad dx = dy W, wgrad dW = dy^T x
SHAPES = [("fwd", 16384, 3072, 1024, 12), ("fwd", 16384, 1024, 1024, 12), ("fwd", 16384, 8192, 1024, 12), ("fwd", 16384, 1024, 4096, 12),
          ("fwd", 131072, 3072, 1024, 3), ("fwd", 131072, 1024, 1024, 6), ("fwd", 131072, 2048, 1024, 3), ("fwd", 131072, 3406, 1024, 1),
          ("dgrad", 16384, 3072, 1024, 12), ("dgrad", 16384, 1024, 1024, 12), ("dgrad", 16384, 8192, 1024, 12), ("dgrad", 16384, 1024, 4096, 12),
          ("dgrad", 131072, 3072, 1024, 3), ("dgrad", 131072, 1024, 1024, 6), ("dgrad", 131072, 2048, 1024, 3), ("dgrad", 131072, 3406, 1024, 1),
          ("wgrad", 16384, 3072, 1024, 12), ("wgrad", 16384, 1024, 1024, 12), ("wgrad", 16384, 8192, 1024, 12), ("wgrad", 16384, 1024, 4096, 12),
          ("wgrad", 131072, 3072, 1024, 3), ("wgrad", 131072, 1024, 1024, 6), ("wgrad", 131072, 2048, 1024, 3), ("wgrad", 131072, 3406, 1024, 1)]


def time_ms(fn, sets, iters=20):
    for i in range(3):
        fn(i % sets)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(iters):
        fn(i % sets)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    g = torch.Generator(device=DEV).manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, generator=g, device=DEV, dtype=torch.float32) * 0.05).to(BF)
    rows = []
    for kind, M, N, K, per_step in SHAPES:
        pitch = (N + 7) // 8 * 8
        nbytes = (M * K + N * K + M * pitch) * 2
        sets = max(2, int(300e6 // nbytes) + 1)
        xs = [rnd(M, K) for _ in range(sets)]
        w = rnd(N, K)
        dys = [torch.zeros(M, pitch, device=DEV, dtype=BF) for _ in range(sets)]
        for d in dys:
            d[:, :N] = rnd(M, N)
        dw = torch.empty(N, K, device=DEV, dtype=BF)
        if kind == "fwd":
            ours = lambda i: ops.linear(xs[i], w, pitch=pitch if pitch != N else None)
            ref = lambda i: torch.matmul(xs[i], w.t())
        elif kind == "dgrad":
            ours = lambda i: ops.linear_dgrad(dys[i], w)
            ref = lambda i: torch.matmul(dys[i][:, :N], w)
        else:
            ours = lambda i: ops.linear_wgrad(dys[i], xs[i], dw, False)
            ref = lambda i: torch.matmul(dys[i][:, :N].t(), xs[i])
        t_o, t_r = time_ms(ours, sets), time_ms(ref, sets)
        fl = 2.0 * M * N * K
        rows.append({"kind": kind, "M": M, "N": N, "K": K, "launches_per_step": per_step, "ours_ms": round(t_o, 4),
                     "cublas_ms": round(t_r, 4), "ours_tflops": round(fl / t_o / 1e9, 1), "cublas_tflops": round(fl / t_r / 1e9, 1),
                     "ratio": round(t_r / t_o, 3)})
        print(f"{kind:6s} rows={M:6d} out={N:5d} in={K:5d} x{per_step:2d}  ours {t_o:7.4f} ms {fl / t_o / 1e9:7.1f} TF/s | cuBLAS {t_r:7.4f} ms "
              f"{fl / t_r / 1e9:7.1f} TF/s | ratio {t_r / t_o:5.3f}", flush=True)
        del xs, dys, w, dw
    tot_o = sum(r["ours_ms"] * r["launches_per_step"] for r in rows)
    tot_r = sum(r["cublas_ms"] * r["launches_per_step"] for r in rows)
    print(f"per-step GEMM time (launch-weighted, isolated): ours {tot_o:.2f} ms, cuBLAS {tot_r:.2f} ms, ratio {tot_r / tot_o:.3f}")
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "gemm_vs_cublas.json"), "w") as f:
        json.dump({"rows": rows, "ours_ms_per_step": tot_o, "cublas_ms_per_step": tot_r}, f, indent=1)


if __name__ == "__main__":
    main()
