"""Bitwise A/B of every GEMM entry point between two builds of the library.

Runs ops.linear, linear_rope, linear_swiglu, linear_dgrad, linear_wgrad (with and without accumulate) and the residual
epilogue on a column view of a wider buffer, on seeded inputs at the 24 GEMM shapes of tools/gemm_vs_cublas.py plus
ragged M/N cases.  Outputs reach ~2 GB, so for each one it records the SHA-256 of the output buffer's bytes (padding
columns and the untouched columns around a view included) and a seeded sample of elements for diagnosing a mismatch.

    python tools/gemm_epilogue_ab.py run OUT.json          # on one build
    python tools/gemm_epilogue_ab.py compare A.json B.json  # exit 1 unless every output is bitwise equal
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def record(t):
    import torch
    flat = t.reshape(-1)
    idx = torch.randint(0, flat.numel(), (256,), generator=torch.Generator(device="cpu").manual_seed(1234))
    host = t.contiguous().view(-1).view(torch.int16).cpu().numpy()
    return {"sha256": hashlib.sha256(host.tobytes()).hexdigest(), "numel": flat.numel(),
            "sample_idx": idx.tolist(), "sample": flat[idx.to(t.device)].float().cpu().tolist()}


def run(out_path):
    sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import torch
    from gemm_vs_cublas import SHAPES
    from midi_b200 import ops

    dev, bf = "cuda", torch.bfloat16
    res = {}

    def rnd(g, *s):
        return (torch.randn(*s, generator=g, device=dev, dtype=torch.float32) * 0.05).to(bf)

    # ragged M / N / K next to the tv2o-medium shapes
    shapes = [(k, M, N, K) for k, M, N, K, _ in SHAPES] + [("fwd", 1000, 1001, 200), ("dgrad", 1000, 1001, 200),
                                                        ("wgrad", 1000, 1001, 200), ("fwd", 333, 1000, 136)]
    for i, (kind, M, N, K) in enumerate(shapes):
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        name = f"{kind}_{M}x{N}x{K}"
        pitch = (N + 7) // 8 * 8
        x, w = rnd(g, M, K), rnd(g, N, K)
        if kind == "fwd":
            res[name] = record(ops.linear(x, w, pitch=pitch if pitch != N else None))
            if N % 8 == 0:
                # residual, in place in a column view of a wider buffer
                buf = rnd(g, M, N + 64)
                yv = buf[:, 64:64 + N]
                ops.gemm(x, w, M, N, K, lda=x.stride(0), ldb=w.stride(0), out=yv, ldc=buf.stride(0), residual=yv)
                res[name + "_residual_inplace_view"] = record(buf)
            if N == 3072:
                D, S = (64, 2048) if M == 16384 else (256, 8)
                inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=dev, dtype=torch.float32) / D))
                cos, sin = ops.rope_table(inv, S)
                res[name + f"_rope_d{D}"] = record(ops.linear_rope(x, w, cos, sin, S, D))
            if N == 8192:
                gu, act = ops.linear_swiglu(x, w)
                res[name + "_swiglu_gu"] = record(gu)
                res[name + "_swiglu_act"] = record(act)
                del gu, act
        elif kind == "dgrad":
            dy = torch.zeros(M, pitch, device=dev, dtype=bf)
            dy[:, :N] = rnd(g, M, N)
            res[name] = record(ops.linear_dgrad(dy, w))
        else:
            dy = torch.zeros(M, pitch, device=dev, dtype=bf)
            dy[:, :N] = rnd(g, M, N)
            dw = torch.full((N, K), float("nan"), device=dev, dtype=bf)
            ops.linear_wgrad(dy, x, dw, False)
            res[name] = record(dw)
            dw = rnd(g, N, K)
            ops.linear_wgrad(dy, x, dw, True)
            res[name + "_accumulate"] = record(dw)
        torch.cuda.synchronize()
        print(name, "done", flush=True)
        torch.cuda.empty_cache()
    meta = {"device": torch.cuda.get_device_name(0)}
    with open(out_path, "w") as f:
        json.dump({"meta": meta, "outputs": res}, f)
    print(f"{len(res)} outputs -> {out_path}")


def compare(a_path, b_path):
    a, b = json.load(open(a_path))["outputs"], json.load(open(b_path))["outputs"]
    bad = 0
    for k in sorted(set(a) | set(b)):
        if k not in a or k not in b:
            print(f"MISSING {k}")
            bad += 1
            continue
        if a[k]["sha256"] != b[k]["sha256"]:
            diff = [(i, x, y) for i, x, y in zip(a[k]["sample_idx"], a[k]["sample"], b[k]["sample"]) if x != y and x == x]
            print(f"DIFF {k}: {len(diff)}/{len(a[k]['sample'])} sampled elements differ, first {diff[:4]}")
            bad += 1
    print(f"{len(a)} outputs compared, {bad} differ")
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "run":
        run(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
