"""Bitwise A/B of the decode entry points and of MIDIModel.generate between two builds of the library.

Calls b200_gemv_bf16, b200_gemv_fused, b200_attn_decode and b200_attn_decode_fused through the C ABI on seeded inputs.
Every output buffer is NaN-prefilled and wider than the output where the call takes a pitch, so pad columns and bytes a
kernel must leave alone are hashed too (the KV pools and the split-T workspace included).  It also records the ids of
MIDIModel.generate on seeded-init tv2o-medium in every B200_GENERATE mode, with a multi-event prompt at batch 2 and 24
(the prefill then runs on the <= 16-row GEMV and on the tensor-core GEMM).  Each entry-point case is timed with CUDA
events over a replayed CUDA graph of 100 launches after a warm-up, so host launch overhead does not mask kernel time;
inputs are L2-resident after the warm-up.

    python tools/decode_ab.py run OUT.json          # on one build
    python tools/decode_ab.py compare A.json B.json  # exit 1 unless every output is bitwise equal; prints both timings
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_epilogue_ab import compare as compare_outputs, record  # noqa: E402


def run(out_path):
    sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
    import torch
    import midi_model as mm
    from midi_b200 import lib, ops
    from midi_b200.synth import synth_batch

    dev, bf = "cuda", torch.bfloat16
    outputs, timings = {}, {}
    seed = [0]

    def rnd(*s, scale=1.0):
        seed[0] += 1
        g = torch.Generator(device=dev).manual_seed(seed[0])
        return (torch.randn(*s, generator=g, device=dev, dtype=torch.float32) * scale).to(bf)

    def nan(*s, dtype=bf):
        return torch.full(s, float("nan"), device=dev, dtype=dtype)

    def case(name, entry, args, bufs):
        """Launch once and hash `bufs`, then time 100 launches replayed from a CUDA graph."""
        call = lambda: lib.call(entry, *args, lib.stream())  # noqa: E731
        call()
        torch.cuda.synchronize()
        for i, b in enumerate(bufs):
            outputs[f"{name}:{i}"] = record(b)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(100):
                call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g.replay()
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        timings[name] = e0.elapsed_time(e1) * 1000.0 / 100
        print(f"{name}: {timings[name]:.2f} us", flush=True)

    # b200_gemv_bf16: the <= 16-row nn.Linear, with and without the residual, and the pitched vocabulary
    for K, N in ((1024, 3072), (4096, 1024)):
        for B in (1, 3, 8, 16):
            for res in (False, True):
                x, w, r, y = rnd(B, K), rnd(N, K, scale=0.05), rnd(B, N) if res else None, nan(B, N)
                case(f"gemv_bf16_K{K}_B{B}{'_res' if res else ''}", "b200_gemv_bf16",
                     (x.data_ptr(), w.data_ptr(), lib.ptr(r), y.data_ptr(), B, N, K, K, K, N if res else 0, N), [y])
    x, w, y = rnd(2, 1024), rnd(3406, 1024, scale=0.05), nan(2, 3408)
    case("gemv_bf16_vocab_pitch3408", "b200_gemv_bf16",
         (x.data_ptr(), w.data_ptr(), None, y.data_ptr(), 2, 3406, 1024, 1024, 1024, 0, 3408), [y])

    # b200_gemv_fused: plain, RMSNorm, RMSNorm + SwiGLU, residual, ids/table input, pitched lm_head
    K, V = 1024, 3406
    norm_w, table = rnd(K, scale=0.5), rnd(V, K)
    ids = torch.randint(0, V, (16, 8), generator=torch.Generator(device=dev).manual_seed(99), device=dev)
    ids[3, 0], ids[5, 0] = -1, V                       # out of range: the kernel reads row 0
    for name, B, N_out, n_w, use_norm, use_res, swiglu, use_ids, ldy in (
            ("plain_B1", 1, 3072, 3072, False, False, 0, False, 3072),
            ("plain_B8", 8, 3072, 3072, False, False, 0, False, 3072),
            ("plain_B16", 16, 3072, 3072, False, False, 0, False, 3072),
            ("norm_B8", 8, 3072, 3072, True, False, 0, False, 3072),
            ("norm_swiglu_B8", 8, 4096, 8192, True, False, 1, False, 4096),
            ("residual_B8", 8, 1024, 1024, False, True, 0, False, 1024),
            ("ids_table_norm_B16", 16, 3072, 3072, True, False, 0, True, 3072),
            ("norm_vocab_pitch3408_B8", 8, V, V, True, False, 0, False, 3408)):
        x, w, y = rnd(B, K), rnd(n_w, K, scale=0.05), nan(B, ldy)
        r = rnd(B, N_out) if use_res else None
        case(f"gemv_fused_{name}", "b200_gemv_fused",
             (None if use_ids else x.data_ptr(), ids.data_ptr() if use_ids else None, 8, table.data_ptr(), V,
              norm_w.data_ptr() if use_norm else None, 1e-6, w.data_ptr(), lib.ptr(r), y.data_ptr(), B, N_out, K, K, K,
              N_out if use_res else 0, ldy, swiglu), [y])

    def paged(Bn, nh, D, page, cap):
        max_pages = cap // page
        pools = rnd(Bn * max_pages, nh, page, D), rnd(Bn * max_pages, nh, page, D)
        perm = torch.randperm(Bn * max_pages, generator=torch.Generator().manual_seed(cap + D)).to(torch.int32)
        return pools, perm.view(Bn, max_pages).to(dev).contiguous(), max_pages

    # b200_attn_decode: post-RoPE q, s_q rows per batch row, past by value or from the device, permuted block table
    Bn = 2
    for D, nh, page, cap, past, splits in ((64, 16, 64, 1024, 295, (1, 4)), (256, 4, 8, 8, 2, (1, 5))):  # 5: empty chunks
        H = nh * D
        (kp, vp), bt, max_pages = paged(Bn, nh, D, page, cap)
        for s_q in (1, 5):
            q = rnd(Bn * s_q, 3 * H)
            for n_split in splits:
                for on_dev in (False, True):
                    out, ws = nan(Bn * s_q, H + 16), nan(Bn * s_q * nh * n_split * (D + 2), dtype=torch.float32)
                    past_dev = torch.tensor([past], dtype=torch.int32, device=dev) if on_dev else None
                    case(f"attn_decode_D{D}_sq{s_q}_split{n_split}_{'devpast' if on_dev else 'past'}", "b200_attn_decode",
                         (q.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), max_pages, page, out.data_ptr(), Bn,
                          s_q, nh, D, 0 if on_dev else past, lib.ptr(past_dev), past + s_q, 3 * H, H + 16, D ** -0.5,
                          n_split, ws.data_ptr(), ws.numel() * 4), [out, ws])

    # b200_attn_decode_fused: RoPE + append + attention for one new token per row
    for D, nh, page, cap, max_T, pos_splits in (
            (64, 16, 64, 1024, 1024, [(63, 1), (64, 1), (64, 2), (200, 2), (200, 16), (700, 16)]),
            (256, 4, 8, 40, 40, [(7, 1), (8, 1), (20, 2)]),           # decode_attn_fused_kernel<256>
            (256, 4, 8, 8, 8, [(0, 1), (5, 1), (7, 1)])):             # max_T <= 32: the warp-per-head kernel
        H = nh * D
        inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=dev, dtype=torch.float32) / D))
        cos, sin = ops.rope_table(inv, cap)
        for pos, n_split in pos_splits:
            for on_dev in (False, True):
                (kp, vp), bt, max_pages = paged(Bn, nh, D, page, cap)
                qkv, out = rnd(Bn, 3 * H), nan(Bn, H + 16)
                ws = nan(Bn * nh * n_split * (D + 2), dtype=torch.float32)
                pos_dev = torch.tensor([pos], dtype=torch.int32, device=dev) if on_dev else None
                case(f"attn_decode_fused_D{D}_T{max_T}_pos{pos}_split{n_split}_{'devpos' if on_dev else 'pos'}",
                     "b200_attn_decode_fused",
                     (qkv.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt.data_ptr(), max_pages, page, cos.data_ptr(),
                      sin.data_ptr(), out.data_ptr(), Bn, nh, D, 0 if on_dev else pos, lib.ptr(pos_dev), max_T, 3 * H,
                      H + 16, D ** -0.5, n_split, ws.data_ptr(), ws.numel() * 4), [out, kp, vp, ws])

    # MIDIModel.generate: every loop, sampled with a fixed generator
    torch.manual_seed(0)
    model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=bf).eval()
    for B in (2, 24):
        prompt = synth_batch(model.tokenizer, B, 6, seed=B).numpy()
        for mode in ("eager", "nograph", "graph", "persist"):
            os.environ["B200_GENERATE"] = mode
            ids_out = model.generate(prompt=prompt, batch_size=B, max_len=40, generator=torch.Generator(dev).manual_seed(7))
            outputs[f"generate_B{B}_{mode}"] = record(torch.from_numpy(ids_out))
            print(f"generate_B{B}_{mode}: {ids_out.shape}", flush=True)
    os.environ.pop("B200_GENERATE")

    meta = {"device": torch.cuda.get_device_name(0)}
    with open(out_path, "w") as f:
        json.dump({"meta": meta, "outputs": outputs, "timings_us": timings}, f)
    print(f"{len(outputs)} outputs, {len(timings)} timed cases -> {out_path}")


def compare(a_path, b_path):
    rc = compare_outputs(a_path, b_path)
    ta, tb = (json.load(open(p)).get("timings_us", {}) for p in (a_path, b_path))
    print(f"{'case':64s} {'A us':>8s} {'B us':>8s} {'B/A':>6s}")
    for k in ta:
        if k in tb:
            print(f"{k:64s} {ta[k]:8.2f} {tb[k]:8.2f} {tb[k] / ta[k]:6.3f}")
    return rc


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "run":
        run(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
