"""One launch of every HBM-bound kernel of the train step on bench-shape tensors (after one warm-up launch each), for
`ncu --set full -k regex:...` captures (kept out of the repository)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from midi_b200 import ops  # noqa: E402

dev, BF, H, V = "cuda", torch.bfloat16, 1024, 3406
g = torch.Generator(device=dev).manual_seed(0)
rnd = lambda *s: torch.randn(*s, generator=g, device=dev).to(BF)
w = (1 + 0.1 * rnd(H).float()).to(BF)
inv = (1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))).to(BF).to(dev)
cos, sin = ops.rope_table(inv, 2048)
for rep in range(2):
    for rows, I in ((16384, 4096), (131072, 1024)):
        x, r = rnd(rows, H), rnd(rows, H)
        h, y, rstd = ops.add_rmsnorm(x, r, w, 1e-6)
        dw = torch.empty(H, dtype=BF, device=dev)
        ops.rmsnorm_bwd(y, x, w, rstd, r, dw, False)
        gu = rnd(rows, 2 * I)
        act = ops.swiglu(gu)
        ops.swiglu_bwd(gu, act)
        del x, r, h, y, gu, act
    qkv = rnd(16384, 3 * H)
    ops.rope_qk_(qkv, cos, sin, 2048, H, 64)
    lg = torch.empty(131072, 3408, dtype=BF, device=dev).normal_(generator=g)
    tg = torch.randint(1, V, (131072,), device=dev, generator=g)
    lac, lse = ops.ce_fwd(lg, tg, V, 0)
    ops.ce_bwd_(lg, tg, lse, lac, V, 0, 1.0)
    qkv_t = rnd(131072, 3 * H)
    cos_t, sin_t = ops.rope_table((1.0 / (10000 ** (torch.arange(0, 256, 2).float() / 256))).to(BF).to(dev), 8)
    o = ops.attn_tiny_fwd(qkv_t, 16384, 8, 4, 256, rope=(cos_t, sin_t))
    ops.attn_tiny_bwd(qkv_t, o, 16384, 8, 4, 256, rope=(cos_t, sin_t))
    torch.cuda.synchronize()
print("done")
