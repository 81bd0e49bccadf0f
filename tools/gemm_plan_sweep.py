"""Sweep (block_n, splits) for the 24 GEMM shapes of one tv2o-medium train step and compare the fastest configuration with
the one the library's cost model (b200_gemm_plan) picks.  Same timing method as tools/gemm_vs_cublas.py.

    python tools/gemm_plan_sweep.py            # writes $MIDI_TOOLS_OUT/gemm_plan_sweep.json
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from gemm_vs_cublas import SHAPES, time_ms  # noqa: E402
from midi_b200 import ops  # noqa: E402

DEV, BF = "cuda", torch.bfloat16


def main():
    g = torch.Generator(device=DEV).manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, generator=g, device=DEV, dtype=torch.float32) * 0.05).to(BF)
    real_plan = ops._plan
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
            fn = lambda i: ops.linear(xs[i], w, pitch=pitch if pitch != N else None)
        elif kind == "dgrad":
            fn = lambda i: ops.linear_dgrad(dys[i], w)
        else:
            fn = lambda i: ops.linear_wgrad(dys[i], xs[i], dw, False)
        seen = {}

        def spy(m, n, k, allow):
            seen["key"] = (m, n, k, allow)
            return real_plan(m, n, k, allow)
        ops._plan = spy
        t_auto = time_ms(fn, sets)
        gm, gn, gk, allow = seen["key"]
        chosen = real_plan(gm, gn, gk, allow)
        num_kb = (gk + 63) // 64
        cands = []
        for bn in (128, 256):
            if bn == 256 and gn < 256:
                continue
            for s in ((1, 2, 3, 4, 5, 6, 8, 9, 12, 16) if allow else (1,)):
                if s > 1 and num_kb // s < 4:
                    continue
                cands.append((bn, s))
        res = {}
        for c in cands:
            ops._plan = lambda m, n, k, a, c=c: c
            try:
                res[c] = time_ms(fn, sets, iters=12)
            except Exception as e:  # a configuration the library refuses
                res[c] = float("inf")
                print("   ", c, "refused:", str(e)[:80])
        ops._plan = real_plan
        best = min(res, key=res.get)
        fl = 2.0 * M * N * K
        rows.append({"kind": kind, "M": M, "N": N, "K": K, "gemm": [gm, gn, gk], "launches_per_step": per_step,
                     "planner": list(chosen), "planner_ms": round(t_auto, 4), "best": list(best), "best_ms": round(res[best], 4),
                     "all": {f"{b}x{s}": round(t, 4) for (b, s), t in res.items()}})
        print(f"{kind:6s} rows={M:6d} out={N:5d} in={K:5d} x{per_step:2d} planner {chosen} {t_auto:7.4f} ms ({fl / t_auto / 1e9:6.0f} TF/s) | "
              f"best {best} {res[best]:7.4f} ms ({fl / res[best] / 1e9:6.0f} TF/s)  gain {100 * (t_auto / res[best] - 1):5.1f} %", flush=True)
        del xs, dys, w, dw
    tot_a = sum(r["planner_ms"] * r["launches_per_step"] for r in rows)
    tot_b = sum(min(r["best_ms"], r["planner_ms"]) * r["launches_per_step"] for r in rows)
    print(f"per-step GEMM time (isolated, launch-weighted): planner {tot_a:.2f} ms, best-of-sweep {tot_b:.2f} ms")
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "gemm_plan_sweep.json"), "w") as f:
        json.dump({"rows": rows, "planner_ms_per_step": tot_a, "best_ms_per_step": tot_b}, f, indent=1)


if __name__ == "__main__":
    main()
