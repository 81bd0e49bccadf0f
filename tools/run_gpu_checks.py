"""Run every GPU parity group of tests/gpu_checks.py in its own subprocess (a trapped kernel cannot
poison the other groups), print a table and write $MIDI_TOOLS_OUT/checks.json.

    python tools/run_gpu_checks.py [group ...]
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
OUT = OUT_DIR


def child(group):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import gpu_checks as G
    from parity_metrics import check_bounds
    g = G.GROUPS[group]
    t0 = time.time()
    m = g()
    torch.cuda.synchronize()
    res = check_bounds(m, g.bounds, g.info)
    print("##RESULT##" + json.dumps({"group": group, "seconds": time.time() - t0,
                                     "results": [[k, v, b, bool(ok)] for k, v, b, ok in res]}))


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        return child(sys.argv[2])
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.makedirs(OUT, exist_ok=True)
    groups = sys.argv[1:]
    if not groups:
        from gpu_checks import GROUPS
        groups = list(GROUPS)
    allres, failed = {}, 0
    for g in groups:
        env = dict(os.environ)
        try:
            r = subprocess.run([sys.executable, __file__, "--child", g], capture_output=True, text=True, timeout=900, env=env)
            out, err, rc = r.stdout, r.stderr, r.returncode
        except subprocess.TimeoutExpired as e:
            out, err, rc = (e.stdout or b"").decode(errors="replace") if isinstance(e.stdout, bytes) else (e.stdout or ""), "TIMEOUT", -9
        line = [l for l in out.splitlines() if l.startswith("##RESULT##")]
        if line:
            d = json.loads(line[0][len("##RESULT##"):])
            allres[g] = d
            bad = [r for r in d["results"] if not r[3]]
            failed += len(bad)
            print(f"[{g}] {len(d['results']) - len(bad)}/{len(d['results'])} ok in {d['seconds']:.1f}s")
            for k, v, b, ok in d["results"]:
                print(f"   {'ok  ' if ok else 'FAIL'} {k:44s} {v:.4g}" + (f"   (bound {b:.3g})" if b is not None else ""))
            extra = [l for l in out.splitlines() if not l.startswith("##RESULT##")]
            if extra:
                print("   | " + "\n   | ".join(extra[-6:]))
        else:
            failed += 1
            allres[g] = {"group": g, "error": (err or "")[-3000:], "stdout": out[-2000:], "rc": rc}
            print(f"[{g}] CRASHED rc={rc}\n{(err or '')[-2500:]}\n{out[-1500:]}")
        with open(os.path.join(OUT, "checks.json"), "w") as f:
            json.dump(allres, f, indent=1)
    print("TOTAL FAILED:", failed)
    return 0


if __name__ == "__main__":
    sys.exit(main())
