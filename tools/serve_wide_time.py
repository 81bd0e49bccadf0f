"""The serving queue (midi_b200/serve.py) at 32 slots on the persistent kernel, and a request with top_k > 64 on it:
tools/serve_time.py's workload (tv2o-medium with seeded random init, bf16, EOS denied, K users, 8 jobs in all, a job is
4 samples of one piece of 1024 ... 2897 events, 512 new events each, temp 1.0, top_p 0.98, top_k 20, seeded per job).

  (a) K = 4 and 8 users on three servers: 16 slots on the persistent kernel, 32 slots on the graph loop (the behaviour
      before the per-request kernels took 32 rows, restored here by giving those servers the old limits of
      GraphGenerator.persistent_ok: 16 slots, top_k <= 64), and 32 slots on the persistent kernel;
  (b) K = 4 on 8 slots with user 0's jobs at top_k = 100: before (old limits: every event with that request live runs as
      launches issued from the host) and after (the persistent kernel).
The arms of each K run one after the other in alternating order, in one process.  Reported per arm: useful events per
second, time to the first event of each job (p50, p95), the mean gap between two streamed events of a job.  Every request
of every arm is checked token by token against generate_stream of its piece at batch 1 seeded as the server seeded it
(the graph-loop arm makes no such guarantee; its mismatches are reported).  The card name and power limit are read in
the same run.  Writes $MIDI_TOOLS_OUT/serve_wide_time.json and prints a summary.

    python tools/serve_wide_time.py
"""
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
for p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import midi_model as mm  # noqa: E402
from midi_b200 import decode as dec  # noqa: E402
from midi_b200.serve import GenerateServer  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

SAMPLES, BUDGET, JOBS_TOTAL = 4, 512, 8
rng = np.random.default_rng(2027)
PIECE_LEN = [int(v) for v in rng.integers(1000, 4001, 8)]        # tools/serve_time.py's pieces
dev = torch.device("cuda", 0)

_new_rule = dec.GraphGenerator.persistent_ok
_old = type("Marking", (), {"on": False})()   # set while an old-limits server starts its worker


def _persistent_ok(self):
    """The new limits, or the previous release's (16 slots, top_k <= 64) for a loop marked old or built while marking."""
    if getattr(self, "_old_rule", False) or _old.on:
        self._old_rule = True
        ks = self.req_top_k if self.rows else [self.top_k]
        return self.B <= 16 and all(1 <= k <= 64 for k in ks) and _new_rule(self)
    return _new_rule(self)


dec.GraphGenerator.persistent_ok = _persistent_ok


def card():
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip() or q.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"not read: {e}"
    return info


def schedule(K):
    """Per user: (start offset, [(pause, piece index, job seed)]) -- tools/serve_time.py's plan."""
    r = np.random.default_rng(100 + K)
    jobs = JOBS_TOTAL // K
    return [(float(r.uniform(0, 0.5)), [(float(r.uniform(0, 0.2)), int(r.integers(0, 8)), int(r.integers(0, 2 ** 31)))
                                         for _ in range(jobs)]) for _ in range(K)]


def run_users(K, server, top_k_of_user, kept):
    plan = schedule(K)
    t_first, t_last, ttfe, gaps, errors = [], [], [], [], []
    lock = threading.Lock()

    def user(u):
        try:
            start, jobs = plan[u]
            time.sleep(start)
            for pause, piece, seed in jobs:
                time.sleep(pause)
                ts = time.perf_counter()
                stamps, rows = [], []
                for ev in server.generate_stream(pieces[piece], batch_size=SAMPLES, max_len=pieces[piece].shape[0] + BUDGET,
                                                 top_k=top_k_of_user(u), generator=torch.Generator().manual_seed(seed)):
                    stamps.append(time.perf_counter())
                    rows.append(ev)
                assert len(stamps) == BUDGET, len(stamps)
                with lock:
                    t_first.append(ts)
                    t_last.append(stamps[-1])
                    ttfe.append(stamps[0] - ts)
                    gaps.append((stamps[-1] - stamps[0]) / (len(stamps) - 1))
                    kept.append((piece, seed, top_k_of_user(u), np.stack(rows)))
        except Exception as e:                                  # noqa: BLE001  reported below
            errors.append(repr(e))

    threads = [threading.Thread(target=user, args=(u,)) for u in range(K)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    if errors:
        raise RuntimeError(errors)
    wall = max(t_last) - min(t_first)
    return {"jobs": len(ttfe), "wall_s": round(wall, 3), "useful_events_per_s": round(len(ttfe) * SAMPLES * BUDGET / wall, 1),
            "ttfe_p50_s": round(float(np.percentile(ttfe, 50)), 4), "ttfe_p95_s": round(float(np.percentile(ttfe, 95)), 4),
            "mean_gap_ms": round(1e3 * float(np.mean(gaps)), 3)}


class First(torch.Generator):
    """A CPU generator whose first torch.randint(0, 2**62, (1,)) draw is `seed` (the seed a server row was given)."""

    def __init__(self, seed):
        super().__init__()
        self.first = seed


_randint = torch.randint


def _randint_first(lo, hi, size, generator=None, device=None, **k):
    if isinstance(generator, First) and generator.first is not None:
        s, generator.first = generator.first, None
        return torch.tensor([s])
    return _randint(lo, hi, size, generator=generator, device=device, **k)


out = {"workload": f"tv2o-medium generate, seeded init, bf16, EOS denied, K users x {JOBS_TOTAL} // K jobs of {SAMPLES} samples "
                   f"of one piece of {sorted(PIECE_LEN)} events, {BUDGET} new events each, temp 1.0, top_p 0.98, top_k 20 "
                   "(user 0: 100 in the top_k arms)", "card": card()}
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
tok = model.tokenizer
songs = synth_batch(tok, 8, max(PIECE_LEN), seed=78).numpy()
pieces = [songs[i, :L] for i, L in enumerate(PIECE_LEN)]
deny = model._deny_ids
model._deny_ids = lambda *a: deny(*a) + [tok.eos_id]          # EOS denied (the grammar mask)
max_len = max(PIECE_LEN) + BUDGET


def server(B, old):
    _old.on = old
    try:
        s = GenerateServer(model, batch_size=B, max_len=max_len)
    finally:
        _old.on = False
    return s


os.environ["B200_GENERATE"] = "persist"
servers = {"persist_16": server(16, False), "graph_32": server(32, True), "persist_32": server(32, False),
           "old_8": server(8, True), "persist_8": server(8, False)}
out["on_persistent_kernel_at_start"] = {k: bool(s._persist) for k, s in servers.items()}
kept = {}
try:
    for p in pieces[:2]:                                        # warm-up: every server once at a small size
        for s in servers.values():
            list(s.generate_stream(p, batch_size=SAMPLES, max_len=p.shape[0] + 8, top_k=100))
    out["arms"] = {}
    plans = [(4, ("persist_16", "graph_32", "persist_32"), False), (8, ("persist_16", "graph_32", "persist_32"), False),
             (4, ("old_8", "persist_8"), True)]
    for i, (K, names, wide) in enumerate(plans):
        for name in (names if i % 2 == 0 else names[::-1]):
            arm = f"K{K}_{name}" + ("_user0_top_k100" if wide else "")
            kept[arm] = []
            out["arms"][arm] = run_users(K, servers[name], (lambda u: 100 if u == 0 else 20) if wide else (lambda u: 20),
                                         kept[arm])
            print(f"{arm}: {out['arms'][arm]}", flush=True)
finally:
    for s in servers.values():
        s.close()
# tokens: every request of every arm against generate_stream of its piece alone, seeded as the server seeded it
torch.randint = _randint_first
solo = {}
try:
    for arm, jobs in kept.items():
        bad = checked = 0
        for piece, seed, top_k, rows in jobs:
            g = torch.Generator().manual_seed(seed)
            for b in range(SAMPLES):
                s = int(_randint(0, 2 ** 62, (1,), generator=g).item())
                if (piece, s, top_k) not in solo:
                    p = pieces[piece]
                    solo[(piece, s, top_k)] = np.stack([e[0] for e in model.generate_stream(
                        p, batch_size=1, max_len=p.shape[0] + BUDGET, top_k=top_k, generator=First(s))])
                ref = solo[(piece, s, top_k)]
                bad += int((ref != rows[:, b]).sum()) if ref.shape == rows[:, b].shape else 10 ** 9
                checked += 1
        out["arms"][arm]["requests_checked_vs_solo_stream"] = checked
        out["arms"][arm]["token_mismatch_vs_solo_stream"] = bad
finally:
    torch.randint = _randint
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "serve_wide_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for arm, r in out["arms"].items():
    print(f"{arm}: {r['useful_events_per_s']} ev/s, ttfe p50/p95 {r['ttfe_p50_s']}/{r['ttfe_p95_s']} s, gap {r['mean_gap_ms']} ms, "
          f"tokens vs solo: {r['requests_checked_vs_solo_stream']} requests, {r['token_mismatch_vs_solo_stream']} mismatches")
