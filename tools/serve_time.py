"""Concurrent app users on today's per-user generate loops against one serving queue (midi_b200/serve.py), on the persistent
generate kernel: tv2o-medium with seeded random init, bf16, EOS denied (so every request produces its budget).

K = 2, 4 and 8 simulated users, one thread each.  A user starts at a seeded offset in [0, 0.5) s and runs 8 / K jobs one
after another, with a seeded pause in [0, 0.2) s before each; a job is 4 samples of one piece (the 8 pieces of
tools/shared_prompt_time.py, 1024 ... 2897 events), 512 new events each, seeded per job.
  (a) today's app: every user calls model.generate_stream(piece, batch_size=4) on their own thread;
  (b) every user calls server.generate_stream(piece, batch_size=4) on one GenerateServer of 8 or 16 slots.
For each K the arms run one after the other in alternating order.  Reported per arm: useful events per second (4 x 512
events per job over the wall time from the first job's start to the last job's last event), time to the first event of
each job (p50, p95) and the mean gap between two streamed events of a job.  Then every request of arm (b) at K = 8 with 8
slots is checked against generate_stream of its piece at batch 1 seeded as the server seeded it.  The card name and power
limit are read in the same run.  Writes $MIDI_TOOLS_OUT/serve_time.json and prints a summary.

    python tools/serve_time.py
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
from midi_b200.serve import GenerateServer  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

USERS, SLOTS, SAMPLES, BUDGET, JOBS_TOTAL = (2, 4, 8), (8, 16), 4, 512, 8
rng = np.random.default_rng(2027)
PIECE_LEN = [int(v) for v in rng.integers(1000, 4001, 8)]
dev = torch.device("cuda", 0)


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
    """Per user: (start offset, [(pause, piece index, job seed)]) -- seeded, the same for both arms."""
    r = np.random.default_rng(100 + K)
    jobs = JOBS_TOTAL // K
    return [(float(r.uniform(0, 0.5)), [(float(r.uniform(0, 0.2)), int(r.integers(0, 8)), int(r.integers(0, 2 ** 31)))
                                         for _ in range(jobs)]) for _ in range(K)]


def run_users(K, stream_fn, keep=None):
    """Every user's jobs on its own thread; stream_fn(piece, generator) yields [4, 8] arrays.  Returns the metrics."""
    plan = schedule(K)
    t_first, t_last, ttfe, gaps, errors = [], [], [], [], []
    lock = threading.Lock()
    t0 = time.perf_counter()

    def user(u):
        try:
            start, jobs = plan[u]
            time.sleep(start)
            for pause, piece, seed in jobs:
                time.sleep(pause)
                ts = time.perf_counter()
                stamps, rows = [], []
                for ev in stream_fn(pieces[piece], torch.Generator().manual_seed(seed)):
                    stamps.append(time.perf_counter())
                    if keep is not None:
                        rows.append(ev)
                assert len(stamps) == BUDGET, len(stamps)
                with lock:
                    t_first.append(ts)
                    t_last.append(stamps[-1])
                    ttfe.append(stamps[0] - ts)
                    gaps.append((stamps[-1] - stamps[0]) / (len(stamps) - 1))
                    if keep is not None:
                        keep.append((piece, seed, np.stack(rows)))
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
    n_jobs = len(ttfe)
    return {"jobs": n_jobs, "wall_s": round(wall, 3), "useful_events_per_s": round(n_jobs * SAMPLES * BUDGET / wall, 1),
            "ttfe_p50_s": round(float(np.percentile(ttfe, 50)), 4), "ttfe_p95_s": round(float(np.percentile(ttfe, 95)), 4),
            "mean_gap_ms": round(1e3 * float(np.mean(gaps)), 3), "since_start_s": round(max(t_last) - t0, 3)}


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
                   f"of one piece of {sorted(PIECE_LEN)} events, {BUDGET} new events each, temp 1.0, top_p 0.98, top_k 20, "
                   "persistent kernel", "card": card()}
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
tok = model.tokenizer
songs = synth_batch(tok, 8, max(PIECE_LEN), seed=78).numpy()
pieces = [songs[i, :L] for i, L in enumerate(PIECE_LEN)]
deny = model._deny_ids
model._deny_ids = lambda *a: deny(*a) + [tok.eos_id]          # EOS denied in both arms (the grammar mask)
max_len = max(PIECE_LEN) + BUDGET


def app_stream(piece, g):
    return model.generate_stream(piece, batch_size=SAMPLES, max_len=piece.shape[0] + BUDGET, generator=g)


servers = {B: GenerateServer(model, batch_size=B, max_len=max_len) for B in SLOTS}
try:
    # warm-up: every arm once at a small size (kernel modules, allocator, the generators of the app arm)
    for p in pieces[:2]:
        list(model.generate_stream(p, batch_size=SAMPLES, max_len=p.shape[0] + 8))
        for B in SLOTS:
            list(servers[B].generate_stream(p, batch_size=SAMPLES, max_len=p.shape[0] + 8))
    out["arms"] = {}
    kept = []
    for i, K in enumerate(USERS):
        arms = [("app", app_stream)] + [(f"server_{B}", lambda piece, g, B=B: servers[B].generate_stream(
            piece, batch_size=SAMPLES, max_len=piece.shape[0] + BUDGET, generator=g)) for B in SLOTS]
        if i % 2:
            arms = arms[::-1]
        for name, fn in arms:
            keep = kept if (K == 8 and name == "server_8") else None
            out["arms"][f"K{K}_{name}"] = run_users(K, fn, keep)
            print(f"K={K} {name}: {out['arms'][f'K{K}_{name}']}", flush=True)
finally:
    for s in servers.values():
        s.close()
# tokens of arm (b): every request of K = 8, 8 slots against generate_stream of its piece alone
torch.randint = _randint_first
bad = checked = 0
try:
    for piece, seed, rows in kept:
        g = torch.Generator().manual_seed(seed)
        for b in range(SAMPLES):
            s = int(_randint(0, 2 ** 62, (1,), generator=g).item())
            p = pieces[piece]
            solo = np.stack([e[0] for e in model.generate_stream(p, batch_size=1, max_len=p.shape[0] + BUDGET,
                                                                  generator=First(s))])
            bad += int((solo != rows[:, b]).sum()) if solo.shape == rows[:, b].shape else 10 ** 9
            checked += 1
finally:
    torch.randint = _randint
out["server_8_K8_requests_checked_vs_solo_stream"] = checked
out["server_8_K8_token_mismatch_vs_solo_stream"] = bad
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "serve_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for K in USERS:
    row = [f"{name}: {out['arms'][f'K{K}_{name}']['useful_events_per_s']} ev/s, ttfe p50/p95 "
           f"{out['arms'][f'K{K}_{name}']['ttfe_p50_s']}/{out['arms'][f'K{K}_{name}']['ttfe_p95_s']} s, gap "
           f"{out['arms'][f'K{K}_{name}']['mean_gap_ms']} ms" for name in ["app"] + [f"server_{B}" for B in SLOTS]]
    print(f"K={K}: " + " | ".join(row))
print(f"arm (b) tokens vs solo streams: {checked} requests, {bad} mismatches")
