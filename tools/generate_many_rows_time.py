"""The per-request queue (`generate_many_requests` with per-request settings and seeds) against the scalar queue, on the
persistent generate kernel: tv2o-medium with seeded random init, bf16, the 64-request workload of tools/generate_many_time.py
(prompts of 100 ... 4000 events, budgets of 64 ... 1024 new events, both seeded), at 8 and 16 slots:
  scalar B -- the scalar queue (b200_decode_events_queue): one set of settings, the slots' counter-based streams;
  same B   -- per-request mode (b200_decode_events_queue_rows) with every request at the scalar arm's settings;
  mixed B  -- per-request mode with mixed settings (temp 0.7 / 1.0 / 1.3, top_p 0.9 / 0.98 / 1.0, top_k 1 / 20 / 64).
Per-request mode cuts each row's event-level attention on the row's own length, as the batch-1 kernel does, so at B > 1
it runs more, shorter attention items than the scalar queue; this measures what that costs.  EOS is denied in every arm,
so every request produces exactly its budget.  Useful events per second = the sum of the budgets over the wall time of
the whole queue, prefills included.  The arms alternate over the rounds, each timed with CUDA events after a warm-up.
With B200_DECODE_PROFILE set, the per-phase cycle totals of CTA 0 (attention, combine) are reported for each arm from one
extra untimed run.  The card name and power limit are read in the same run.  Writes
$MIDI_TOOLS_OUT/generate_many_rows_time.json and prints a summary.

    python tools/generate_many_rows_time.py [requests] [rounds]
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
for p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import midi_model as mm  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

N_REQ = int(sys.argv[1]) if len(sys.argv) > 1 else 64
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 2
SLOTS = (8, 16)
rng = np.random.default_rng(2026)
LENGTHS = [int(v) for v in rng.integers(100, 4001, N_REQ)]
BUDGETS = [int(v) for v in rng.integers(64, 1025, N_REQ)]
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


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


PROFILE = bool(os.environ.get("B200_DECODE_PROFILE"))
MIXED = [(0.7, 0.9, 1), (1.0, 0.98, 20), (1.3, 1.0, 64)]
out = {"workload": f"tv2o-medium generate, seeded init, bf16, EOS denied, {N_REQ} requests: prompts of {min(LENGTHS)} ... "
                   f"{max(LENGTHS)} events, budgets of {min(BUDGETS)} ... {max(BUDGETS)} new events (sum {sum(BUDGETS)}), "
                   "persistent kernel; scalar and same arms at temp 1.0, top_p 0.98, top_k 20", "rounds": ROUNDS,
       "card": card()}
t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
tok = model.tokenizer
songs = synth_batch(tok, N_REQ, max(LENGTHS), seed=77)
prompts = [songs[i, :L].to(dev) for i, L in enumerate(LENGTHS)]
out["setup_s"] = round(time.time() - t0, 1)
model._rt()
q_len = max(L + n for L, n in zip(LENGTHS, BUDGETS))
seeds = [int(v) for v in np.random.default_rng(7).integers(0, 2 ** 62, N_REQ)]
settings = {"same": [(1.0, 0.98, 20, seeds[i], [tok.eos_id]) for i in range(N_REQ)],
            "mixed": [(*MIXED[i % 3], seeds[i], [tok.eos_id]) for i in range(N_REQ)]}
gens = {}
for B in SLOTS:
    gens[B] = {"scalar": model._checkout_generator(B, q_len, 1.0, 0.98, 20, torch.Generator().manual_seed(B)),
               "rows": model._checkout_generator(B, q_len, 1.0, 0.98, 20, None, per_row=True)}
    gens[B]["scalar"][1].set_deny([tok.eos_id])


def queue(B, arm, reqs=None):
    idx = list(range(N_REQ)) if reqs is None else reqs
    gg = gens[B]["scalar" if arm == "scalar" else "rows"][1]
    st = None if arm == "scalar" else [settings[arm][i] for i in idx]
    if st is not None:
        gg.rows, gg.req_top_k = True, [s[2] for s in st]
        assert gg.persistent_ok()
    res = gg.run_queue([prompts[i] for i in idx], [BUDGETS[i] for i in idx], use_graph="persist", settings=st)
    assert [r.shape[0] for r in res] == [LENGTHS[i] + BUDGETS[i] for i in idx]


PHASES = {"attention": 1, "combine": 2}


def phase_split(B, arm):
    """Cycles CTA 0 spent in the event-level attention and combine phases over one run of the arm (B200_DECODE_PROFILE)."""
    gg = gens[B]["scalar" if arm == "scalar" else "rows"][1]
    gg._persistent()
    gg.prof.zero_()
    queue(B, arm)
    torch.cuda.synchronize()
    prof = gg.prof.cpu().tolist()
    total = sum(prof[:14])
    return {name: {"cycles": prof[i], "share_of_all_phases": round(prof[i] / max(1, total), 4)} for name, i in PHASES.items()}


with torch.inference_mode():
    arms = {}
    for B in SLOTS:
        for arm in ("scalar", "same", "mixed"):
            queue(B, arm, reqs=list(range(min(N_REQ, 2 * B))))          # warm-up: every kernel shape of the arm
            arms[f"{arm}_{B}"] = lambda B=B, arm=arm: queue(B, arm)
    times = {name: [] for name in arms}
    for rnd in range(ROUNDS):
        for name in (list(arms) if rnd % 2 == 0 else list(arms)[::-1]):
            times[name].append(timed(arms[name]))
    split = {f"{arm}_{B}": phase_split(B, arm) for B in SLOTS for arm in ("scalar", "same", "mixed")} if PROFILE else None
for B in SLOTS:
    gens[B]["scalar"][1].set_deny(())
    for name in ("scalar", "rows"):
        model._return_generator(*gens[B][name])
useful = sum(BUDGETS)
out["arms"] = {name: {"s": [round(t, 3) for t in ts], "useful_events_per_s": round(useful / min(ts), 1)}
               for name, ts in times.items()}
for B in SLOTS:
    for arm in ("same", "mixed"):
        out[f"ratio_{arm}_over_scalar_{B}"] = round(out["arms"][f"{arm}_{B}"]["useful_events_per_s"] /
                                                    out["arms"][f"scalar_{B}"]["useful_events_per_s"], 3)
if split is not None:
    out["phase_split"] = split
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "generate_many_rows_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for name, r in out["arms"].items():
    print(f"{name:>9}: {r['useful_events_per_s']} useful events/s ({useful} events, windows {r['s']} s, best taken)")
for B in SLOTS:
    print(f"per-request / scalar useful events per second at B = {B}: same settings {out[f'ratio_same_over_scalar_{B}']}, "
          f"mixed {out[f'ratio_mixed_over_scalar_{B}']}")
