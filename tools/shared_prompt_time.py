"""Shared prompts in the request queue against the same queue with sharing turned off, on the persistent generate kernel:
tv2o-medium with seeded random init, bf16, 8 pieces of 1000 ... 4000 events (seeded) with 4 samples of each, in piece
order, budget 512 new events, per-request mode with one seed per request, at 8 and 16 slots:
  shared B -- `generate_many_requests`' queue as shipped: each piece prefilled once per stretch in which one of its samples
              is resident, its whole pages read from one copy in every layer;
  off B    -- decode._share_keys patched to share nothing: every sample prefilled into its slot's own pages.
The two arms run the same kernels on different block tables, and every request's events are checked equal across them.
EOS is denied, so every request produces exactly its budget.  Useful events per second = the sum of the budgets over the
wall time of the whole queue, prefills included.  The arms alternate over the rounds, each timed with CUDA events after
a warm-up.  Then, with B200_DECODE_PROFILE set for one extra untimed run of each arm, the per-phase cycle totals of CTA 0
(attention, combine) are reported.  The card name and power limit are read in the same run.  Writes
$MIDI_TOOLS_OUT/shared_prompt_time.json and prints a summary.

    python tools/shared_prompt_time.py [rounds]
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
from midi_b200 import decode  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
SLOTS = (8, 16)
N_PIECES, SAMPLES, BUDGET = 8, 4, 512
rng = np.random.default_rng(2027)
PIECE_LEN = [int(v) for v in rng.integers(1000, 4001, N_PIECES)]
N_REQ = N_PIECES * SAMPLES
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


out = {"workload": f"tv2o-medium generate, seeded init, bf16, EOS denied, {N_PIECES} pieces of {sorted(PIECE_LEN)} events x "
                   f"{SAMPLES} samples, budget {BUDGET} new events each (sum {N_REQ * BUDGET}), per-request seeds at temp 1.0, "
                   "top_p 0.98, top_k 20, persistent kernel", "rounds": ROUNDS, "card": card()}
t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
tok = model.tokenizer
songs = synth_batch(tok, N_PIECES, max(PIECE_LEN), seed=78)
pieces = [songs[i, :L].to(dev) for i, L in enumerate(PIECE_LEN)]
prompts = [pieces[i // SAMPLES] for i in range(N_REQ)]
out["setup_s"] = round(time.time() - t0, 1)
model._rt()
q_len = max(PIECE_LEN) + BUDGET
seeds = [int(v) for v in np.random.default_rng(8).integers(0, 2 ** 62, N_REQ)]
settings = [(1.0, 0.98, 20, seeds[i], [tok.eos_id]) for i in range(N_REQ)]
gens = {B: model._checkout_generator(B, q_len, 1.0, 0.98, 20, None, per_row=True) for B in SLOTS}
share_keys = decode._share_keys
results = {}


def queue(B, arm, reqs=None):
    idx = list(range(N_REQ)) if reqs is None else reqs
    gg = gens[B][1]
    gg.rows, gg.req_top_k = True, [settings[i][2] for i in idx]
    assert gg.persistent_ok()
    decode._share_keys = share_keys if arm == "shared" else (lambda ps, page: [None] * len(ps))
    try:
        res = gg.run_queue([prompts[i] for i in idx], [BUDGET] * len(idx), use_graph="persist",
                           settings=[settings[i] for i in idx])
    finally:
        decode._share_keys = share_keys
    assert [r.shape[0] for r in res] == [prompts[i].shape[0] + BUDGET for i in idx]
    if reqs is None:
        results[(B, arm)] = res


PHASES = {"attention": 1, "combine": 2}


def phase_split(B, arm):
    """Cycles CTA 0 spent in the event-level attention and combine phases over one run of the arm (B200_DECODE_PROFILE)."""
    gg = gens[B][1]
    gg._persist = None                                      # rebuilt with the profile buffer
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
        for arm in ("shared", "off"):
            queue(B, arm, reqs=list(range(min(N_REQ, 2 * B))))          # warm-up: every kernel shape of the arm
            arms[f"{arm}_{B}"] = lambda B=B, arm=arm: queue(B, arm)
    times = {name: [] for name in arms}
    for rnd in range(ROUNDS):
        for name in (list(arms) if rnd % 2 == 0 else list(arms)[::-1]):
            times[name].append(timed(arms[name]))
    mismatch = {B: sum(int((a != b).sum()) for a, b in zip(results[(B, "shared")], results[(B, "off")])) for B in SLOTS}
    os.environ["B200_DECODE_PROFILE"] = "1"
    split = {f"{arm}_{B}": phase_split(B, arm) for B in SLOTS for arm in ("shared", "off")}
    os.environ.pop("B200_DECODE_PROFILE")
for B in SLOTS:
    gens[B][1]._persist = None
    model._return_generator(*gens[B])
useful = N_REQ * BUDGET
out["arms"] = {name: {"s": [round(t, 3) for t in ts], "useful_events_per_s": round(useful / min(ts), 1)}
               for name, ts in times.items()}
for B in SLOTS:
    out[f"ratio_shared_over_off_{B}"] = round(out["arms"][f"shared_{B}"]["useful_events_per_s"] /
                                              out["arms"][f"off_{B}"]["useful_events_per_s"], 3)
    out[f"token_mismatch_shared_vs_off_{B}"] = mismatch[B]
out["phase_split"] = split
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "shared_prompt_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for name, r in out["arms"].items():
    print(f"{name:>9}: {r['useful_events_per_s']} useful events/s ({useful} events, windows {r['s']} s, best taken)")
for B in SLOTS:
    print(f"shared / off useful events per second at B = {B}: {out[f'ratio_shared_over_off_{B}']} "
          f"(token mismatches {mismatch[B]})")
