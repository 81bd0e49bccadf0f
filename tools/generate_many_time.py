"""A request queue (`generate_many`, continuous batching) against lockstep ragged batches of the same requests, on the
persistent generate kernel: tv2o-medium with seeded random init, bf16, sampling at top_k 20.  N_REQ prompts of
100 ... 4000 events (seeded) each want their own number of new events, 64 ... 1024 (seeded):
  queue B   -- generate_many's scheduler with B slots: a finished request's slot takes the next request at once;
  lockstep B -- the requests in input order, B at a time, as ragged batches (generate_ragged's loop), each batch running
               until its largest budget, so a row whose budget ended early keeps computing until then.
EOS is denied in both arms (the loop's sampling mask), so a randomly initialised model cannot end a request early and
every request produces exactly its budget.  Useful events per second = the sum of the budgets over the wall time of the
whole queue, prefills included.  The arms alternate over the rounds, each timed with CUDA events after a warm-up; the
prefills (batch-1 per request for the queue, one ragged prefill per lockstep batch) are timed on their own as well.  The
card name and power limit are read in the same run.  Writes $MIDI_TOOLS_OUT/generate_many_time.json and prints a summary.

    python tools/generate_many_time.py [requests] [rounds]
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


out = {"workload": f"tv2o-medium generate, seeded init, bf16, top_k 20, EOS denied, {N_REQ} requests: prompts of "
                   f"{min(LENGTHS)} ... {max(LENGTHS)} events, budgets of {min(BUDGETS)} ... {max(BUDGETS)} new events "
                   f"(sum {sum(BUDGETS)}), persistent kernel", "rounds": ROUNDS, "card": card()}
t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
tok = model.tokenizer
songs = synth_batch(tok, N_REQ, max(LENGTHS), seed=77)
prompts = [songs[i, :L].to(dev) for i, L in enumerate(LENGTHS)]
out["setup_s"] = round(time.time() - t0, 1)
model._rt()
gens = {}
for B in SLOTS:
    q_len = max(L + n for L, n in zip(LENGTHS, BUDGETS))
    groups = [list(range(i, min(i + B, N_REQ))) for i in range(0, N_REQ, B)]
    l_len = max(max(LENGTHS[j] for j in g) + max(BUDGETS[j] for j in g) for g in groups)
    gens[B] = {"queue": model._checkout_generator(B, q_len, 1.0, 0.98, 20, torch.Generator().manual_seed(B)),
               "lockstep": model._checkout_generator(B, l_len, 1.0, 0.98, 20, torch.Generator().manual_seed(B + 1)),
               "groups": groups}
    for _, gg in (gens[B]["queue"], gens[B]["lockstep"]):
        assert gg.persistent_ok()
        gg.set_deny([tok.eos_id])


def queue(B, reqs=None):
    idx = range(N_REQ) if reqs is None else reqs
    res = gens[B]["queue"][1].run_queue([prompts[i] for i in idx], [BUDGETS[i] for i in idx], use_graph="persist")
    assert [r.shape[0] for r in res] == [LENGTHS[i] + BUDGETS[i] for i in idx]


def lockstep(B, groups=None):
    gg = gens[B]["lockstep"][1]
    for g in (gens[B]["groups"] if groups is None else groups):
        lens = [LENGTHS[j] for j in g]
        P = max(lens)
        batch = torch.full((B, P, songs.shape[2]), tok.pad_id, dtype=torch.long, device=dev)
        for r, j in enumerate(g):
            batch[r, :lens[r]] = prompts[j]
        lens += [1] * (B - len(g))                       # a short last batch: idle rows of one pad event
        gg.run(batch, use_graph="persist", stop_on_eos=False, max_new=max(BUDGETS[j] for j in g), lengths=lens)


def prefill_queue(B):
    gg = gens[B]["queue"][1]
    for p_ in prompts:
        gg._admit(0, p_)


def prefill_lockstep(B):
    gg = gens[B]["lockstep"][1]
    for g in gens[B]["groups"]:
        lens = [LENGTHS[j] for j in g] + [1] * (B - len(g))
        batch = torch.full((B, max(lens), songs.shape[2]), tok.pad_id, dtype=torch.long, device=dev)
        for r, j in enumerate(g):
            batch[r, :LENGTHS[j]] = prompts[j]
        gg._set_lengths(batch, lens)
        gg._set_state(batch)
        gg.lengths = None


with torch.inference_mode():
    arms = {}
    for B in SLOTS:
        queue(B, reqs=list(range(min(N_REQ, 2 * B))))                  # warm-up: every kernel shape of the arm
        lockstep(B, groups=gens[B]["groups"][:1])
        arms[f"queue_{B}"] = lambda B=B: queue(B)
        arms[f"lockstep_{B}"] = lambda B=B: lockstep(B)
    times = {name: [] for name in arms}
    for rnd in range(ROUNDS):
        for name in (list(arms) if rnd % 2 == 0 else list(arms)[::-1]):
            times[name].append(timed(arms[name]))
    pre = {}
    for B in SLOTS:
        pre[f"queue_{B}"] = min(timed(lambda: prefill_queue(B)) for _ in range(2))
        pre[f"lockstep_{B}"] = min(timed(lambda: prefill_lockstep(B)) for _ in range(2))
for B in SLOTS:
    for name in ("queue", "lockstep"):
        gens[B][name][1].set_deny(())
        model._return_generator(*gens[B][name])
useful = sum(BUDGETS)
out["arms"] = {name: {"s": [round(t, 3) for t in ts], "useful_events_per_s": round(useful / min(ts), 1),
                      "prefill_s": round(pre[name], 3)} for name, ts in times.items()}
for B in SLOTS:
    out[f"ratio_queue_over_lockstep_{B}"] = round(out["arms"][f"queue_{B}"]["useful_events_per_s"] /
                                                  out["arms"][f"lockstep_{B}"]["useful_events_per_s"], 3)
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "generate_many_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for name, r in out["arms"].items():
    print(f"{name:>11}: {r['useful_events_per_s']} useful events/s ({useful} events, windows {r['s']} s, best taken), "
          f"prefills {r['prefill_s']} s")
for B in SLOTS:
    print(f"queue / lockstep useful events per second at B = {B}: {out[f'ratio_queue_over_lockstep_{B}']}")
