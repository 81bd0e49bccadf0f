"""Ragged generation (`generate_ragged(prompt, lengths)`) against continuing the same prompts one call at a time, on the
persistent generate kernel: tv2o-medium with seeded random init, bf16, sampling at top_k 20.  Eight prompts of
4000 ... 100 events each get N_NEW new events:
  ragged -- one batch of 8 (lengths = the prompt lengths, right-padded to 4000 events);
  solo   -- each prompt alone at batch 1, one after the other.
Both arms run exactly N_NEW events per prompt (the stop rule is off) on loops sized for 4000 + N_NEW positions, and
alternate in one process, each timed with CUDA events after a warm-up.  The prefill (loading the prompt into the KV
cache) is timed on its own as well.  The card name and power limit are read in the same run.  Writes
$MIDI_TOOLS_OUT/ragged_generate_time.json and prints a summary.

    python tools/ragged_generate_time.py [new events] [rounds]
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
import torch  # noqa: E402

import midi_model as mm  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

N_NEW = int(sys.argv[1]) if len(sys.argv) > 1 else 512
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 2
LENGTHS = [4000, 3500, 3000, 2000, 1500, 1000, 500, 100]
B, P = len(LENGTHS), max(LENGTHS)
MAX_LEN = P + N_NEW
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


out = {"workload": f"tv2o-medium generate, seeded init, bf16, top_k 20, {B} prompts of {LENGTHS} events, {N_NEW} new events "
                   "each, persistent kernel", "rounds": ROUNDS, "card": card()}
t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).eval()
pad = model.tokenizer.pad_id
prompt = synth_batch(model.tokenizer, B, P, seed=77).to(dev)
for b, L in enumerate(LENGTHS):
    prompt[b, L:] = pad
out["setup_s"] = round(time.time() - t0, 1)
model._rt()
key8, gg8 = model._checkout_generator(B, MAX_LEN, 1.0, 0.98, 20, torch.Generator().manual_seed(1))
key1, gg1 = model._checkout_generator(1, MAX_LEN, 1.0, 0.98, 20, torch.Generator().manual_seed(2))
assert gg8.persistent_ok() and gg1.persistent_ok()


def ragged():
    return gg8.run(prompt, use_graph="persist", stop_on_eos=False, max_new=N_NEW, lengths=LENGTHS)


def solo():
    for b, L in enumerate(LENGTHS):
        gg1.run(prompt[b:b + 1, :L], use_graph="persist", stop_on_eos=False, max_new=N_NEW)


def prefill_ragged():
    gg8._set_lengths(prompt, LENGTHS)
    gg8._set_state(prompt)
    gg8.lengths = None


def prefill_solo():
    for b, L in enumerate(LENGTHS):
        gg1._set_state(prompt[b:b + 1, :L])


with torch.inference_mode():
    res = ragged()
    assert res.shape == (B, P + N_NEW, 8)
    solo()
    arms = {"ragged": ragged, "solo": solo}
    times = {name: [] for name in arms}
    for rnd in range(ROUNDS):
        for name in (list(arms) if rnd % 2 == 0 else list(arms)[::-1]):
            times[name].append(timed(arms[name]))
    pre = {"ragged": [timed(prefill_ragged) for _ in range(2)], "solo": [timed(prefill_solo) for _ in range(2)]}
model._return_generator(key8, gg8)
model._return_generator(key1, gg1)
events = B * N_NEW
out["arms"] = {name: {"s": [round(t, 3) for t in ts], "events_per_s": round(events / min(ts), 1),
                      "prefill_s": round(min(pre[name]), 3)} for name, ts in times.items()}
out["ratio_ragged_over_solo_events_per_s"] = round(out["arms"]["ragged"]["events_per_s"] /
                                                   out["arms"]["solo"]["events_per_s"], 3)
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "ragged_generate_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for name, r in out["arms"].items():
    print(f"{name:>6}: {r['events_per_s']} events/s ({events} events, windows {r['s']} s, best taken), "
          f"prefill {r['prefill_s']} s")
print(f"ragged / solo events per second: {out['ratio_ragged_over_solo_events_per_s']}")
