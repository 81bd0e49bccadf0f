"""Fused-trainer step time of ragged batches (`training_loss(batch, lengths=...)`) against the padded step, at the
benchmark shape (tv2o-medium, B = 8, a 2049-event padded batch x 8 tokens, bf16): one step = training_loss +
fused_optimizer_step.  Two length sets:
  full   -- every sample 2049 events: the packed layout is the padded one (no-regression check);
  varied -- [2049, 2049, 1537, 1200, 900, 640, 400, 257].
For each, the padded and ragged arms alternate in one process, each timed with CUDA events after a warm-up; peak memory
is the allocator's peak over each arm's timed window.  Real tokens are the non-pad targets, the same in both arms.  The
card name and power limit are read in the same run.  Writes $MIDI_TOOLS_OUT/ragged_step_time.json and prints a summary.

    python tools/ragged_step_time.py [steps per window] [rounds]
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

K = int(sys.argv[1]) if len(sys.argv) > 1 else 10
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
B, S1 = 8, 2049
CASES = {"full": [S1] * B, "varied": [2049, 2049, 1537, 1200, 900, 640, 400, 257]}
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


out = {"workload": f"tv2o-medium fused train step (training_loss + fused_optimizer_step), B={B}, {S1}-event padded batch x "
                   "8 tokens, bf16", "steps_per_window": K, "rounds": ROUNDS, "card": card()}
t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).train()
pad = model.tokenizer.pad_id
out["setup_s"] = round(time.time() - t0, 1)
state = {"step": 0}


def step(b, lengths):
    state["step"] += 1
    loss = model.training_loss(b, lengths=lengths)
    model.fused_optimizer_step(lr=1e-4, step=state["step"])
    return loss


out["cases"] = {}
for case, lengths in CASES.items():
    batches = []
    for i in range(2):
        b = synth_batch(model.tokenizer, B, S1, seed=1234 + i)
        for j, L in enumerate(lengths):
            b[j, L:] = pad
        batches.append(b.to(dev))
    real_tokens = int((batches[0][:, 1:] != pad).sum())
    packed = sum((max(L - 1, 0) + 63) // 64 * 64 for L in lengths)
    arms = {"padded": None, "ragged": lengths}
    for name, ln in arms.items():            # warm-up: every shape of both arms
        for i in range(3):
            step(batches[i % 2], ln)
    torch.cuda.synchronize()
    res = {name: {"ms_per_step": [], "peak_mem_gb": [], "loss_last": None} for name in arms}
    for rnd in range(ROUNDS):
        order = list(arms) if rnd % 2 == 0 else list(arms)[::-1]
        for name in order:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(K):
                loss = step(batches[i % 2], arms[name])
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms_per_step"].append(round(e0.elapsed_time(e1) / K, 2))
            res[name]["peak_mem_gb"].append(round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))
            res[name]["loss_last"] = round(float(loss), 4)
    for name, r in res.items():
        ms = sorted(r["ms_per_step"])[len(r["ms_per_step"]) // 2]
        r["median_ms"] = ms
        r["real_tokens_per_s"] = round(real_tokens / (ms / 1e3))
    out["cases"][case] = {"lengths": lengths, "rows": {"padded": B * (S1 - 1), "packed": packed},
                          "real_tokens_per_step": real_tokens, "arms": res}
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "ragged_step_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for case, c in out["cases"].items():
    rows = c["rows"]
    print(f"{case}: packed/padded rows {rows['packed']}/{rows['padded']} = {rows['packed'] / rows['padded']:.3f}")
    for name, r in c["arms"].items():
        print(f"  {name:>7}: {r['median_ms']:.2f} ms per step (median of {len(r['ms_per_step'])} windows of {K}; all "
              f"{r['ms_per_step']}), peak memory {max(r['peak_mem_gb']):.2f} GiB, {r['real_tokens_per_s']} real tokens/s")
    pr, rg = c["arms"]["padded"]["median_ms"], c["arms"]["ragged"]["median_ms"]
    print(f"  ragged / padded step time: {rg / pr:.3f}")
