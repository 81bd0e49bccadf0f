"""Fused-trainer step time with and without train.py --sample-seq at the benchmark shape (tv2o-medium, B = 8 x 2048
events x 8 tokens, bf16): one step = training_loss (+ sample_idx drawn by train.py's own expression, train.py:173) +
fused_optimizer_step.  The two arms alternate in one process, each timed with CUDA events after a warm-up; peak memory
is the allocator's peak over each arm's timed window.  The card name and power limit are read in the same run.
Writes $MIDI_TOOLS_OUT/sample_seq_step_time.json and prints a summary.

    python tools/sample_seq_step_time.py [steps per window] [rounds]
"""
import json
import os
import random
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
B, S = 8, 2048
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


def rand_idx():
    return [-1] + random.sample(list(range(S - 2)), min(127, (S - 2) // 2))          # train.py:173


out = {"workload": f"tv2o-medium fused train step (training_loss + fused_optimizer_step), B={B}, {S} events x 8 tokens, "
                   "bf16", "steps_per_window": K, "rounds": ROUNDS, "card": card()}
t0 = time.time()
torch.manual_seed(0)
random.seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).train()
batches = [synth_batch(model.tokenizer, B, S + 1, seed=1234 + i).to(dev) for i in range(2)]
out["setup_s"] = round(time.time() - t0, 1)
arms = {"full": lambda: None, "sample_seq": rand_idx}
state = {"step": 0}


def step(b, idx):
    state["step"] += 1
    loss = model.training_loss(b, sample_idx=idx)
    model.fused_optimizer_step(lr=1e-4, step=state["step"])
    return loss


for name, draw in arms.items():                 # warm-up: every shape of both arms
    for i in range(3):
        step(batches[i % 2], draw())
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
            loss = step(batches[i % 2], arms[name]())
        e1.record()
        torch.cuda.synchronize()
        res[name]["ms_per_step"].append(round(e0.elapsed_time(e1) / K, 2))
        res[name]["peak_mem_gb"].append(round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))
        res[name]["loss_last"] = round(float(loss), 4)
out["arms"] = res
out["card_after"] = card()
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "sample_seq_step_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
for name, r in res.items():
    ms = sorted(r["ms_per_step"])
    print(f"{name:>10}: {ms[len(ms) // 2]:.2f} ms per step (median of {len(ms)} windows of {K}; all {r['ms_per_step']}), "
          f"peak memory {max(r['peak_mem_gb']):.2f} GiB")
