"""Fused-trainer step time and peak memory with and without activation checkpointing
(`model.gradient_checkpointing_enable()`).  One step = training_loss + fused_optimizer_step, bf16.

  * tv2o-medium, B = 8 x 2048 events x 8 tokens (the benchmark shape): both arms, alternating in one process, each timed
    with CUDA events after a warm-up; peak memory is the allocator's peak over each arm's timed window.
  * tv2o-large, B = 8 x 4096 (BASELINE.json config 5): checkpointed.  The default arm runs only when its estimated peak
    fits the free device memory: the checkpointed arm's measured peak plus the activations checkpointing does not keep,
    counted from the shapes.  Otherwise it is recorded as not run -- the card is shared, and running out of memory on
    purpose is not a measurement.

The card name and power limit are read in the same run.  Writes $MIDI_TOOLS_OUT/recompute_step_time.json and
recompute_step_time.txt (the summary) and prints them.

    python tools/recompute_step_time.py [steps per window] [rounds]
"""
import gc
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
GiB = 2 ** 30
MARGIN = 4 * GiB              # kept free beyond the estimate (backward transients, fragmentation)
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


def saved_bytes(cfg, B, S, checkpoint):
    """Activations a training forward keeps for backward (engine.StackEngine.forward), from the shapes: per event-level
    row and layer x, n1, h, n2, attn (H each), qkv (3H), gu (2I), act (I) in bf16, two fp32 rstd and the fp32 lse per
    head; with checkpointing x, attn and lse.  The token-level stack has 8 rows per event and no lse."""
    total = 0
    for c, rows, lse in ((cfg.net_config, B * S, True), (cfg.net_token_config, B * S * 8, False)):
        H, I, nh = c.hidden_size, c.intermediate_size, c.num_attention_heads
        per_row = 2 * 2 * H if checkpoint else 2 * (8 * H + 3 * I) + 2 * 4
        per_row += 4 * nh if lse else 0
        total += c.num_hidden_layers * rows * per_row
    return total


def build(name, B, S):
    torch.manual_seed(0)
    cfg = mm.MIDIModelConfig.from_name(name)
    model = mm.MIDIModel(cfg).to(dev, dtype=torch.bfloat16).train()
    batches = [synth_batch(model.tokenizer, B, S + 1, seed=1234 + i).to(dev) for i in range(2)]
    return cfg, model, batches


def run_arms(model, batches, arms, warmup=3):
    state = {"step": 0}

    def step(b):
        state["step"] += 1
        loss = model.training_loss(b)
        model.fused_optimizer_step(lr=1e-4, step=state["step"])
        return loss

    def switch(on):
        if on:
            model.gradient_checkpointing_enable()
        else:
            model.gradient_checkpointing_disable()

    for name, on in arms.items():                    # warm-up of every arm
        switch(on)
        for i in range(warmup):
            step(batches[i % 2])
    torch.cuda.synchronize()
    res = {name: {"ms_per_step": [], "peak_mem_gib": [], "loss_last": None} for name in arms}
    for rnd in range(ROUNDS):
        order = list(arms) if rnd % 2 == 0 else list(arms)[::-1]
        for name in order:
            switch(arms[name])
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(K):
                loss = step(batches[i % 2])
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms_per_step"].append(round(e0.elapsed_time(e1) / K, 2))
            res[name]["peak_mem_gib"].append(round(torch.cuda.max_memory_allocated(dev) / GiB, 2))
            res[name]["loss_last"] = round(float(loss), 4)
    return res


out = {"card": card(), "steps_per_window": K, "rounds": ROUNDS,
       "step": "training_loss + fused_optimizer_step, bf16, synthetic batches (midi_b200.synth)"}
t0 = time.time()

# tv2o-medium, B = 8 x 2048: both arms
cfg, model, batches = build("tv2o-medium", 8, 2048)
out["medium"] = {"workload": "tv2o-medium, B=8, 2048 events x 8 tokens",
                 "saved_activation_estimate_gib": {a: round(saved_bytes(cfg, 8, 2048, a == "checkpointed") / GiB, 2)
                                                   for a in ("default", "checkpointed")},
                 "arms": run_arms(model, batches, {"default": False, "checkpointed": True})}
del model, batches
gc.collect()
torch.cuda.empty_cache()

# tv2o-large, B = 8 x 4096 (config 5): checkpointed, then the default arm only if its estimate fits
cfg, model, batches = build("tv2o-large", 8, 4096)
large = {"workload": "tv2o-large, B=8, 4096 events x 8 tokens (BASELINE.json config 5)",
         "saved_activation_estimate_gib": {a: round(saved_bytes(cfg, 8, 4096, a == "checkpointed") / GiB, 2)
                                           for a in ("default", "checkpointed")}}
large["arms"] = run_arms(model, batches, {"checkpointed": True}, warmup=2)
peak_ck = max(large["arms"]["checkpointed"]["peak_mem_gib"]) * GiB
estimate = peak_ck + saved_bytes(cfg, 8, 4096, False) - saved_bytes(cfg, 8, 4096, True)
gc.collect()
torch.cuda.empty_cache()
free, total = torch.cuda.mem_get_info(dev)
headroom = free + torch.cuda.memory_allocated(dev)     # what this process could hold: its own tensors stay
large["default_estimate_gib"] = round(estimate / GiB, 2)
large["free_for_this_process_gib"] = round(headroom / GiB, 2)
if estimate + MARGIN <= headroom:
    large["arms"].update(run_arms(model, batches, {"default": False}, warmup=2))
else:
    large["default"] = (f"not run: estimate {estimate / GiB:.1f} GiB (+ {MARGIN / GiB:.0f} GiB margin) > free "
                        f"{headroom / GiB:.1f} GiB")
out["large"] = large
out["card_after"] = card()
out["wall_s"] = round(time.time() - t0, 1)

lines = [f"card: {out['card']['device']} | nvidia-smi (name, power.limit, clocks.max.sm): {out['card']['nvidia_smi']}",
         f"card after the run: {out['card_after']['nvidia_smi']}",
         f"one step = {out['step']}; {K} steps per window, {ROUNDS} windows per arm, arms alternating", ""]
for key in ("medium", "large"):
    w = out[key]
    lines.append(f"{w['workload']}  (saved activations from the shapes: default "
                 f"{w['saved_activation_estimate_gib']['default']} GiB, checkpointed "
                 f"{w['saved_activation_estimate_gib']['checkpointed']} GiB)")
    for name, r in w["arms"].items():
        ms = sorted(r["ms_per_step"])
        lines.append(f"  {name:>12}: {ms[len(ms) // 2]:8.2f} ms/step (median; all {r['ms_per_step']}), "
                     f"peak allocated {max(r['peak_mem_gib']):6.2f} GiB, last loss {r['loss_last']}")
    if "default" in w:
        lines.append(f"  {'default':>12}: {w['default']}")
    lines.append("")
med = out["medium"]["arms"]
md = sorted(med["default"]["ms_per_step"])[ROUNDS // 2]
mc = sorted(med["checkpointed"]["ms_per_step"])[ROUNDS // 2]
lines.append(f"medium: checkpointing costs {100 * (mc / md - 1):.1f} % step time and peak memory goes from "
             f"{max(med['default']['peak_mem_gib']):.2f} to {max(med['checkpointed']['peak_mem_gib']):.2f} GiB")
text = "\n".join(lines) + "\n"
os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "recompute_step_time.json"), "w") as f:
    json.dump(out, f, indent=1)
with open(os.path.join(OUT_DIR, "recompute_step_time.txt"), "w") as f:
    f.write(text)
print(json.dumps(out, indent=1))
print(text)
