"""LoRA step time at the benchmark shape (tv2o-medium, B=8 x 2048 events x 8 tokens): train.py --task lora
(r = 64, lora_alpha = 128, all seven projections, frozen base; train.py:439-449) on the fused trainer
(training_loss + fused_optimizer_step over the adapter tail), then the full-training step of the same model for comparison.
Writes $MIDI_TOOLS_OUT/lora_step_time.json after each leg.

    python tools/lora_step_time.py [steps]
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
for p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402

import midi_model as mm  # noqa: E402
from midi_b200 import lib, lora, ops  # noqa: E402
from midi_b200.synth import synth_batch  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 5
dev = torch.device("cuda", 0)
out = {"workload": "tv2o-medium train step, B=8, 2048 events x 8 tokens, bf16", "steps": K}
os.makedirs(OUT_DIR, exist_ok=True)


def dump():
    with open(os.path.join(OUT_DIR, "lora_step_time.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out), flush=True)


def timed(model, batches, tag):
    state = {"s": 0}

    def step(b):
        state["s"] += 1
        loss = model.training_loss(b)
        model.fused_optimizer_step(lr=1e-4, step=state["s"])
        return loss

    for i in range(3):
        step(batches[i % len(batches)])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    l0 = lib.query("b200_launch_count")
    ops.GEMM_PROFILE = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K):
        loss = step(batches[i % len(batches)])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    out[tag] = {"ms_per_step": round(ms, 3), "tokens_per_s": round(8 * 2048 * 8 / ms * 1e3), "loss_last": float(loss),
                "launches_per_step": (lib.query("b200_launch_count") - l0) / K,
                "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    dump()


t0 = time.time()
torch.manual_seed(0)
model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).train()
batches = [synth_batch(model.tokenizer, 8, 2049, seed=1234 + i).to(dev) for i in range(2)]
out["setup_s"] = round(time.time() - t0, 1)
model.requires_grad_(False)
model.add_adapter(lora.LoraAdapterConfig(r=64, lora_alpha=128, lora_dropout=0, bias="none", task_type="CAUSAL_LM",
                                         target_modules=["q_proj", "o_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "down_proj"]))
rt = model._rt()
out["adapter_params"] = int(rt.store.numel - rt.store.base_numel)
timed(model, batches, "lora")
del model, rt
torch.cuda.empty_cache()
torch.manual_seed(0)
full = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).train()
timed(full, batches, "full")
