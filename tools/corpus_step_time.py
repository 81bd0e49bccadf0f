"""The fused trainer fed from an on-disk corpus (midi_b200/corpus.py) against the same batches pre-built in pinned memory,
at tv2o-medium, B = 8, max_len 2048: one step = Prefetcher item -> data.augment_ -> training_loss(batch, lengths) +
fused_optimizer_step, the ragged step.

  loader   -- Corpus.batches (one background thread cropping from the memory map into pinned batches);
  prebuilt -- the very batches the loader arm gets (epoch 0, in order), built before timing in pinned memory and fed
              through the same Prefetcher and augment_.

The arms alternate in one process, each timed with CUDA events after a warm-up.  Also reported: the loader thread's host
time per batch, the augment kernel's time (CUDA events over repeated launches on one batch), and the builder's files/s on
this machine's CPU.  The corpus is synthetic: a few thousand files of 300 ... 8000 events of random well-formed v2 rows,
stored as raw int16 rows, so the builder's rate here covers reading, the filters, the row checks, the metadata and the
writes, and not MIDI parsing or tokenising (that is the reference's midi2score + tokenize, paid once per file).  The card
name and power limit are read in the same run.  Writes $MIDI_TOOLS_OUT/corpus_step_time.json and prints a summary.

    python tools/corpus_step_time.py [steps per window] [rounds] [files]
"""
import json
import os
import platform
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
for p in (os.path.join(ROOT, "midi-model_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402

import midi_model as mm  # noqa: E402
from midi_b200 import corpus as CO, data  # noqa: E402
from midi_b200.tokenizer_tables import TokenizerTables  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 20
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 4
N_FILES = int(sys.argv[3]) if len(sys.argv) > 3 else 3000
B, MAX_LEN, WARMUP = 8, 2048, 6
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


def cpu():
    name = platform.processor()
    try:
        with open("/proc/cpuinfo") as f:
            name = next((ln.split(":", 1)[1].strip() for ln in f if ln.startswith("model name")), name)
    except OSError:
        pass
    return {"model": name, "machine": platform.machine(), "logical_cpus": os.cpu_count()}


class RowTokenizer(TokenizerTables):
    """The v2 tables; a 'score' here is already the token rows (see rows_score)."""

    def tokenize(self, score):
        return score[1]


def rows_score(datas: bytes):
    return [480, np.frombuffer(datas, dtype="<i2").reshape(-1, 8)]


def synth_files(tok, n_files, path, seed=0):
    """Random well-formed v2 files of 300 ... 8000 events (BOS / EOS included), raw int16 rows."""
    rng = np.random.default_rng(seed)
    ev_ids = np.array([tok.event_ids[e] for e in tok.events])
    lo = np.full((len(ev_ids), 8), tok.pad_id)
    span = np.ones((len(ev_ids), 8), np.int64)
    for k, (name, ps) in enumerate(tok.events.items()):
        for j, p in enumerate(ps):
            lo[k, 1 + j] = tok.parameter_ids[p][0]
            span[k, 1 + j] = tok.event_parameters[p]
    pitch_col, note_k = 1 + tok.events["note"].index("pitch"), list(tok.events).index("note")
    special = np.full((1, 8), tok.pad_id)
    paths = []
    for i in range(n_files):
        n = int(rng.integers(300, 8001))
        k = rng.integers(0, len(ev_ids), n - 2)
        rows = lo[k] + (rng.random((n - 2, 8)) * span[k]).astype(np.int64)
        rows[:, 0] = ev_ids[k]
        notes = k == note_k
        rows[notes, pitch_col] = tok.parameter_ids["pitch"][0] + rng.integers(24, 100, int(notes.sum()))
        bos, eos = special.copy(), special.copy()
        bos[0, 0], eos[0, 0] = tok.bos_id, tok.eos_id
        p = os.path.join(path, f"{i:05d}.mid")
        with open(p, "wb") as f:
            f.write(np.concatenate([bos, rows, eos]).astype("<i2").tobytes())
        paths.append(p)
    return paths


out = {"workload": f"tv2o-medium ragged fused train step (augment_ + training_loss(batch, lengths) + fused_optimizer_step), "
                   f"B={B}, max_len {MAX_LEN}, bf16", "steps_per_window": K, "rounds": ROUNDS, "card": card(), "cpu": cpu()}
tmp = tempfile.mkdtemp(prefix="corpus_step_time_")
try:
    tok = RowTokenizer("v2")
    t0 = time.time()
    paths = synth_files(tok, N_FILES, tmp)
    out["synth_files_s"] = round(time.time() - t0, 1)
    build = {}
    for workers in sorted({1, min(8, os.cpu_count() or 1)}):
        t0 = time.perf_counter()
        man = CO.build_corpus(paths, os.path.join(tmp, f"corpus{workers}"), tok, workers=workers, midi2score=rows_score)
        dt = time.perf_counter() - t0
        build[f"workers_{workers}"] = {"files_per_s": round(len(paths) / dt, 1), "s": round(dt, 2)}
    out["builder"] = {"files": len(paths), "events": man["n_events"], "skipped": man["skipped"], **build}
    corpus = CO.Corpus(os.path.join(tmp, f"corpus{workers}"), tok)

    torch.manual_seed(0)
    model = mm.MIDIModel(mm.MIDIModelConfig.from_name("tv2o-medium")).to(dev, dtype=torch.bfloat16).train()
    n_steps = WARMUP + K * ROUNDS
    loader = corpus.batches(B, MAX_LEN, seed=0, epoch=0)
    if len(loader) < n_steps:
        raise SystemExit(f"{len(corpus)} files give {len(loader)} batches per epoch; the run needs {n_steps}")
    prebuilt = [loader.batch(i) for i in range(n_steps)]
    feeds = {"loader": iter(data.Prefetcher(loader, dev)), "prebuilt": iter(data.Prefetcher(iter(prebuilt), dev))}
    state = {"step": 0, "tokens": {"loader": 0, "prebuilt": 0}}

    def step(name):
        tokens, lengths, aug = next(feeds[name])
        data.augment_(tokens, aug)
        state["step"] += 1
        loss = model.training_loss(tokens, lengths=lengths)
        model.fused_optimizer_step(lr=1e-4, step=state["step"])
        state["tokens"][name] += sum(lengths)
        return loss

    for name in feeds:                        # warm-up: module loads, GEMM plans of several packed sizes
        for _ in range(WARMUP):
            step(name)
    torch.cuda.synchronize()
    res = {name: {"ms_per_step": []} for name in feeds}
    for rnd in range(ROUNDS):
        order = list(feeds) if rnd % 2 == 0 else list(feeds)[::-1]
        for name in order:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            state["tokens"][name] = 0
            e0.record()
            for _ in range(K):
                loss = step(name)
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms_per_step"].append(round(e0.elapsed_time(e1) / K, 2))
            res[name].setdefault("events_per_window", []).append(state["tokens"][name])
    for r in res.values():
        r["median_ms"] = sorted(r["ms_per_step"])[len(r["ms_per_step"]) // 2]
    out["arms"] = res
    assert res["loader"]["events_per_window"] == res["prebuilt"]["events_per_window"]
    host = np.array(loader.host_s) * 1e3
    out["loader_host_ms_per_batch"] = {"n": int(host.size), "median": round(float(np.median(host)), 3),
                                      "p90": round(float(np.percentile(host, 90)), 3), "max": round(float(host.max()), 3)}

    # augment kernel alone, on a full batch (B x 2048 rows), many launches between two events
    loader.close()
    tokens, lengths, aug = prebuilt[0]
    tb, ab = tokens.to(dev), aug.to(dev)
    for _ in range(10):
        data.augment_(tb, ab)
    torch.cuda.synchronize()
    n_launch = 500
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_launch):
        data.augment_(tb, ab)
    e1.record()
    torch.cuda.synchronize()
    out["augment_kernel_us"] = {"rows": int(tb.shape[0] * tb.shape[1]), "us_per_launch": round(e0.elapsed_time(e1) * 1e3 / n_launch, 2)}
    out["card_after"] = card()
finally:
    shutil.rmtree(tmp, ignore_errors=True)

os.makedirs(OUT_DIR, exist_ok=True)
with open(os.path.join(OUT_DIR, "corpus_step_time.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out, indent=1))
ld_ms, pb_ms = out["arms"]["loader"]["median_ms"], out["arms"]["prebuilt"]["median_ms"]
print(f"loader {ld_ms:.2f} ms/step vs prebuilt {pb_ms:.2f} ms/step: loader / prebuilt = {ld_ms / pb_ms:.4f}")
print(f"loader thread {out['loader_host_ms_per_batch']['median']:.3f} ms per batch (median), augment kernel "
      f"{out['augment_kernel_us']['us_per_launch']:.2f} us per launch, builder {out['builder']}")
