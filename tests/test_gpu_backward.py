"""GPU tests (`pytest -m gpu`) of the training backward that chains the sm_90a kernels: StackEngine.backward of both stacks
and the fused step's _inner_backward / training_loss, scored gradient by gradient against float64 autograd.

Every kernel has its own conformance group; what those cannot see is the wiring between them -- the wrong saved tensor
fed to a kernel, a residual gradient (`dres`) or an `accumulate` flag one gradient ignores, the LoRA scale at one site,
the weight-gradient GEMMs on the side stream and their operands' lifetimes, the checkpoint recompute, the segment path.
Such a mistake stays inside one tensor, one head or one layer, under the global gradient norm the model-level checks
bound.  So each gradient is scored on its own (tests/parity_metrics.grad_report): relative Frobenius error per tensor,
worst head of dWq / dWk / dWv / dWo, worst output row of every weight, worst token row of dx, worst element of every norm
weight; and each of those as a ratio to the same error of the bf16 eager oracle under autograd (the reference's own
rounding), which is the forward's noise-floor protocol applied per tensor.

The reference (parity_metrics.stack64) is float64 throughout, on the same bf16 weights and inputs, with the engine's own
RoPE tables (scored by the rope group), one sequence at a time.  Exact claims are bounded at 0; every other bound is
about 5x the worst value measured on an H100, which is given beside it.  `min:` counters make a smaller sweep fail."""
import contextlib

import pytest
import torch

import gpu_model as GM
import parity_metrics as P
from host_model import BF, TARGETS, make_batch
from parity_metrics import assert_within

DEV = "cuda"
EV_SHAPES = [(2, 1000), (3, 129), (1, 2048)]     # event-level (n_seq, S): partial 64-row tiles, and one long sequence
TOK_SHAPES = [512, 1000]                         # token-level sequences of 8 tokens
SWITCH_EV, SWITCH_TOK = (3, 129), 512            # the shapes the switches, accumulate and LoRA run at
SEG_LENGTHS = [700, 65, 1300]                    # packed sequences that leave gap rows
STEP_B, STEP_S1, STEP_PAD = 2, 66, 3             # the whole fused step: check_model_train's batch
HANDOVER_S1 = 130

# metric-name prefix -> bound.  Measured worst values over every case of this file (H100 80GB HBM3, 700 W power limit) in
# the comments; each tensor's error sits within 1.15x of the bf16 floor's in norm and per head.
BOUNDS = [
    ("floor_ratio_fro", 1.5),                    # 1.11  (q_proj, step with sample_idx)
    ("floor_ratio_head", 1.5),                   # 1.15  (k_proj, step with lengths)
    ("floor_ratio_row", 3.0),                    # 2.10  (q_proj rows, step with sample_idx)
    ("floor_ratio_elem", 2.5),                   # 1.57  (post_attention_layernorm, step)
    ("floor_ratio_dxrow", 1.5),                  # 0.94  (event-level LoRA)
    ("fro", 7e-2),                               # 1.37e-2 (q_proj, step with sample_idx)
    ("row", 1.2),                                # 0.243 (a q_proj row of small norm, step with sample_idx)
    ("dxrow", 3e-2),                             # 5.97e-3 (event-level LoRA)
    ("head", 0.13),                              # 2.59e-2 (k_proj, step with lengths)
    ("elem", 7e-3),                              # 1.46e-3 (post_attention_layernorm, step with sample_idx)
    ("min:n_tensors", 1.0),
    ("min:n_heads", 1.0),
    ("min:cases", 1.0),
    ("gemm_mismatch", 0.0),                      # GEMM-produced gradients and dx that must agree bit for bit
    ("atomic_rel", 1e-3),                        # 2.7e-5: norm-weight gradients summed with fp32 atomics, global relative
    ("gap_dx_nonzero", 0.0),                     # dx on gap rows of the packed layout
    ("lora_frozen_span_written", 0.0),           # frozen base span of the flat gradient buffer written by a LoRA run
    ("embed_changed", 0.0),                      # token-level embedding gradient under n_ids = 0
    ("embed_nonzero", 0.0),
    ("loss_abs", 3e-3),                          # 5.3e-4 (step with sample_idx)
    ("handover_mismatch", 0.0),                  # elements of a handed-over slice that changed after the hand-over
    ("handover_cover_error", 0.0),
    ("min:handover_calls", 1.0),
]
INFO = ("fused_mismatch", "peak_gib", "seconds")     # reported without a bound


def check(m, bounds=()):
    """assert_within over `bounds` (placed before the table, so they take precedence) and BOUNDS, INFO names reported."""
    assert_within(m, list(bounds) + BOUNDS, tuple(k for k in m if k.startswith(INFO)))


def _sync():
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def medium():
    """tv2o-medium (12 event-level layers, 3 token-level) in bf16, seeded."""
    model = GM.cuda_model(GM.config("tv2o-medium"))
    yield model
    del model
    torch.cuda.empty_cache()


def _add_lora(model):
    """train.py:440-449 with r = 64, lora_alpha = 128 on all seven projections; B non-zero (B = 0 makes dA vanish)."""
    from midi_b200 import lora
    model.requires_grad_(False)
    model.add_adapter(lora.LoraAdapterConfig(r=64, lora_alpha=128, target_modules=TARGETS, lora_dropout=0, bias="none",
                                             task_type="CAUSAL_LM"))
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if ".lora_B." in n:
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device, BF))
    return model


@pytest.fixture(scope="module")
def medium_lora():
    model = _add_lora(GM.cuda_model(GM.config("tv2o-medium")))
    yield model
    del model
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ one stack, two layers
@contextlib.contextmanager
def _two_layers(eng):
    """The stack cut to its first two layers, so that the add between layers (add_rmsnorm) and its dres are exercised."""
    keep = eng.layers
    eng.layers = keep[:2]
    try:
        yield eng
    finally:
        eng.layers = keep


def _in_two(eng, name):
    p = eng.cfg.prefix
    if name == f"{p}.norm.weight":
        return True
    return name.startswith(f"{p}.layers.") and int(name.split(".")[2]) < 2


def _inv(model, eng):
    return (model.net if eng.cfg.prefix == "net" else model.net_token).rotary_emb.inv_freq


def _randn(shape, seed, scale=1.0):
    """bf16 normal values times `scale`, a power of two (so it commutes with the rounding)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV).to(BF) * scale


class Case:
    """One stack backward: inputs x / dy [rows, H], the sequences as row-index groups [B, S] for the reference, and how
    the engine runs (n_seq, S, seg)."""

    def __init__(self, eng, n_seq, S, seed, seg=None, groups=None, live=None):
        H = eng.cfg.hidden
        self.n_seq, self.S, self.seg = n_seq, S, seg
        rows = n_seq * S
        self.x = _randn((rows, H), seed)
        self.dy = _randn((rows, H), seed + 1, 2.0 ** -8)
        if live is not None:
            self.dy[~live] = 0
        if groups is None:
            idx = torch.arange(rows, device=DEV).view(n_seq, S)
            groups = [idx[b:b + 1] for b in range(n_seq)] if eng.cfg.prefix == "net" else [idx]
        self.groups = groups


def _names(eng, grads):
    names = [n for n in eng.names if _in_two(eng, n)]
    return [n for n, v in zip(names, grads.named(names)) if v is not None]


def run_engine(eng, model, case, grads=None, checkpoint=False, accumulate=False, g0=None):
    """forward(save=True) + backward of the (cut) stack -> {name: gradient, "dx": dx} (clones)."""
    y, sv = eng.forward(case.x, case.n_seq, case.S, _inv(model, eng), save=True, checkpoint=checkpoint, seg=case.seg)
    g = eng.fresh_grads() if grads is None else grads
    names = _names(eng, g)
    if g0 is not None:
        for n, v in zip(names, g.named(names)):
            v.copy_(g0[n])
    dx = eng.backward(sv, case.dy, g, accumulate=accumulate)
    _sync()
    out = {n: v.clone() for n, v in zip(names, g.named(names))}
    out["dx"] = dx.clone()
    return out


def reference(eng, model, case, names, lora_scale=None, floor=True):
    """fp64 autograd of stack64 over the first two layers, group by group (weight gradients summed), and the same
    gradients of the bf16 eager oracle (oracle.midi_oracle.llama_stack on bf16 leaves) -> (ref, floor)."""
    from midi_b200 import ops
    from oracle import midi_oracle as O
    c = eng.cfg
    cfg2 = O.StackCfg(c.prefix, 2, c.n_head, c.hidden, c.inner, c.eps)
    inv = _inv(model, eng)
    cos, sin = ops.rope_table(inv, max(gr.shape[1] for gr in case.groups))
    store = eng.store
    params = [n for n in eng.names if _in_two(eng, n)]
    wnames = [n for n in names if n != "dx"]
    out = []
    for dt in ((torch.float64, BF) if floor else (torch.float64,)):
        acc = {n: torch.zeros(store.views[n].shape, dtype=torch.float64, device=DEV) for n in wnames}
        acc["dx"] = torch.zeros(case.x.shape, dtype=torch.float64, device=DEV)
        for idx in case.groups:
            leaf = {n: store.views[n].detach().to(dt).requires_grad_(n in acc) for n in params}
            sd = O.lora_effective_sd(leaf, lora_scale) if lora_scale is not None else leaf
            xb = case.x[idx].to(dt).requires_grad_(True)
            if dt == torch.float64:
                y = P.stack64(sd, cfg2, xb, cos, sin)
            else:
                y = O.llama_stack(sd, cfg2, xb, inv)
            gr = torch.autograd.grad(y, [xb] + [leaf[n] for n in wnames], case.dy[idx].to(dt))
            acc["dx"][idx.reshape(-1)] = gr[0].double().reshape(-1, c.hidden)
            for n, t in zip(wnames, gr[1:]):
                acc[n] += t.double()
            del leaf, sd, xb, y, gr
        out.append(acc)
    return out[0], (out[1] if floor else None)


def score(got, ref, fl, eng, tag):
    return P.grad_report(got, ref, tag, eng.cfg.n_head, fl)


def exact(a, b, tag):
    """Bit-for-bit agreement of two runs, except the norm-weight gradients (fp32 atomics in a run-dependent order)."""
    gemm = [n for n in a if not GM.atomic(n)]
    atom = [n for n in a if GM.atomic(n)]
    m = {f"gemm_mismatch_{tag}": float(sum(int((a[n] != b[n]).sum()) for n in gemm))}
    if atom:
        m[f"atomic_rel_{tag}"] = GM.global_rel({n: b[n] for n in atom}, {n: a[n] for n in atom})
    return m


def mismatch(a, b):
    """Differing elements of GEMM-produced gradients and dx (the norm-weight gradients differ between any two runs)."""
    return float(sum(int((a[n] != b[n]).sum()) for n in a if not GM.atomic(n)))


def _stacks(model):
    rt = model._rt()
    return [("ev", rt.outer, shape) for shape in EV_SHAPES] + [("tok", rt.inner, (n, 8)) for n in TOK_SHAPES]


def _peak(m, tag, t0):
    import time
    m[f"peak_gib_{tag}"] = torch.cuda.max_memory_allocated() / 2 ** 30
    m[f"seconds_{tag}"] = time.time() - t0


# ------------------------------------------------------------------------------------------ (a) teacher-forced stacks
@pytest.mark.gpu
def test_stack_backward_vs_fp64(medium):
    """Two layers of each stack, random bf16 x and dy, every gradient and dx against fp64 and the bf16 floor."""
    import time
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    m = {}
    cases = 0
    for kind, eng, (n_seq, S) in _stacks(medium):
        with _two_layers(eng):
            case = Case(eng, n_seq, S, seed=10 + n_seq + S)
            got = run_engine(eng, medium, case)
            ref, fl = reference(eng, medium, case, list(got))
            m.update(score(got, ref, fl, eng, f"{kind}_{n_seq}x{S}"))
            cases += 1
            del got, ref, fl
    m["cases_stack"] = float(cases)
    _peak(m, "stack", t0)
    check(m, [("min:cases_stack", len(EV_SHAPES) + len(TOK_SHAPES))])


# ------------------------------------------------------------------------------------------ (b) switches
def _switch_runs(monkeypatch, model, eng, case, tag):
    """The default run, then every switch that claims the same result -> metrics."""
    from midi_b200 import engine
    m = {}
    base = run_engine(eng, model, case)
    ref, fl = reference(eng, model, case, list(base))
    with monkeypatch.context() as mp:
        mp.setattr(engine, "WGRAD_STREAM", False)
        m.update(exact(base, run_engine(eng, model, case), f"{tag}_one_stream"))
    m.update(exact(base, run_engine(eng, model, case, checkpoint=True), f"{tag}_checkpoint"))
    for name, val in (("FUSE_ROPE", False), ("FUSE_ROPE_FWD", True), ("FUSE_SWIGLU", False)):
        with monkeypatch.context() as mp:
            mp.setattr(engine, name, val)
            got = run_engine(eng, model, case)
        sw = f"{tag}_{name.lower()}_{int(val)}"
        m.update(score(got, ref, fl, eng, sw))
        m[f"fused_mismatch_{sw}"] = mismatch(got, base)
    return m


@pytest.mark.gpu
def test_switches_claiming_identical_results(medium, monkeypatch):
    """WGRAD_STREAM off and checkpoint=True: bit-identical.  FUSE_ROPE=0, FUSE_ROPE_FWD=1, FUSE_SWIGLU=0: scored against
    fp64 with the same bounds (their mismatch count against the default path is reported)."""
    rt = medium._rt()
    m = {}
    with _two_layers(rt.outer):
        m.update(_switch_runs(monkeypatch, medium, rt.outer, Case(rt.outer, *SWITCH_EV, seed=20), "ev"))
    with _two_layers(rt.inner):
        m.update(_switch_runs(monkeypatch, medium, rt.inner, Case(rt.inner, SWITCH_TOK, 8, seed=21), "tok"))
    check(m)


# ------------------------------------------------------------------------------------------ (c) accumulate
@pytest.mark.gpu
def test_accumulate_adds_to_every_gradient(medium):
    """Every gradient view pre-filled with a non-zero G0 (random, the size of the gradient itself), backward with
    accumulate=True, scored against fp64 G0 + g: a gradient that ignores the flag is off by the size of G0."""
    import midi_model as mm
    from midi_b200 import ops
    rt = medium._rt()
    m = {}
    for tag, eng, (n_seq, S) in (("ev", rt.outer, SWITCH_EV), ("tok", rt.inner, (SWITCH_TOK, 8))):
        with _two_layers(eng):
            case = Case(eng, n_seq, S, seed=30 + n_seq)
            got = run_engine(eng, medium, case)
            names = [n for n in got if n != "dx"]
            ref, _ = reference(eng, medium, case, names + ["dx"], floor=False)
            g0 = {n: _randn(ref[n].shape, 40 + i, 1.0) * float(ref[n].pow(2).mean().sqrt()) for i, n in enumerate(names)}
            got = run_engine(eng, medium, case, accumulate=True, g0=g0)
            ref = {n: (v + g0[n].double() if n in g0 else v) for n, v in ref.items()}
            m.update(P.grad_report(got, ref, f"{tag}_accumulate", eng.cfg.n_head))
    # token-level input without ids (n_ids = 0): the embedding gradient is zeroed only when not accumulating, and
    # lm_head's gradient accumulates on the side stream
    eng = rt.inner
    with _two_layers(eng):
        N = 64
        x = _randn((N, rt.H), 50)
        for acc in (False, True):
            hs, sv = eng.forward(x, N, 1, _inv(medium, eng), save=True)
            dl = torch.zeros((N, rt.pitch), dtype=BF, device=DEV)
            dl[:, :rt.V] = _randn((N, rt.V), 51, 2.0 ** -6)
            g = eng.fresh_grads()
            g0 = _randn(g.embed.shape, 52)
            g.embed.copy_(g0)
            h0 = _randn(rt.lm_head.shape, 53, 2.0 ** -4)
            g_head = h0.clone()
            mm._inner_backward(rt, medium, sv, hs, dl, None, N, 1, 0, True, g, g_head, acc)
            _sync()
            if acc:
                m["embed_changed_n_ids0"] = float((g.embed != g0).sum())
                want = h0.double() + dl[:, :rt.V].double().T @ hs.double()
                m["fro_lm_head_accumulate"] = P._rel(g_head.double(), want)
            else:
                m["embed_nonzero_n_ids0"] = float((g.embed != 0).sum())
    check(m)


# ------------------------------------------------------------------------------------------ (d) segment path
@pytest.mark.gpu
def test_segment_packed_backward(medium):
    """The event-level stack on sequences packed tile-aligned (midi_model._ragged_layout) with gap rows; the reference
    runs each sequence alone and sums the weight gradients; dx is exactly 0 on gap rows (their dy is 0)."""
    import midi_model as mm
    rt = medium._rt()
    eng = rt.outer
    stride = max(SEG_LENGTHS) + 1
    src, seg = mm._ragged_layout(SEG_LENGTHS, stride, torch.device(DEV))
    src = src.long()
    live = src >= 0
    groups = [torch.nonzero(live & (src // stride == b))[:, 0][None] for b in range(len(SEG_LENGTHS))]
    m = {}
    with _two_layers(eng):
        case = Case(eng, 1, seg.rows, seed=60, seg=seg, groups=groups, live=live)
        got = run_engine(eng, medium, case)
        ref, fl = reference(eng, medium, case, list(got))
        m.update(score(got, ref, fl, eng, "ev_segments"))
        m["gap_dx_nonzero"] = float((got["dx"][~live] != 0).sum())
        m["cases_gap_rows"] = float((~live).sum())
    check(m)


# ------------------------------------------------------------------------------------------ (e) LoRA
@pytest.mark.gpu
def test_lora_backward(medium_lora, monkeypatch):
    """r = 64, lora_alpha = 128 on all seven projections: the A and B gradients of every site against fp64 autograd of
    the effective weights W + scale B A, with and without the side stream.  The run writes the store's own flat
    gradient buffer, whose frozen base span is NaN beforehand and must still be afterwards."""
    from midi_b200 import engine
    rt = medium_lora._rt()
    store = rt.store
    m = {}
    for tag, eng, (n_seq, S) in (("ev", rt.outer, SWITCH_EV), ("tok", rt.inner, (SWITCH_TOK, 8))):
        with _two_layers(eng):
            case = Case(eng, n_seq, S, seed=70 + n_seq)
            runs = []
            for side in (True, False):
                with monkeypatch.context() as mp:
                    mp.setattr(engine, "WGRAD_STREAM", side)
                    store.gflat[:store.base_numel].fill_(float("nan"))
                    runs.append(run_engine(eng, medium_lora, case, grads=eng.main_grads))
                    m[f"lora_frozen_span_written_{tag}_side{int(side)}"] = float((~torch.isnan(store.gflat[:store.base_numel])).sum())
            got = runs[0]
            assert all(".lora_" in n for n in got if n != "dx") and len(got) == 1 + 2 * 7 * 2
            scale = eng.layers[0].lora["q"].scale
            ref, fl = reference(eng, medium_lora, case, list(got), lora_scale=scale)
            m.update(score(got, ref, fl, eng, f"{tag}_lora"))
            m.update(P.grad_report(runs[1], ref, f"{tag}_lora_one_stream", eng.cfg.n_head, fl, show=False))
            m.update(exact(runs[0], runs[1], f"{tag}_lora_one_stream"))
    check(m)


# ------------------------------------------------------------------------------------------ (f) the whole fused step
def _step_reference(model, batch, sample_idx=None, lora_scale=None):
    """fp64 train_loss64 and the bf16 eager oracle's autograd on the model's bf16 weights -> (loss64, ref, floor);
    with adapters (lora_scale) over the effective weights W + scale B A."""
    import torch.nn.functional as F
    from midi_b200 import ops
    from oracle import midi_oracle as O
    ocfg = O.cfg_from_hf(model.config)
    S, T = batch.shape[1] - 1, batch.shape[2]
    rope_net = ops.rope_table(model.net.rotary_emb.inv_freq, S)
    rope_tok = ops.rope_table(model.net_token.rotary_emb.inv_freq, T)
    out = []
    for dt in (torch.float64, BF):
        leaf = {n: p.detach().to(dt).requires_grad_(True) for n, p in model.named_parameters()}
        out.append((leaf, O.lora_effective_sd(leaf, lora_scale) if lora_scale is not None else leaf))
    (leaf, sd), (l16, sd16) = out
    loss = P.train_loss64(sd, ocfg, batch, rope_net, rope_tok, sample_idx)
    loss.backward()
    ref = {n: t.grad for n, t in leaf.items()}
    x, y = batch[:, :-1], batch[:, 1:]
    hidden = O.forward(sd16, ocfg, x, inv_freq=model.net.rotary_emb.inv_freq)
    if sample_idx is not None:
        hidden, y = hidden[:, list(sample_idx)], y[:, list(sample_idx)]
    y = y.reshape(-1, T)
    logits = O.forward_token(sd16, ocfg, hidden.reshape(-1, hidden.shape[-1]), y[:, :-1],
                             inv_freq=model.net_token.rotary_emb.inv_freq)
    F.cross_entropy(logits.reshape(-1, ocfg.vocab), y.reshape(-1), ignore_index=ocfg.pad_id).backward()
    return float(loss.detach()), ref, {n: t.grad for n, t in l16.items()}


def _heads(model):
    return {n: (model.config.net_config if n.startswith("net.") else model.config.net_token_config).num_attention_heads
            for n, _ in model.named_parameters()}


@pytest.mark.gpu
def test_fused_step_per_tensor():
    """model.training_loss (4 event-level layers, B = 2, S = 65 with a pad tail) against fp64: every named parameter's
    gradient bounded on its own, per tensor and as a ratio to its floor; also with sample_idx and with lengths."""
    model = GM.cuda_model()
    tok = model.tokenizer
    m = {}
    padded = make_batch(model, STEP_B, STEP_S1, seed=77, pad_tail=STEP_PAD).to(DEV)
    ragged = make_batch(model, seed=78, S1=STEP_S1, lengths=[STEP_S1, STEP_S1 - 25]).to(DEV)
    idx = GM.rand_idx(STEP_S1 - 1)
    for tag, batch, kw in (("step", padded, {}), ("step_sample_idx", padded, {"sample_idx": idx}),
                           ("step_lengths", ragged, {"lengths": [STEP_S1, STEP_S1 - 25]})):
        loss64, ref, fl = _step_reference(model, batch, kw.get("sample_idx"))
        loss, got, _ = GM.step(model, lambda gr: model.training_loss(batch, **kw))
        m[f"loss_abs_{tag}"] = abs(float(loss) - loss64)
        m.update(P.grad_report(got, ref, tag, _heads(model), fl))
        m[f"cases_{tag}"] = float(len(got) == len(ref))
    del model
    torch.cuda.empty_cache()
    check(m, [("min:n_tensors_step", 4 * 9 + 1 * 9 + 5)])


# ------------------------------------------------------------------------------------------ (g) the hand-over contract
def _handover(model, batch, tag):
    """training_loss with a grad_ready that snapshots every handed-over slice on the current stream (what GradSync.ready
    orders its all-reduce after): each snapshot must equal the final gradient bit for bit."""
    store = model._rt().store
    snaps = []

    def cb(lo, hi):
        snaps.append((lo, hi, store.gflat[lo:hi].clone()))
    for p in model.parameters():
        p.grad = None
    model.training_loss(batch, grad_ready=cb)
    _sync()
    bad = sum(int((s != store.gflat[lo:hi]).sum()) for lo, hi, s in snaps)
    m = {f"handover_mismatch_{tag}": float(bad), f"handover_calls_{tag}": float(len(snaps))}
    m.update({k.replace("grad_ready_cover_error", "handover_cover_error"): v
              for k, v in GM.cover(model, [(lo, hi) for lo, hi, _ in snaps], tag).items()})
    return m


@pytest.mark.gpu
def test_grad_ready_hands_over_final_values(medium, medium_lora):
    """12 event-level layers: layer_done hands over groups of three layers, then the last three one by one (8 calls in
    all); under LoRA the adapter tail is handed over at the end (1 call).  WGRAD_STREAM is on (the default)."""
    from midi_b200 import engine
    assert engine.WGRAD_STREAM
    m = {}
    m.update(_handover(medium, make_batch(medium, 2, HANDOVER_S1, seed=90).to(DEV), "full"))
    m.update(_handover(medium_lora, make_batch(medium_lora, 2, HANDOVER_S1, seed=91).to(DEV), "lora"))
    check(m, [("min:handover_calls_full", 8.0)])
