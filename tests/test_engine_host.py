"""Host logic of the engine on CPU: the layer schedule, gradient placement, LoRA composition (train.py:439-449), the
optimizer span and the autograd Functions, run over the CPU stand-in for the kernel layer (tests/mock_kernels.py) and
compared with the oracle's autograd.  The CUDA kernels themselves are checked on the GPU (tests/gpu_checks.py)."""
import os

import pytest
import torch
import torch.nn.functional as F

import host_model
import mock_kernels
from host_model import BF, TARGETS, oracle_padded as _oracle_grads


def _tiny_model(seed=0):
    import midi_model as mm
    model = host_model.tiny_model(seed)
    return mm, model.config, model


def _batch(model, B=2, S1=6, seed=1):
    from midi_b200.synth import synth_batch
    return synth_batch(model.tokenizer, B, S1, seed=seed)


def _stream(model, **kw):
    """Events of generate_stream as private copies (on the CPU stand-in `.cpu()` is a view of the loop's own buffer, which the
    next generation overwrites; on the GPU it is a copy)."""
    return [e.copy() for e in model.generate_stream(**kw)]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def test_engine_schedule_matches_oracle_autograd(monkeypatch):
    mock_kernels.install(monkeypatch)
    mm, cfg, model = _tiny_model()
    batch = _batch(model)
    ref_loss, ref = _oracle_grads(model, batch)
    loss = model.training_loss(batch)
    assert abs(float(loss) - ref_loss) < 3e-2
    num = sum(float((p.grad.double() - ref[n].double()).pow(2).sum()) for n, p in model.named_parameters())
    den = sum(float(ref[n].double().pow(2).sum()) for n in ref)
    assert (num / den) ** 0.5 < 3e-2
    rt = model._rt()
    assert rt.store.base_numel == rt.store.numel and rt.store.train_dense and (rt.store.train_lo, rt.store.train_hi) == (0, rt.store.numel)


def _lora_model(monkeypatch):
    mock_kernels.install(monkeypatch)
    mm, cfg, model = _tiny_model()
    return mm, host_model.add_lora(model)


def test_lora_container_layout_and_flat_store(monkeypatch):
    mm, model = _lora_model(monkeypatch)
    names = [n for n, _ in model.named_parameters()]
    assert "net.layers.0.self_attn.q_proj.base_layer.weight" in names
    assert "net.layers.0.self_attn.q_proj.lora_A.default.weight" in names
    assert "net_token.layers.0.mlp.down_proj.lora_B.default.weight" in names
    assert all(p.requires_grad == (".lora_" in n) for n, p in model.named_parameters())
    assert model._hf_peft_config_loaded and model.active_adapters() == ["default"]
    sd = model.get_adapter_state_dict("default")
    assert "net.layers.0.self_attn.q_proj.lora_A.weight" in sd and len(sd) == 2 * 7 * 5           # 4 + 1 layers
    rt = model._rt()
    st = rt.store
    # adapters form the contiguous trainable tail of the flat buffer; base layout unchanged (fused q|k|v, gate|up views)
    assert st.base_numel < st.numel and (st.train_lo, st.train_hi) == (st.base_numel, st.numel) and st.train_dense
    assert all((st.offsets[n] >= st.base_numel) == (".lora_" in n) for n in st.names)
    a = "net.layers.2.self_attn."
    aq, ak, av = (st.views[a + f"{p}_proj.lora_A.default.weight"] for p in "qkv")
    assert ak.data_ptr() == aq.data_ptr() + aq.numel() * 2 and av.data_ptr() == ak.data_ptr() + ak.numel() * 2
    assert rt.outer.layers[2].qkv.shape == (3 * 256, 256) and not rt.outer.layers[2].tr_qkv
    assert set(rt.outer.layers[0].lora) == {"q", "k", "v", "o", "gate", "up", "down"} and rt.has_lora
    assert rt.outer.main_grads.layers[0].qkv is None and rt.outer.main_grads.embed is None


def test_lora_fused_training_matches_oracle(monkeypatch):
    mm, model = _lora_model(monkeypatch)
    batch = _batch(model)
    ref_loss, ref = _oracle_grads(model, batch, lora_scale=2.0)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    calls = []
    loss = model.training_loss(batch, grad_ready=lambda a, b: calls.append((a, b)))
    assert abs(float(loss) - ref_loss) < 3e-2
    rt = model._rt()
    assert calls == [(rt.store.base_numel, rt.store.numel)]                  # one hand-over: the adapter tail
    worst = 0.0
    for n, p in model.named_parameters():
        if ".lora_" in n:
            assert p.grad is not None and ref[n].abs().max() > 0
            worst = max(worst, _rel(p.grad.float(), ref[n]))
        else:
            assert p.grad is None
    assert worst < 6e-2, worst
    # the fused optimizer runs over the adapter tail only: frozen base bit-identical, every adapter matrix moved
    model.fused_optimizer_step(lr=1e-2, step=1)
    for n, p in model.named_parameters():
        assert torch.equal(p, before[n]) != (".lora_" in n), n
    osd = model.optimizer_state_dict()
    assert osd["step"] == 1 and set(osd["state"]) == {n for n in before if ".lora_" in n}
    model.load_optimizer_state_dict(osd)


def test_lora_dropin_autograd_path_matches_fused(monkeypatch):
    mm, model = _lora_model(monkeypatch)
    batch = _batch(model)
    model.training_loss(batch)
    fused = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    for p in model.parameters():
        p.grad = None
    x, y = batch[:, :-1].contiguous(), batch[:, 1:].contiguous()             # train.py:169-185
    hidden = model.forward(x)
    hidden = hidden.reshape(-1, hidden.shape[-1])
    y = y.reshape(-1, y.shape[-1])
    logits = model.forward_token(hidden, y[:, :-1])
    loss = F.cross_entropy(logits.view(-1, model.tokenizer.vocab_size), y.view(-1), reduction="mean",
                           ignore_index=model.tokenizer.pad_id)
    loss.backward()
    for n, p in model.named_parameters():
        if ".lora_" in n:
            assert _rel(p.grad.float(), fused[n].float()) < 2e-2, n
        else:
            assert p.grad is None, n


def test_lora_save_merge_roundtrip_and_merged_decode_weights(monkeypatch, tmp_path):
    """train.py:234-244 writes adapter_config.json + adapter_model.safetensors; midi_model.py:109-114 merges them.  The
    merged weights the decode path folds on the device (engine.MergedStack) must be the same W + scale * B A."""
    from safetensors.torch import save_file
    from midi_b200.engine import MergedStack
    mm, model = _lora_model(monkeypatch)
    d = str(tmp_path / "lora")
    name = model.active_adapters()[0]
    model.peft_config[name].save_pretrained(d)
    save_file(model.get_adapter_state_dict(name), os.path.join(d, "adapter_model.safetensors"), metadata={"format": "pt"})
    base_sd = {n.replace(".base_layer", ""): p.detach().clone() for n, p in model.named_parameters() if ".lora_" not in n}
    fresh = mm.MIDIModel(model.config).to(BF)
    fresh.load_state_dict(base_sd)
    merged = fresh.load_merge_lora(d)
    rt = model._rt()
    ms = MergedStack(rt.outer)
    H = 256
    for li in (0, 3):
        a = f"net.layers.{li}.self_attn."
        for j, pn in enumerate(("q_proj", "k_proj", "v_proj")):
            W = dict(merged.named_parameters())[a + pn + ".weight"]
            got = ms.layers[li].qkv[j * H:(j + 1) * H]
            assert not torch.equal(W, base_sd[a + pn + ".weight"])
            assert _rel(got.float(), W.float()) < 1e-2                       # double vs single rounding of the sum
        Wd = dict(merged.named_parameters())[f"net.layers.{li}.mlp.down_proj.weight"]
        assert _rel(ms.layers[li].down.float(), Wd.float()) < 1e-2
    assert ms.layers[0].ln1 is rt.outer.layers[0].ln1 and ms.norm is rt.outer.norm
    # resume: adapter weights load back into an injected model without merging
    from midi_b200 import lora
    fresh2 = mm.MIDIModel(model.config).to(BF)
    fresh2.load_state_dict(base_sd)
    fresh2.requires_grad_(False)
    fresh2.add_adapter(lora.LoraAdapterConfig.from_pretrained(d))
    fresh2.load_adapter_weights(d)
    for (n1, p1), (n2, p2) in zip(model.named_parameters(), fresh2.named_parameters()):
        assert n1 == n2 and torch.equal(p1, p2), n1


def test_lora_rejects_what_the_engine_does_not_implement():
    import midi_model as mm
    from midi_b200 import lora
    from midi_b200.lib import B200Error
    torch.manual_seed(0)
    model = mm.MIDIModel(mm.MIDIModelConfig.get_config("v2", True, n_layer=4, n_head=4, n_embd=256, n_inner=512))
    with pytest.raises(B200Error):
        model.add_adapter(lora.LoraAdapterConfig(r=8, target_modules=TARGETS, lora_dropout=0.1))
    with pytest.raises(B200Error):
        model.add_adapter(lora.LoraAdapterConfig(r=6, target_modules=TARGETS))
    with pytest.raises(ValueError):
        model.add_adapter(lora.LoraAdapterConfig(r=8, target_modules=["no_such_proj"]))
    model.add_adapter(dict(r=8, lora_alpha=16, target_modules=["q_proj", "v_proj"]))
    with pytest.raises(ValueError):
        model.add_adapter(dict(r=8, lora_alpha=16, target_modules=["q_proj"]))          # same adapter name again
    with pytest.raises(B200Error):
        model.net.layers[0].self_attn.q_proj(torch.zeros(1, 256))                      # containers do not compute


def test_merged_decode_weights_follow_the_adapters(monkeypatch):
    """generate() on a model with injected adapters reads merged copies (engine.MergedStack); they must be re-folded after
    every kind of adapter update -- the fused AdamW (raw pointers), a torch optimizer (in-place ops), load_adapter_weights --
    and idle generate loops built on the old copies must be retired."""
    mm, model = _lora_model(monkeypatch)
    rt = model._rt()
    s0 = model._cached_stack("outer")
    assert s0.eng is not rt.outer and model._cached_stack("outer") is s0          # merged view, cached while nothing changes
    assert model._cached_stack("inner").eng is not rt.inner
    w0 = s0.eng.layers[0].qkv.clone()
    rt.gen_pool[("stale",)] = [object()]
    model.training_loss(_batch(model))
    model.fused_optimizer_step(lr=1e-2, step=1)                                      # (a) fused AdamW
    s1 = model._cached_stack("outer")
    assert s1 is not s0 and not torch.equal(s1.eng.layers[0].qkv, w0) and not rt.gen_pool
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-1)
    opt.step()                                                                       # (b) torch optimizer (grads are published)
    s2 = model._cached_stack("outer")
    assert s2 is not s1 and not torch.equal(s2.eng.layers[0].qkv, s1.eng.layers[0].qkv)
    sd = {k: torch.zeros_like(v) for k, v in model.get_adapter_state_dict().items()}
    model.load_adapter_weights(sd)                                                   # (c) B = 0: merged == base
    s3 = model._cached_stack("outer")
    assert s3 is not s2 and torch.equal(s3.eng.layers[0].qkv, rt.outer.layers[0].qkv)
    # a model without adapters keeps reading the engine's own weights
    mm2, cfg2, plain = _tiny_model()
    assert plain._cached_stack("outer").eng is plain._rt().outer


def test_kv_cached_call_modes_match_the_full_forward(monkeypatch):
    """midi_model.py:116-150 with a caller-owned DynamicCache (app.py:56-64 / midi_model.py:192-221): prefill + single-event
    steps across a KV page boundary (64 positions) == one full forward; forward_token's three call modes chained over the
    token-level cache == the uncached call.  Host logic (PagedKV, block tables, positions, call modes) over the mock kernels."""
    from transformers import DynamicCache
    mock_kernels.install(monkeypatch)
    mm, cfg, model = _tiny_model()
    model.eval()
    batch = _batch(model, B=2, S1=71, seed=3)
    with torch.no_grad():
        x = batch[:, :70]
        full = model.forward(x)
        c = DynamicCache()
        parts = [model.forward(x[:, :60], cache=c)] + [model.forward(x[:, t:t + 1], cache=c) for t in range(60, 70)]
        cached = torch.cat(parts, 1)
        assert _rel(cached.float(), full.float()) < 2e-2
        assert _rel(cached[:, 60:].float(), full[:, 60:].float()) < 2e-2             # the steps past the page boundary
        hidden = full[:, -1]
        toks = batch[:, 70, :7]
        ref = model.forward_token(hidden, toks)                                      # (hidden, x): [B, 8, V]
        c2 = DynamicCache()
        steps = [model.forward_token(hidden, None, cache=c2)]                        # (hidden, None, cache)
        steps += [model.forward_token(None, toks[:, i:i + 1], cache=c2) for i in range(7)]      # (None, x, cache)
        got = torch.cat(steps, 1)
        assert got.shape == ref.shape == (2, 8, model.tokenizer.vocab_size)
        assert _rel(got.float(), ref.float()) < 2e-2


def test_reference_shaped_generate_loop_is_greedy_and_grammar_valid(monkeypatch):
    """MIDIModel.generate's host-driven loop (B200_GENERATE=eager; midi_model.py:167-250: prompt handling, per-event cached
    forward, per-token cached forward_token + grammar mask + sampling, early exit after the event's last parameter, padding)
    over the mock kernels: every generated event parses, pads follow the parameters, and every greedy choice is the argmax of
    the ORACLE's fp32 logits for the same prefix up to a bf16-sized margin."""
    from oracle import midi_oracle as O
    mock_kernels.install(monkeypatch)
    monkeypatch.setenv("B200_GENERATE", "eager")
    mm, cfg, model = _tiny_model()
    model.eval()
    tok = model.tokenizer
    P, n_new, B = 5, 6, 2
    prompt = _batch(model, B=B, S1=P, seed=9).numpy()
    ids = model.generate(prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    assert ids.shape == (B, P + n_new, 8) and (ids[:, :P] == prompt).all()
    sd32 = {k: v.detach().float() for k, v in model.state_dict().items()}
    ocfg = O.cfg_from_hf(model.config)
    seq = torch.from_numpy(ids)
    exact = total = 0
    worst = 0.0
    n_types = len(tok.event_ids)
    for e in range(P, P + n_new):
        with torch.no_grad():
            hid = O.forward(sd32, ocfg, seq[:, :e], inv_freq=model.net.rotary_emb.inv_freq)[:, -1]
            lg = O.forward_token(sd32, ocfg, hid, seq[:, e, :7], inv_freq=model.net_token.rotary_emb.inv_freq)    # [B, 8, V]
        for b in range(B):
            row = ids[b, e]
            ev = int(row[0])
            assert tok.eos_id <= ev <= tok.eos_id + n_types
            if ev != tok.eos_id:
                assert tok.tokens2event(row.tolist()) != [], row                       # a complete, valid event
            name = {v: k for k, v in tok.event_ids.items()}.get(ev)
            params = tok.events[name] if name else []
            for t in range(8):
                if t == 0:
                    lo, hi = tok.eos_id, tok.eos_id + 1 + n_types
                elif t - 1 < len(params):
                    pid = tok.parameter_ids[params[t - 1]]
                    lo, hi = pid[0], pid[-1] + 1
                else:
                    assert row[t] == tok.pad_id                                        # midi_model.py:239-241
                    continue
                assert lo <= row[t] < hi
                margin = float(lg[b, t, lo:hi].max() - lg[b, t, row[t]])
                worst = max(worst, margin)
                exact += int(margin == 0.0)
                total += 1
    print("generate vs oracle fp32: worst margin", worst, "exact argmax", exact, "of", total)
    assert worst < 0.1 and exact >= 0.8 * total, (worst, exact, total)


def test_device_resident_loop_and_app_stream_host_logic(monkeypatch):
    """The device-resident loop issued from the host (B200_GENERATE=nograph: GraphGenerator state, device-side positions,
    per-event commit, stop rule) produces the events of the reference-shaped loop; `generate_stream` (app.py:27-120) yields
    the same events one by one, its `disable_*` options are a mask on top of the grammar, and a finished generation hands
    its loop state back for reuse."""
    mock_kernels.install(monkeypatch)
    mm, cfg, model = _tiny_model()
    model.eval()
    tok = model.tokenizer
    P, n_new, B = 4, 5, 2
    prompt = _batch(model, B=B, S1=P, seed=11).numpy()
    monkeypatch.setenv("B200_GENERATE", "eager")
    ref = model.generate(prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    monkeypatch.setenv("B200_GENERATE", "nograph")
    ids = model.generate(prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    assert ids.shape == ref.shape and (ids == ref).all()
    evs = _stream(model, prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    assert len(evs) == n_new and all(e.shape == (B, 8) and e.dtype.kind == "i" for e in evs)
    assert (torch.from_numpy(ids[:, P:]) == torch.stack([torch.from_numpy(e) for e in evs], 1)).all()
    rt = model._rt()
    key = (B, P + n_new, 1.0, 0.98, 1)
    assert len(rt.gen_pool.get(key, [])) == 1                               # the loop state went back to the pool ...
    gg = rt.gen_pool[key][0]
    # ... and is reused.  app.py:73-87 options are a mask on top of the grammar.  Make the plain run emit what the options can
    # forbid: boost patch_change (an event with a channel parameter) over the event type the model currently prefers.
    first = int(evs[0][0, 0])
    assert first not in (tok.eos_id, tok.event_ids["patch_change"])
    with torch.no_grad():
        model.lm_head.weight[tok.event_ids["patch_change"]] = 8 * model.lm_head.weight[first]
    plain = _stream(model, prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    assert rt.gen_pool[key][0] is gg
    pc = [e[0] for e in plain if int(e[0, 0]) == tok.event_ids["patch_change"]]
    assert pc, "the boosted event type must show up in the plain run"
    c0 = int(pc[0][4])                                                       # patch_change: time1 time2 track channel patch
    assert c0 in tok.parameter_ids["channel"]
    no_chan = _stream(model, prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1,
                      disable_channels=[tok.parameter_ids["channel"].index(c0)])
    assert c0 not in {int(v) for e in no_chan for v in e.reshape(-1)}
    assert any(int(e[0, 0]) == tok.event_ids["patch_change"] for e in no_chan)          # still allowed, on another channel
    no_pc = _stream(model, prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1, disable_patch_change=True,
                    disable_control_change=True)
    types = {int(e[b, 0]) for e in no_pc for b in range(B)}
    assert not (types & {tok.event_ids["patch_change"], tok.event_ids["control_change"]})
    assert int(gg.mask.sum()) == gg.mask.numel()                                      # mask reset when the loop is handed back
    for e in no_chan + no_pc:
        for b in range(B):
            assert int(e[b, 0]) == tok.eos_id or tok.tokens2event(e[b].tolist()) != []
    # prompt already at max_len: nothing to generate (app.py / midi_model.py:183-190)
    assert list(model.generate_stream(prompt=prompt, batch_size=B, max_len=P, top_k=1)) == []
    assert (model.generate(prompt=prompt, batch_size=B, max_len=P, top_k=1) == prompt).all()


def test_concurrent_streams_own_their_loop_state(monkeypatch):
    """gradio serves app.generate from several worker threads sharing one model and may resume a suspended generator on
    another thread (app.py:496): two interleaved `generate_stream` generators with the same settings must each own a loop state
    (no lock held across `yield`), produce what a lone run produces, and hand both states back to the pool."""
    import threading
    mock_kernels.install(monkeypatch)
    monkeypatch.setenv("B200_GENERATE", "nograph")
    mm, cfg, model = _tiny_model()
    model.eval()
    P, n_new, B = 3, 4, 1
    p1, p2 = _batch(model, B=B, S1=P, seed=21).numpy(), _batch(model, B=B, S1=P, seed=22).numpy()
    lone1 = _stream(model, prompt=p1, batch_size=B, max_len=P + n_new, top_k=1)
    lone2 = _stream(model, prompt=p2, batch_size=B, max_len=P + n_new, top_k=1)
    g1 = model.generate_stream(prompt=p1, batch_size=B, max_len=P + n_new, top_k=1)
    g2 = model.generate_stream(prompt=p2, batch_size=B, max_len=P + n_new, top_k=1)
    got1, got2, errors = [next(g1).copy()], [next(g2).copy()], []          # both suspended mid-generation on this thread ...

    def drain(g, out):
        try:
            out.extend(e.copy() for e in g)                    # ... and resumed on other threads
        except Exception as e:                                 # noqa: BLE001
            errors.append(e)

    t1, t2 = threading.Thread(target=drain, args=(g1, got1)), threading.Thread(target=drain, args=(g2, got2))
    t1.start(); t2.start(); t1.join(); t2.join()
    assert not errors, errors
    # (a stream ends early when its row emits EOS, app.py:119 -- the two prompts give streams of different lengths)
    assert all((a == b).all() for a, b in zip(got1, lone1)) and 1 <= len(got1) == len(lone1) <= n_new
    assert all((a == b).all() for a, b in zip(got2, lone2)) and 1 <= len(got2) == len(lone2) <= n_new
    rt = model._rt()
    idle = rt.gen_pool[(B, P + n_new, 1.0, 0.98, 1)]
    assert len(idle) == 2 and idle[0] is not idle[1]
