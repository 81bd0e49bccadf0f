"""GPU tests (`pytest -m gpu`) of ragged generation (`generate_ragged`, `generate_stream_ragged`): the `_ragged` kernel entries against
their counterparts run on one row alone at that row's position, the ragged persistent kernel against the ragged
launch-per-phase loop, and greedy / sampled generation of a trained model against the oracle's solo generation."""
import math
import os

import numpy as np
import pytest
import torch

import gpu_checks as GC
import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF, _paged_pools, _same, randn
from midi_b200 import lib, ops
from oracle import midi_oracle as O

pytestmark = pytest.mark.gpu

# every ragged entry is bit-identical to its counterpart on the row alone; nothing else is written
KERNEL_BOUNDS = [
    ("rg_rope_vs_solo_mismatch", 0.0), ("rg_append_vs_solo_mismatch", 0.0), ("rg_attn_vs_solo_mismatch", 0.0),
    ("rg_fused_vs_solo_mismatch", 0.0), ("rg_commit_mismatch", 0.0), ("rg_zero_off_vs_batch_mismatch", 0.0),
    ("rg_attn_nan_out", 0.0), ("rg_pool_other_slots_changed", 0.0), ("min:rg_empty_splits_run", 1.0),
]
# layer 0 bit-identical; deeper layers within the bound of the rectangular check (persist_vs_phase: 5e-2 per row)
PERSIST_BOUNDS = [
    ("pr_l0_kv_persist_vs_phase_mismatch", 0.0), ("pr_other_slots_changed", 0.0), ("pr_counter_advance_error", 0.0),
    ("pr_pos_advance_error", 0.0), ("pr_seq_commit_mismatch", 0.0), ("pr_persist_k_row", 5e-2), ("pr_persist_v_row", 5e-2),
    ("pr_phase_k_row", 5e-2), ("pr_phase_v_row", 5e-2), ("min:pr_rows_with_empty_chunks", 1.0),
]
MODEL_BOUNDS = [
    ("gen_greedy_vs_oracle_solo_mismatch", 0.0), ("gen_loops_mismatch", 0.0), ("gen_b24_vs_oracle_solo_mismatch", 0.0),
    ("gen_b24_loops_mismatch", 0.0), ("gen_full_lengths_vs_rect_mismatch", 0.0), ("gen_garbage_mismatch", 0.0),
    ("gen_stream_vs_generate_mismatch", 0.0), ("gen_sampled_graph_vs_nograph_mismatch", 0.0),
    ("min:gen_sampled_persist_vs_graph_agree", 0.95), ("gen_sampled_invalid_events", 0.0),
    ("gen_layout_errors", 0.0), ("gen_loss_last", 1.5),
]


def _offsets(B, pos):
    """0, -1, -31, -32, -33 and the largest spread (a row at position 0), clipped to positions >= 0."""
    cyc = [0, -1, -31, -32, -33, -pos]
    return torch.tensor([max(cyc[b % len(cyc)], -pos) for b in range(B)], dtype=torch.int32, device=DEV)


def test_ragged_kernels_match_their_counterparts_row_by_row():
    m = {}

    def add(name, v):
        m[name] = max(m.get(name, 0.0), float(v))

    nh, D, page, cap = 16, 64, 64, 4096
    H = nh * D
    scale = 1.0 / math.sqrt(D)
    inv = O.default_inv_freq(D).to(BF).to(DEV)
    cos, sin = ops.rope_table(inv, cap + 8)
    empty = 0
    for B in (1, 5, 16, 24):
        for pos in (33, 64, 65, 1000, 4095):
            off = _offsets(B, pos)
            offs = off.tolist()
            pdev = torch.tensor([pos], dtype=torch.int32, device=DEV)
            kp, vp, bt, mp = _paged_pools(nh, D, page, B, cap, seed=pos + B)
            # each row's history: positions 0 .. its own position - 1 (later slots stay NaN)
            for b in range(B):
                n = pos + offs[b]
                if n:
                    hist = randn(n, 3 * H, seed=1000 * b + pos)
                    lib.call("b200_kv_append", hist.data_ptr(), kp.data_ptr(), vp.data_ptr(), bt[b].data_ptr(), mp, page, nh,
                             D, 1, n, 0, None, hist.stride(0), lib.stream())
            k0, v0 = kp.clone(), vp.clone()
            vals = randn(B, 3 * H, seed=pos * 7 + B)
            qkv = P.poisoned(vals, B + 1, 3 * H + 8)

            # ---- b200_rope_qk_ragged (S = 1 and S = 3)
            for S in (1, 3):
                rows = randn(B * S, 3 * H, seed=pos + S)
                got = rows.clone()
                ops.rope_qk_ragged_(got, cos, sin, S, H, D, off, pos0=0, pos0_dev=pdev)
                ref = rows.clone()
                for b in range(B):
                    ops.rope_qk_(ref[b * S:(b + 1) * S], cos, sin, S, H, D, pos0=pos + offs[b])
                add("rg_rope_vs_solo_mismatch", (~_same(got, ref)).sum())

            # ---- b200_kv_append_ragged (one new row per batch row)
            ka, va = k0.clone(), v0.clone()
            lib.call("b200_kv_append_ragged", qkv.data_ptr(), ka.data_ptr(), va.data_ptr(), bt.data_ptr(), mp, page, nh, D, B,
                     1, 0, pdev.data_ptr(), qkv.stride(0), off.data_ptr(), lib.stream())
            ks, vs = k0.clone(), v0.clone()
            for b in range(B):
                lib.call("b200_kv_append", qkv[b].data_ptr(), ks.data_ptr(), vs.data_ptr(), bt[b].data_ptr(), mp, page, nh, D,
                         1, 1, pos + offs[b], None, qkv.stride(0), lib.stream())
            add("rg_append_vs_solo_mismatch", (~_same(ka, ks)).sum() + (~_same(va, vs)).sum())
            slot = torch.zeros(ka.shape[0], page, dtype=torch.bool, device=DEV)
            for b in range(B):
                p_ = pos + offs[b]
                slot[int(bt[b, p_ // page]), p_ % page] = True
            other = ~slot[:, None, :, None].expand_as(ka)
            add("rg_pool_other_slots_changed", ((~_same(ka, k0)) & other).sum() + ((~_same(va, v0)) & other).sum())

            # ---- b200_attn_decode_ragged over the appended pools (query = the q third, any values)
            for n_split in (4, 16):
                nbytes = lib.query("b200_attn_decode_workspace_bytes", B, nh, D, n_split)
                ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
                o = P.nan_buffer((B + 1, H + 8), device=DEV)
                lib.call("b200_attn_decode_ragged", qkv.data_ptr(), ka.data_ptr(), va.data_ptr(), bt.data_ptr(), mp, page,
                         o.data_ptr(), B, 1, nh, D, 0, pdev.data_ptr(), cap, qkv.stride(0), o.stride(0), scale, n_split,
                         ws.data_ptr(), nbytes, off.data_ptr(), lib.stream())
                o_s = P.nan_buffer((B + 1, H + 8), device=DEV)
                for b in range(B):
                    ws1 = torch.full((nbytes // 4,), float("nan"), device=DEV)
                    lib.call("b200_attn_decode", qkv[b].data_ptr(), ka.data_ptr(), va.data_ptr(), bt[b].data_ptr(), mp, page,
                             o_s[b].data_ptr(), 1, 1, nh, D, pos + offs[b], None, cap, qkv.stride(0), o_s.stride(0), scale,
                             n_split, ws1.data_ptr(), nbytes, lib.stream())
                    Tb = pos + offs[b] + 1
                    empty += sum(1 for s in range(n_split) if s * ((Tb + n_split - 1) // n_split) >= Tb)
                add("rg_attn_vs_solo_mismatch", (~_same(o, o_s)).sum())
                add("rg_attn_nan_out", torch.isnan(o[:B, :H].float()).sum())

                # ---- b200_attn_decode_fused_ragged: RoPE + append + attention at each row's own position
                kf, vf = k0.clone(), v0.clone()
                of = P.nan_buffer((B + 1, H + 8), device=DEV)
                lib.call("b200_attn_decode_fused_ragged", qkv.data_ptr(), kf.data_ptr(), vf.data_ptr(), bt.data_ptr(), mp,
                         page, cos.data_ptr(), sin.data_ptr(), of.data_ptr(), B, nh, D, 0, pdev.data_ptr(), cap,
                         qkv.stride(0), of.stride(0), scale, n_split, ws.data_ptr(), nbytes, off.data_ptr(), lib.stream())
                kq, vq = k0.clone(), v0.clone()
                oq = P.nan_buffer((B + 1, H + 8), device=DEV)
                for b in range(B):
                    ws1 = torch.full((nbytes // 4,), float("nan"), device=DEV)
                    lib.call("b200_attn_decode_fused", qkv[b].data_ptr(), kq.data_ptr(), vq.data_ptr(), bt[b].data_ptr(), mp,
                             page, cos.data_ptr(), sin.data_ptr(), oq[b].data_ptr(), 1, nh, D, pos + offs[b], None, cap,
                             qkv.stride(0), oq.stride(0), scale, n_split, ws1.data_ptr(), nbytes, lib.stream())
                add("rg_fused_vs_solo_mismatch", (~_same(of, oq)).sum() + (~_same(kf, kq)).sum() + (~_same(vf, vq)).sum())
                add("rg_pool_other_slots_changed", ((~_same(kf, k0)) & other).sum() + ((~_same(vf, v0)) & other).sum())

                # ---- all offsets 0: the ragged entries are their counterparts on the whole batch
                z = torch.zeros(B, dtype=torch.int32, device=DEV)
                outs = []
                for name in ("b200_attn_decode_fused_ragged", "b200_attn_decode_fused"):
                    k_, v_ = k0.clone(), v0.clone()
                    o_ = P.nan_buffer((B + 1, H + 8), device=DEV)
                    extra = (z.data_ptr(),) if name.endswith("ragged") else ()
                    p0 = min(offs) + pos            # a position every row's history reaches
                    lib.call(name, qkv.data_ptr(), k_.data_ptr(), v_.data_ptr(), bt.data_ptr(), mp, page, cos.data_ptr(),
                             sin.data_ptr(), o_.data_ptr(), B, nh, D, p0, None, cap, qkv.stride(0), o_.stride(0), scale, n_split,
                             ws.data_ptr(), nbytes, *extra, lib.stream())
                    outs.append((o_, k_, v_))
                add("rg_zero_off_vs_batch_mismatch", sum(float((~_same(a, b_)).sum()) for a, b_ in zip(*outs)))

            # ---- b200_event_commit_ragged
            T, max_len = 8, cap + 1
            ev_t = torch.randint(0, 3000, (T, B), dtype=torch.int64, device=DEV)
            seq = torch.full((B, max_len, T), -1, dtype=torch.int64, device=DEV)
            nxt = torch.zeros(B, T, dtype=torch.int64, device=DEV)
            pc = pdev.clone()
            lib.call("b200_event_commit_ragged", ev_t.data_ptr(), seq.data_ptr(), nxt.data_ptr(), pc.data_ptr(), B, T, max_len,
                     off.data_ptr(), lib.stream())
            exp = torch.full_like(seq, -1)
            for b in range(B):
                exp[b, pos + offs[b] + 1] = ev_t[:, b]
            add("rg_commit_mismatch", (seq != exp).sum() + (nxt != ev_t.t()).sum() + abs(int(pc) - pos - 1))
    torch.cuda.synchronize()
    m["rg_empty_splits_run"] = float(empty)
    P.assert_within(m, KERNEL_BOUNDS)


def test_ragged_persistent_kernel_matches_the_phase_loop():
    """One event of b200_decode_events_ragged against one event of the ragged launch-per-phase loop from the same ragged
    snapshot (check_persist_vs_phase's protocol, per row at its own position)."""
    m = {}

    def add(name, v):
        m[name] = max(m.get(name, 0.0), float(v))

    cfg = GM.config()
    cfg.net_config.num_hidden_layers = 2
    model = GM.cpu_model(cfg).to(DEV, dtype=BF).eval()
    V = model.tokenizer.vocab_size
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    max_len = 4097
    rows_empty = 0
    for B in (5, 16):
        key, gg = model._checkout_generator(B, max_len, 1.0, 0.98, 20, None)
        try:
            assert gg.persistent_ok()
            eng, kv = gg.outer.eng, gg.kv1
            nh, D, page = eng.cfg.n_head, eng.cfg.head_dim, kv.page
            for pos in (33, 65, 4095):
                offs = _offsets(B, pos).tolist()
                lengths = [pos + 1 + o for o in offs]
                target = min(160, max(1, sms * 16 // (B * nh)))          # decode_persist.cu chunk grid on pos + 1
                chunk = ((pos + 1 + target - 1) // target + 31) // 32 * 32
                n_chunks = (pos + 1 + chunk - 1) // chunk
                rows_empty += sum(1 for L in lengths if (L + chunk - 1) // chunk < n_chunks)
                g = torch.Generator(device=DEV).manual_seed(pos + B)
                prompt = torch.randint(0, V, (B, pos + 1, 8), generator=g, device=DEV)
                gg._set_lengths(prompt, lengths)
                gg._set_state(prompt)
                own = torch.arange(kv.max_pages * page, device=DEV)[None, :] >= torch.tensor([L - 1 for L in lengths],
                                                                                           device=DEV)[:, None]
                past = own.view(B, kv.max_pages, 1, page, 1)
                for pool in kv.k + kv.v:
                    pool.view(B, kv.max_pages, nh, page, D).masked_fill_(past, float("nan"))
                state = kv.k + kv.v + [gg.pos, gg.ev_in, gg.counter, gg.seq]
                snap = [t.clone() for t in state]
                slot = torch.zeros(B, kv.max_pages * page, dtype=torch.bool, device=DEV)
                for b, L in enumerate(lengths):
                    slot[b, L - 1] = True
                slot = slot.view(B, kv.max_pages, 1, page, 1).expand(B, kv.max_pages, nh, page, D).reshape(kv.k[0].shape)
                runs = {}
                for name in ("persist", "phase"):
                    for t, s in zip(state, snap):
                        t.copy_(s)
                    if name == "persist":
                        gg._events_persistent(1)
                    else:
                        gg._event()
                    torch.cuda.synchronize()
                    pools = kv.k + kv.v
                    add("pr_other_slots_changed", sum(float((~_same(p_, s_) & ~slot).sum()) for p_, s_ in zip(pools, snap)))
                    add("pr_counter_advance_error", abs(int(gg.counter[0]) - int(snap[-2][0]) - 8))
                    add("pr_pos_advance_error", abs(int(gg.pos) - pos - 1))
                    ev = gg.ev_in.clone()
                    add("pr_seq_commit_mismatch", sum(float((gg.seq[b, L] != ev[b]).sum()) for b, L in enumerate(lengths)))
                    runs[name] = [torch.stack([p_.view(B, kv.max_pages, nh, page, D)[b, (L - 1) // page, :, (L - 1) % page]
                                               for b, L in enumerate(lengths)]) for p_ in pools]
                Ln = len(eng.layers)
                add("pr_l0_kv_persist_vs_phase_mismatch", sum(float((runs["persist"][i] != runs["phase"][i]).sum())
                                                              for i in (0, Ln)))
                e = ops.embed_sum(snap[-3], eng.embed)
                for b, L in enumerate(lengths):
                    ref = GC._event_step64(eng, e[b:b + 1], snap[:Ln], snap[Ln:2 * Ln], kv.block_table[b:b + 1], page, L - 1,
                                           gg.outer.cos, gg.outer.sin)
                    for li in range(Ln):
                        atol = 1e-3 * float(ref[li][1].norm(dim=-1).median())
                        for n_ in runs:
                            add(f"pr_{n_}_k_row", P.row_worst(runs[n_][li][b:b + 1], ref[li][0], atol=atol))
                            add(f"pr_{n_}_v_row", P.row_worst(runs[n_][Ln + li][b:b + 1], ref[li][1], atol=atol))
        finally:
            gg.lengths = None
            model._return_generator(key, gg)
    m["pr_rows_with_empty_chunks"] = float(rows_empty)
    P.assert_within(m, PERSIST_BOUNDS)


def _loops(model, **kw):
    """The same generate_ragged call on the persistent kernel, the CUDA-graph loop and the host-issued loop."""
    out = {}
    for mode in ("persist", "graph", "nograph"):
        os.environ["B200_GENERATE"] = mode
        try:
            out[mode] = model.generate_ragged(**kw)
        finally:
            os.environ.pop("B200_GENERATE")
    return out


def _mismatch(a, b):
    return float((a != b).sum()) if a.shape == b.shape else 1e9


def _vs_oracle_solo(model, sd16, ocfg, prompt, lengths, n_new, ids):
    """Tokens by which row b differs from the oracle's greedy generation of prompt b[:L_b] alone."""
    tok = model.tokenizer
    bad, layout = 0.0, 0.0
    P_ = max(lengths)
    n_done = ids.shape[1] - P_
    for b, L in enumerate(lengths):
        ref = O.generate(sd16, ocfg, tok, prompt[b:b + 1, :L], batch_size=1, max_len=L + n_new, top_k=1,
                         inv_freq_net=model.net.rotary_emb.inv_freq, inv_freq_tok=model.net_token.rotary_emb.inv_freq)[0]
        k = ref.shape[0] - L
        bad += _mismatch(ids[b, :L + min(k, n_done)], ref[:L + min(k, n_done)])
        if not (k == n_done or (k < n_done and ref[-1, 0] == tok.eos_id)):
            bad += abs(k - n_done)
        layout += float((ids[b, L + n_done:] != tok.pad_id).sum())
    return bad, layout


def test_ragged_generate_of_a_trained_model():
    m = {}
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    tok = model.tokenizer
    for step in range(1, 241):                              # check_model_peaked_greedy's training
        batch = GC._song_batch(tok, 16, 66, seed=step).to(DEV)
        loss = model.training_loss(batch)
        model.fused_optimizer_step(lr=3e-4 * min(1.0, step / 20), step=step, weight_decay=0.01)
    m["gen_loss_last"] = float(loss)
    model.eval()
    sd16 = GC._sd(model, BF)
    n_new = 24
    lengths = [9, 3, 14, 6]
    prompt = GC._song_batch(tok, 4, 14, seed=999).numpy()
    kw = dict(prompt=prompt, batch_size=4, max_len=14 + n_new, top_k=1)
    ids = _loops(model, **kw, lengths=lengths)
    m["gen_loops_mismatch"] = max(_mismatch(ids["persist"], ids["graph"]), _mismatch(ids["persist"], ids["nograph"]))
    m["gen_greedy_vs_oracle_solo_mismatch"], m["gen_layout_errors"] = _vs_oracle_solo(model, sd16, ocfg, prompt, lengths,
                                                                                     n_new, ids["persist"])
    # B = 24: the unfused graph path (the persistent kernel and the fused attention take B <= 16)
    p24 = GC._song_batch(tok, 24, 14, seed=998).numpy()
    l24 = [3 + (5 * b) % 12 for b in range(24)]
    l24[7] = 14
    ids24 = _loops(model, prompt=p24, batch_size=24, max_len=14 + 12, top_k=1, lengths=l24)
    m["gen_b24_loops_mismatch"] = max(_mismatch(ids24["persist"], ids24["graph"]), _mismatch(ids24["graph"], ids24["nograph"]))
    m["gen_b24_vs_oracle_solo_mismatch"], lay = _vs_oracle_solo(model, sd16, ocfg, p24, l24, 12, ids24["graph"])
    m["gen_layout_errors"] += lay
    # full lengths = the rectangular call; garbage past the lengths is never read
    m["gen_full_lengths_vs_rect_mismatch"] = _mismatch(model.generate_ragged(**kw, lengths=[14] * 4), model.generate(**kw))
    junk = prompt.copy()
    rng = np.random.default_rng(1)
    for b, L in enumerate(lengths):
        junk[b, L:] = rng.integers(-5, 10 ** 6, size=junk[b, L:].shape)
    m["gen_garbage_mismatch"] = _mismatch(model.generate_ragged(**{**kw, "prompt": junk}, lengths=lengths), ids["persist"])
    # generate_stream_ragged yields row b's events L_b, L_b + 1, ...
    evs = list(model.generate_stream_ragged(**kw, lengths=lengths))
    n_done = ids["persist"].shape[1] - 14
    bad = abs(len(evs) - n_done)
    for b, L in enumerate(lengths):
        got = np.stack([e[b] for e in evs[:n_done]])
        bad += _mismatch(got, ids["persist"][b, L:L + len(got)])
    m["gen_stream_vs_generate_mismatch"] = float(bad)
    # sampled: the same draws on every loop, grammar-valid events
    sk = dict(prompt=prompt, batch_size=4, max_len=14 + n_new, top_k=20, lengths=lengths)
    runs = {}
    for mode in ("persist", "graph", "nograph"):
        os.environ["B200_GENERATE"] = mode
        try:
            runs[mode] = model.generate_ragged(**sk, generator=torch.Generator(DEV).manual_seed(3))
        finally:
            os.environ.pop("B200_GENERATE")
    # the graph and host-issued loops run the same kernels; the persistent kernel cuts the attention into other chunks, so
    # a draw that lands within its rounding of a cumulative-probability boundary may differ
    m["gen_sampled_graph_vs_nograph_mismatch"] = _mismatch(runs["graph"], runs["nograph"])
    a, b_ = runs["persist"], runs["graph"]
    m["gen_sampled_persist_vs_graph_agree"] = float((a == b_).mean()) if a.shape == b_.shape else 0.0
    s_done = runs["persist"].shape[1] - 14
    invalid = 0
    for b, L in enumerate(lengths):
        for row in runs["persist"][b, L:L + s_done]:
            if int(row[0]) != tok.eos_id and tok.tokens2event(row.tolist()) == []:
                invalid += 1
    m["gen_sampled_invalid_events"] = float(invalid)
    P.assert_within(m, MODEL_BOUNDS)
