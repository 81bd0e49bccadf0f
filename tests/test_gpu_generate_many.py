"""GPU tests (`pytest -m gpu`) of the request queue (`generate_many`): the queue persistent kernel against the ragged one
when no row finishes, the per-row stop (row_last, the launch's exit, no commit past a row's end) on the persistent kernel
and on the phase loop event by event, isolation of rows that are not live, and greedy / sampled generation of a trained
model against the oracle's solo generation and against `generate`."""
import os

import numpy as np
import pytest
import torch

import gpu_checks as GC
import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF, _same
from oracle import midi_oracle as O

pytestmark = pytest.mark.gpu

KERNEL_BOUNDS = [
    ("q_vs_ragged_mismatch", 0.0), ("q_row_last_error", 0.0), ("q_exit_event_error", 0.0), ("q_seq_past_end_written", 0.0),
    ("q_seq_commit_missing", 0.0), ("q_eos_rows_not_eos", 0.0), ("q_persist_vs_phase_row_last", 0.0),
    ("q_persist_vs_phase_pos", 0.0), ("q_persist_vs_phase_commits", 0.0), ("q_l0_kv_persist_vs_phase_mismatch", 0.0),
    ("q_not_live_pages_changed", 0.0), ("q_isolation_live_mismatch", 0.0), ("q_isolation_not_live_seq_changed", 0.0),
    ("min:q_rows_finished_mid_launch", 1.0),
]
MODEL_BOUNDS = [
    ("gen_loss_last", 1.5), ("gen_persist_vs_oracle_solo_mismatch", 0.0), ("gen_graph_vs_oracle_solo_mismatch", 0.0),
    ("gen_nograph_vs_oracle_solo_mismatch", 0.0), ("gen_b24_graph_vs_oracle_solo_mismatch", 0.0),
    ("gen_one_request_vs_generate_mismatch", 0.0), ("gen_sampled_invalid_events", 0.0), ("gen_sampled_repeat_mismatch", 0.0),
]
MODEL_INFO = ("gen_sampled_persist_vs_graph_agree",)


def _offsets(B, pos):
    """0, -1, -31, -32, -33 and the largest spread (a row at position 0), clipped to positions >= 0."""
    cyc = [0, -1, -31, -32, -33, -pos]
    return [max(cyc[b % len(cyc)], -pos) for b in range(B)]


def _tiny():
    cfg = GM.config()
    cfg.net_config.num_hidden_layers = 2
    return GM.cpu_model(cfg).to(DEV, dtype=BF).eval()


def _snapshot(gg, B, pos, seed):
    """A ragged state at shared position pos (row b at pos + off[b]), switched to queue mode with every row live and no
    budget reached within the test's events; returns (offsets, the state tensors, their snapshot)."""
    V = gg.V
    offs = _offsets(B, pos)
    g = torch.Generator(device=DEV).manual_seed(seed)
    prompt = torch.randint(0, V, (B, pos + 1, 8), generator=g, device=DEV)
    gg._set_lengths(prompt, [pos + 1 + o for o in offs])
    gg._set_state(prompt)
    gg.row_end.fill_(gg.max_len - 1)
    gg.row_last.fill_(-1)
    state = gg.kv1.k + gg.kv1.v + [gg.pos, gg.ev_in, gg.counter, gg.seq, gg.row_end, gg.row_last]
    return offs, state, [t.clone() for t in state]


def _restore(state, snap):
    for t, s in zip(state, snap):
        t.copy_(s)


def _deny_event_types(gg, rows):
    """Rows in `rows` may only emit EOS at step 0; every other row may not emit it."""
    ev = list(range(gg.g.eos + 1, gg.g.eos + 1 + gg.g.n_event_types))
    gg.mask.fill_(1)
    for b in range(gg.B):
        if b in rows:
            gg.mask[b, ev] = 0
        else:
            gg.mask[b, gg.g.eos] = 0


def test_queue_kernel_rows_stop_on_their_own():
    m = {}

    def add(name, v):
        m[name] = max(m.get(name, 0.0), float(v))

    model = _tiny()
    max_len = 4104
    finished_mid = 0
    for B in (5, 16):
        key, gg = model._checkout_generator(B, max_len, 1.0, 0.98, 1, None)
        try:
            assert gg.persistent_ok()
            kv = gg.kv1
            nh, D, page, mp = kv.cfg.n_head, kv.cfg.head_dim, kv.page, kv.max_pages
            for pos in (33, 65, 4095):
                # ---- all rows live, no budget reached: the queue kernel is the ragged kernel
                _deny_event_types(gg, ())
                offs, state, snap = _snapshot(gg, B, pos, seed=pos + B)
                gg._events_persistent(4)
                ragged = [t.clone() for t in state]
                _restore(state, snap)
                gg.lengths, gg.queue = None, True
                gg._events_queue(4, exit_on_done=True)
                add("q_vs_ragged_mismatch", sum(float((~_same(a, b_)).sum()) for a, b_ in zip(state, ragged)))

                # ---- rows that finish: budgets of 1 .. 4 events, EOS-only rows, one row never finishing in the launch
                eos_rows = {b for b in range(B) if b % 5 == 2}
                k_fin = [1 if b in eos_rows else 1 + b % 4 for b in range(B)]
                k_fin[0] = 6 if 0 not in eos_rows else 1
                _deny_event_types(gg, eos_rows)
                offs, state, snap = _snapshot(gg, B, pos, seed=pos + 2 * B)
                gg.lengths, gg.queue = None, True
                ends = [pos + offs[b] + k_fin[b] for b in range(B)]
                gg.row_end.copy_(torch.tensor(ends, dtype=torch.int32))
                snap[-2].copy_(gg.row_end)
                for exit_on_done in (False, True):
                    _restore(state, snap)
                    gg._events_queue(8, exit_on_done=exit_on_done)
                    torch.cuda.synchronize()
                    n_run = min(k_fin) if exit_on_done else max(k_fin)
                    add("q_exit_event_error", abs(int(gg.pos) - pos - n_run))
                    last = gg.row_last.tolist()
                    for b in range(B):
                        r = pos + offs[b]
                        want = r + k_fin[b] if k_fin[b] <= n_run else -1
                        add("q_row_last_error", abs(last[b] - want))
                        n_commit = min(k_fin[b], n_run)
                        written = (gg.seq[b] != snap[-3][b]).any(-1)
                        add("q_seq_past_end_written", written[r + 1 + n_commit:].sum())
                        add("q_seq_commit_missing", (~written[r + 1:r + 1 + n_commit]).sum())
                        if b in eos_rows:
                            add("q_eos_rows_not_eos", int(gg.seq[b, r + 1, 0]) != gg.g.eos)
                        # a finished row appends nothing after its last event: its pages past it are unchanged
                        pg = torch.arange(mp * page, device=DEV) > r + n_commit - 1
                        for p_, s_ in zip(kv.k + kv.v, snap[:2 * len(kv.k)]):
                            pv, sv = p_.view(B, mp, nh, page, D)[b], s_.view(B, mp, nh, page, D)[b]
                            changed = (~_same(pv, sv)).any(-1).any(1).reshape(-1)        # [mp * page]
                            add("q_not_live_pages_changed", (changed & pg).sum())
                    finished_mid += sum(1 for k in k_fin if 1 < k < n_run)

                # ---- persistent kernel vs phase loop, event by event, from the persistent kernel's own states
                _restore(state, snap)
                L0 = len(gg.outer.eng.layers)
                for e in range(max(k_fin)):
                    s_e = [t.clone() for t in state]
                    live = [b for b in range(B) if int(gg.row_last[b]) == -1]
                    rec = {}
                    for name in ("phase", "persist"):
                        _restore(state, s_e)
                        if name == "persist":
                            gg._events_queue(1, exit_on_done=False)
                        else:
                            gg._event()
                        torch.cuda.synchronize()
                        p_now = int(s_e[-6])
                        rows = [torch.stack([pool.view(B, mp, nh, page, D)[b, (p_now + offs[b]) // page, :,
                                                                            (p_now + offs[b]) % page] for b in live])
                                for pool in (kv.k[0], kv.v[0])] if live else []
                        rec[name] = (gg.row_last.clone(), int(gg.pos), (gg.seq != s_e[-3]).any(-1), rows)
                    a, b_ = rec["persist"], rec["phase"]
                    add("q_persist_vs_phase_row_last", (a[0] != b_[0]).sum())
                    add("q_persist_vs_phase_pos", abs(a[1] - b_[1]))
                    add("q_persist_vs_phase_commits", (a[2] != b_[2]).sum())
                    add("q_l0_kv_persist_vs_phase_mismatch", sum(float((~_same(x, y)).sum()) for x, y in zip(a[3], b_[3])))

                # ---- isolation: NaN pages and garbage ev_in in rows that are not live change no live row
                _deny_event_types(gg, ())
                offs, state, snap = _snapshot(gg, B, pos, seed=pos + 3 * B)
                gg.lengths, gg.queue = None, True
                dead = [b for b in range(B) if b % 3 == 1]
                alive = [b for b in range(B) if b % 3 != 1]
                gg.row_last.copy_(torch.tensor([(-2 if b % 2 else pos + offs[b]) if b in dead else -1 for b in range(B)],
                                               dtype=torch.int32))
                snap[-1].copy_(gg.row_last)
                runs = []
                for poison in (False, True):
                    _restore(state, snap)
                    if poison:
                        for pool in kv.k + kv.v:
                            pool.view(B, mp, nh, page, D)[dead] = float("nan")
                        gg.ev_in[dead] = torch.tensor([10 ** 6, -3, 7, 2 ** 40, -1, 0, 5, 3], device=DEV)
                    gg._events_queue(3, exit_on_done=False)
                    torch.cuda.synchronize()
                    runs.append([t.clone() for t in state])
                clean, dirty = runs
                n_l = len(kv.k) * 2
                bad = sum(float((~_same(c.view(B, mp, nh, page, D)[alive], d.view(B, mp, nh, page, D)[alive])).sum())
                          for c, d in zip(clean[:n_l], dirty[:n_l]))
                pos_c, ev_c, ctr_c, seq_c, _, last_c = clean[n_l:]
                pos_d, ev_d, ctr_d, seq_d, _, last_d = dirty[n_l:]
                bad += float((seq_c[alive] != seq_d[alive]).sum()) + float((ev_c[alive] != ev_d[alive]).sum())
                bad += float((pos_c != pos_d).sum() + (ctr_c != ctr_d).sum() + (last_c != last_d).sum())
                add("q_isolation_live_mismatch", bad)
                add("q_isolation_not_live_seq_changed", (seq_d[dead] != snap[-3][dead]).sum())
        finally:
            gg.lengths, gg.queue = None, False
            gg.set_deny(())
            model._return_generator(key, gg)
    m["q_rows_finished_mid_launch"] = float(finished_mid)
    P.assert_within(m, KERNEL_BOUNDS)


def _mode(mode, fn):
    os.environ["B200_GENERATE"] = mode
    try:
        return fn()
    finally:
        os.environ.pop("B200_GENERATE")


def _vs_oracle(model, sd16, ocfg, prompts, budgets, got):
    bad = 0.0
    for p, n, g in zip(prompts, budgets, got):
        ref = O.generate(sd16, ocfg, model.tokenizer, p[None], batch_size=1, max_len=p.shape[0] + n, top_k=1,
                         inv_freq_net=model.net.rotary_emb.inv_freq, inv_freq_tok=model.net_token.rotary_emb.inv_freq)[0]
        bad += float((g != ref).sum()) if g.shape == ref.shape else 1e9
    return bad


def test_generate_many_of_a_trained_model():
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
    songs = GC._song_batch(tok, 10, 14, seed=997).numpy()
    lengths = [1, 14, 3, 9, 6, 12, 2, 14, 5, 8]
    budgets = [24, 3, 17, 8, 24, 5, 12, 20, 3, 10]
    prompts = [songs[i, :L] for i, L in enumerate(lengths)]
    for mode in ("persist", "graph", "nograph"):
        got = _mode(mode, lambda: model.generate_many(prompts, budgets, batch_size=4, top_k=1))
        m[f"gen_{mode}_vs_oracle_solo_mismatch"] = _vs_oracle(model, sd16, ocfg, prompts, budgets, got)
    # B = 24 slots for 30 requests: the unfused graph path (the persistent kernel and the fused attention take B <= 16)
    p30 = [GC._song_batch(tok, 1, 14, seed=900 + i).numpy()[0, :1 + (5 * i) % 14] for i in range(30)]
    b30 = [3 + (7 * i) % 14 for i in range(30)]
    got = _mode("graph", lambda: model.generate_many(p30, b30, batch_size=24, top_k=1))
    m["gen_b24_graph_vs_oracle_solo_mismatch"] = _vs_oracle(model, sd16, ocfg, p30, b30, got)
    # one request in one slot is generate at batch 1, greedy and sampled, on each device-resident loop
    bad = 0.0
    for mode in ("persist", "graph"):
        for top_k in (1, 20):
            def both():
                a = model.generate_many([prompts[3]], 20, batch_size=1, top_k=top_k,
                                        generator=torch.Generator(DEV).manual_seed(4))[0]
                b_ = model.generate(prompt=prompts[3], batch_size=1, max_len=9 + 20, top_k=top_k,
                                    generator=torch.Generator(DEV).manual_seed(4))[0]
                return a, b_
            a, b_ = _mode(mode, both)
            bad += float((a != b_).sum()) if a.shape == b_.shape else 1e9
    m["gen_one_request_vs_generate_mismatch"] = bad
    # sampled: grammar-valid events, reproducible for the same seed; persist vs graph agreement recorded
    runs = {}
    for mode in ("persist", "graph"):
        runs[mode] = _mode(mode, lambda: model.generate_many(prompts, budgets, batch_size=4, top_k=20,
                                                             generator=torch.Generator(DEV).manual_seed(7)))
    again = _mode("persist", lambda: model.generate_many(prompts, budgets, batch_size=4, top_k=20,
                                                         generator=torch.Generator(DEV).manual_seed(7)))
    m["gen_sampled_repeat_mismatch"] = sum(float((a != b_).sum()) if a.shape == b_.shape else 1e9
                                           for a, b_ in zip(runs["persist"], again))
    invalid = 0
    for p, g in zip(prompts, runs["persist"]):
        for row in g[p.shape[0]:]:
            if int(row[0]) != tok.eos_id and tok.tokens2event(row.tolist()) == []:
                invalid += 1
    m["gen_sampled_invalid_events"] = float(invalid)
    same = [float((a == b_).mean()) for a, b_ in zip(runs["persist"], runs["graph"]) if a.shape == b_.shape]
    m["gen_sampled_persist_vs_graph_agree"] = sum(same) / len(prompts)
    P.assert_within(m, MODEL_BOUNDS, MODEL_INFO)
