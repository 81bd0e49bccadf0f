"""GPU tests (`pytest -m gpu`) of the per-request queue (`generate_many_requests`: per-request settings, grammar options
and seeds): the per-row sampler and keyed uniforms against their scalar counterparts, the ROWS persistent kernel row by row
against the batch-1 kernel, isolation of rows that are not live, and a trained model's requests against generating each
alone (the oracle, `generate`, `generate_stream`) at any batch size and order."""
import os

import numpy as np
import pytest
import torch

import gpu_checks as GC
import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF, _same
from midi_b200 import lib
from oracle import midi_oracle as O
from test_gpu_generate_many import _mode, _offsets, _restore, _snapshot, _tiny, _vs_oracle

pytestmark = pytest.mark.gpu

SAMPLER_BOUNDS = [("s_rows_vs_scalar_mismatch", 0.0), ("u_rows_vs_batch1_mismatch", 0.0)]
KERNEL_BOUNDS = [
    ("r_events_vs_batch1_mismatch", 0.0), ("r_kv_vs_batch1_mismatch", 0.0), ("r_row_last_error", 0.0),
    ("r_pos_error", 0.0), ("r_isolation_live_mismatch", 0.0), ("min:r_sampled_rows_checked", 20.0),
]
MODEL_BOUNDS = [
    ("gen_loss_last", 1.5), ("gen_persist_greedy_vs_oracle_mismatch", 0.0), ("gen_graph_greedy_vs_oracle_mismatch", 0.0),
    ("gen_nograph_greedy_vs_oracle_mismatch", 0.0), ("gen_persist_vs_generate_mismatch", 0.0),
    ("gen_persist_vs_generate_stream_mismatch", 0.0), ("gen_batch_size_order_mismatch", 0.0),
    ("gen_grammar_option_violations", 0.0), ("gen_repeat_mismatch", 0.0), ("min:gen_sampled_events_compared", 50.0),
]
MODEL_INFO = ("gen_graph_vs_persist_agree",)

TEMPS, TOP_PS, TOP_KS = (0.7, 1.0, 1.3), (0.5, 0.98, 1.0), (1, 20, 64, 200)


def _f32(v):
    return torch.tensor(v, dtype=torch.float32, device=DEV)


def _i32(v):
    return torch.tensor(v, dtype=torch.int32, device=DEV)


def test_sampler_and_uniforms_per_row():
    m = {"s_rows_vs_scalar_mismatch": 0.0, "u_rows_vs_batch1_mismatch": 0.0}
    model = _tiny()
    rt = model._rt()
    from midi_b200 import decode
    g = decode.GrammarLUT(model.tokenizer, DEV)
    V, pitch = rt.V, rt.pitch
    gen = torch.Generator(device=DEV).manual_seed(5)
    combos = [(t, p, k) for t in TEMPS for p in TOP_PS for k in TOP_KS]
    for B in (1, 5, 16):
        for step in range(8):
            for c0 in range(0, len(combos), B):
                sel = [combos[(c0 + r) % len(combos)] for r in range(B)]
                logits = (torch.randn((B, pitch), generator=gen, device=DEV) * 3).to(BF)
                ev = torch.randint(g.eos, g.eos + 1 + g.n_event_types, (B,), generator=gen, device=DEV)
                u = torch.rand(B, generator=gen, device=DEV)
                for masked in (False, True):
                    mask = (torch.rand((B, V), generator=gen, device=DEV) > 0.3).to(torch.uint8) if masked else None
                    out = torch.full((B,), -7, dtype=torch.long, device=DEV)
                    # held until the launch is issued: a freed temporary's memory would be reused by the next one
                    temp, top_p, top_k = _f32([s[0] for s in sel]), _f32([s[1] for s in sel]), _i32([s[2] for s in sel])
                    lib.call("b200_sample_from_logits_rows", logits.data_ptr(), B, V, pitch, temp.data_ptr(), top_p.data_ptr(),
                             top_k.data_ptr(), step, ev.data_ptr(), g.lut.data_ptr(), g.n_event_types, g.eos, g.pad,
                             lib.ptr(mask), u.data_ptr(), out.data_ptr(), 1, lib.stream())
                    ref = torch.full((B,), -7, dtype=torch.long, device=DEV)
                    for r, (t, p, k) in enumerate(sel):
                        lib.call("b200_sample_from_logits", logits[r:].data_ptr(), 1, V, pitch, t, p, k, step, ev[r:].data_ptr(),
                                 g.lut.data_ptr(), g.n_event_types, g.eos, g.pad, lib.ptr(mask[r:] if masked else None),
                                 u[r:].data_ptr(), ref[r:].data_ptr(), 1, lib.stream())
                    m["s_rows_vs_scalar_mismatch"] += float((out != ref).sum())
    # keyed uniforms: row b's draw is b200_uniform_fill of a batch-1 loop seeded row_seed[b] at counter 8 j + t
    u = torch.empty(16, dtype=torch.float32, device=DEV)
    u1 = torch.empty(1, dtype=torch.float32, device=DEV)
    for B in (1, 5, 16):
        for pos in (0, 33, 65, 4095):
            offs = _offsets(B, pos)
            first = [max(0, pos + o - (7 * b) % 40) for b, o in enumerate(offs)]
            seeds = [int(x) for x in torch.randint(0, 2 ** 62, (B,), generator=torch.Generator().manual_seed(pos + B))]
            pos_d, off_d, first_d = _i32([pos]), _i32(offs), _i32(first)
            seed_d = torch.tensor(seeds, dtype=torch.int64, device=DEV)
            for t in range(8):
                lib.call("b200_uniform_fill_rows", u.data_ptr(), B, pos_d.data_ptr(), off_d.data_ptr(), first_d.data_ptr(),
                         seed_d.data_ptr(), t, lib.stream())
                for b in range(B):
                    j = pos + offs[b] - first[b]
                    state = torch.tensor([8 * j + t, seeds[b]], dtype=torch.int64, device=DEV)
                    lib.call("b200_uniform_fill", u1.data_ptr(), 1, 0, state.data_ptr(), lib.stream())
                    m["u_rows_vs_batch1_mismatch"] += float(u[b] != u1[0])
    P.assert_within(m, SAMPLER_BOUNDS)


def _set_rows(gg, B, pos, offs, seed):
    """Mixed per-row settings, seeds, row_first and mask rows for a snapshot; returns them."""
    rng = np.random.default_rng(seed)
    sel = [(TEMPS[b % 3], TOP_PS[(b // 3) % 3], (1, 20, 64)[b % 3 if b % 4 else 2]) for b in range(B)]
    seeds = [int(s) for s in rng.integers(0, 2 ** 62, B)]
    first = [max(0, pos + o - int(rng.integers(0, 30))) for o in offs]
    gg.alloc_rows()
    gg.row_temp.copy_(_f32([s[0] for s in sel]))
    gg.row_top_p.copy_(_f32([s[1] for s in sel]))
    gg.row_top_k.copy_(_i32([s[2] for s in sel]))
    gg.row_seed.copy_(torch.tensor(seeds, dtype=torch.int64))
    gg.row_first.copy_(_i32(first))
    gg.mask.fill_(1)
    gg.mask[:, gg.g.eos] = 0                                 # no row finishes within the test's events
    for b in range(B):
        if b % 2:
            deny = rng.choice(gg.V, 40, replace=False)
            gg.mask[b, torch.tensor(deny, device=DEV)] = 0
    return sel, seeds, first


def test_rows_kernel_equals_each_row_alone():
    """From a ragged snapshot, each live row of the ROWS kernel commits what the batch-1 kernel commits for it alone."""
    m = {"r_events_vs_batch1_mismatch": 0.0, "r_kv_vs_batch1_mismatch": 0.0, "r_row_last_error": 0.0, "r_pos_error": 0.0,
         "r_isolation_live_mismatch": 0.0}
    model = _tiny()
    max_len, n_ev = 4104, 3
    checked = 0
    key1, g1 = model._checkout_generator(1, max_len, 1.0, 0.98, 20, None)
    try:
        for B in (5, 16):
            key, gg = model._checkout_generator(B, max_len, 1.0, 1.0, 1, None, per_row=True)
            try:
                kv, kv1 = gg.kv1, g1.kv1
                nh, D, page, mp = kv.cfg.n_head, kv.cfg.head_dim, kv.page, kv.max_pages
                assert kv1.max_pages == mp
                for pos in (33, 65, 4095):
                    offs, state, snap = _snapshot(gg, B, pos, seed=pos + 7 * B)
                    sel, seeds, first = _set_rows(gg, B, pos, offs, seed=pos + B)
                    gg.lengths, gg.queue, gg.rows = None, True, True
                    mask0 = gg.mask.clone()
                    gg._events_queue(n_ev, exit_on_done=True)
                    torch.cuda.synchronize()
                    m["r_pos_error"] = max(m["r_pos_error"], abs(int(gg.pos) - pos - n_ev))
                    m["r_row_last_error"] = max(m["r_row_last_error"], float((gg.row_last != -1).sum()))
                    d1, _, _ = g1._persistent()
                    for b in range(B):
                        r = pos + offs[b]
                        for li in range(len(kv.k)):                     # row b's pages, alone
                            for pool1, snap_pool in ((kv1.k[li], snap[li]), (kv1.v[li], snap[len(kv.k) + li])):
                                pool1.copy_(snap_pool.view(B, mp, nh, page, D)[b].reshape(pool1.shape))
                        g1.pos.fill_(r)
                        g1.ev_in.copy_(snap[-5][b:b + 1])
                        g1.seq.copy_(snap[-3][b:b + 1])
                        g1.counter.copy_(torch.tensor([8 * (r - first[b]), seeds[b]], dtype=torch.int64))
                        g1.mask.copy_(mask0[b:b + 1])
                        d1.temp, d1.top_p, d1.top_k = sel[b]
                        g1.lengths, g1.queue, g1.rows = None, False, False
                        g1._events_persistent(n_ev)
                        torch.cuda.synchronize()
                        m["r_events_vs_batch1_mismatch"] += float(
                            (g1.seq[0, r + 1:r + 1 + n_ev] != gg.seq[b, r + 1:r + 1 + n_ev]).sum())
                        m["r_pos_error"] = max(m["r_pos_error"], abs(int(g1.pos) - r - n_ev))
                        for li in range(len(kv.k)):
                            for pool, pool1 in ((kv.k[li], kv1.k[li]), (kv.v[li], kv1.v[li])):
                                a = pool.view(B, mp, nh, page, D)[b].permute(0, 2, 1, 3).reshape(mp * page, nh, D)[r:r + n_ev]
                                c = pool1.view(mp, nh, page, D).permute(0, 2, 1, 3).reshape(mp * page, nh, D)[r:r + n_ev]
                                m["r_kv_vs_batch1_mismatch"] += float((~_same(a, c)).sum())
                        checked += sel[b][2] > 1
                    # isolation: NaN pages, garbage ev_in and invalid settings in rows that are not live change no live row
                    dead = [b for b in range(B) if b % 3 == 1]
                    alive = [b for b in range(B) if b % 3 != 1]
                    last0 = _i32([(-2 if b % 2 else pos + offs[b]) if b in dead else -1 for b in range(B)])
                    runs = []
                    for poison in (False, True):
                        _restore(state, snap)
                        _set_rows(gg, B, pos, offs, seed=pos + B)
                        gg.row_last.copy_(last0)
                        if poison:
                            for pool in kv.k + kv.v:
                                pool.view(B, mp, nh, page, D)[dead] = float("nan")
                            gg.ev_in[dead] = torch.tensor([10 ** 6, -3, 7, 2 ** 40, -1, 0, 5, 3], device=DEV)
                            gg.row_temp[dead] = 0.0
                            gg.row_top_k[dead] = 0
                            gg.row_first[dead] = 10 ** 6
                        gg._events_queue(n_ev, exit_on_done=False)
                        torch.cuda.synchronize()
                        runs.append([t.clone() for t in state])
                    n_l = len(kv.k) * 2
                    bad = sum(float((~_same(c.view(B, mp, nh, page, D)[alive], d.view(B, mp, nh, page, D)[alive])).sum())
                              for c, d in zip(runs[0][:n_l], runs[1][:n_l]))
                    bad += sum(float((c[alive] != d[alive]).sum()) for c, d in zip(runs[0][n_l + 1:n_l + 2] + runs[0][n_l + 3:],
                                                                                runs[1][n_l + 1:n_l + 2] + runs[1][n_l + 3:]))
                    bad += float((runs[0][n_l] != runs[1][n_l]).sum())
                    m["r_isolation_live_mismatch"] += bad
            finally:
                gg.lengths, gg.queue, gg.rows = None, False, False
                gg.set_deny(())
                model._return_generator(key, gg)
    finally:
        model._return_generator(key1, g1)
    m["r_sampled_rows_checked"] = float(checked)
    P.assert_within(m, KERNEL_BOUNDS)


def test_generate_many_rows_of_a_trained_model():
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
    budgets = [24, 4, 17, 8, 24, 5, 12, 20, 4, 10]
    prompts = [songs[i, :L] for i, L in enumerate(lengths)]
    N = len(prompts)
    greedy = [i for i in range(N) if i % 3 == 0]
    top_k = [1 if i in greedy else 64 for i in range(N)]
    temp = [1.0 if i in greedy else 1.3 for i in range(N)]      # greedy: argmax of the unscaled logits, as the oracle's
    top_p = [0.98 if i in greedy else 0.9 for i in range(N)]
    patch = [i % 3 == 1 for i in range(N)]
    chans = [[0, 1] if i in (2, 4) else None for i in range(N)]              # never on a greedy request
    seeds = [int(torch.randint(0, 2 ** 62, (1,), generator=torch.Generator().manual_seed(1000 + i))) for i in range(N)]

    def many(order, bs, mode="persist"):
        k = dict(temp=[temp[i] for i in order], top_p=[top_p[i] for i in order], top_k=[top_k[i] for i in order],
                 disable_patch_change=[patch[i] for i in order], disable_channels=[chans[i] for i in order],
                 seeds=[seeds[i] for i in order])
        got = _mode(mode, lambda: model.generate_many_requests([prompts[i] for i in order],
                                                               [budgets[i] for i in order], batch_size=bs, **k))
        out = [None] * N
        for pos_, i in enumerate(order):
            out[i] = got[pos_]
        return out

    ident = list(range(N))
    runs = {mode: many(ident, 4, mode) for mode in ("persist", "graph", "nograph")}
    for mode, got in runs.items():
        m[f"gen_{mode}_greedy_vs_oracle_mismatch"] = _vs_oracle(model, sd16, ocfg, [prompts[i] for i in greedy],
                                                                [budgets[i] for i in greedy], [got[i] for i in greedy])
    got = runs["persist"]
    bad_gen = bad_stream = compared = 0.0
    for i in range(N):
        def solo():
            return model.generate(prompt=prompts[i], batch_size=1, max_len=lengths[i] + budgets[i], temp=temp[i], top_p=top_p[i],
                                  top_k=top_k[i], generator=torch.Generator().manual_seed(1000 + i))[0]
        new = got[i][lengths[i]:]
        if not patch[i] and chans[i] is None:
            ref = _mode("persist", solo)
            bad_gen += float((ref != got[i]).sum()) if ref.shape == got[i].shape else 1e9
        else:
            evs = _mode("persist", lambda: list(model.generate_stream(
                prompt=prompts[i], batch_size=1, max_len=lengths[i] + budgets[i], temp=temp[i], top_p=top_p[i], top_k=top_k[i],
                disable_patch_change=patch[i], disable_channels=chans[i], generator=torch.Generator().manual_seed(1000 + i))))
            ref = np.stack([e[0] for e in evs]) if evs else np.zeros((0, 8), dtype=np.int64)
            n = min(len(ref), len(new))
            bad_stream += float((ref[:n] != new[:n]).sum()) + (0 if n > 0 else 1e9)
        if i not in greedy:
            compared += len(new)
    m["gen_persist_vs_generate_mismatch"] = bad_gen
    m["gen_persist_vs_generate_stream_mismatch"] = bad_stream
    m["gen_sampled_events_compared"] = compared
    bad = 0.0
    perm = [7, 2, 9, 0, 5, 3, 8, 1, 6, 4]
    for order, bs in [(ident, 1), (ident, 3), (ident, 8), (ident, 16), (perm, 4)]:
        other = many(order, bs)
        bad += sum(float((a != b).sum()) if a.shape == b.shape else 1e9 for a, b in zip(other, got))
    m["gen_batch_size_order_mismatch"] = bad
    viol = 0
    for i in range(N):
        deny = set(model._deny_ids(patch[i], False, chans[i]))
        viol += sum(1 for row in got[i][lengths[i]:] if deny & set(row.tolist()))
    m["gen_grammar_option_violations"] = float(viol)
    again = many(ident, 4)
    m["gen_repeat_mismatch"] = sum(float((a != b).sum()) if a.shape == b.shape else 1e9 for a, b in zip(again, got))
    same = [float((a == b).mean()) for a, b in zip(runs["persist"], runs["graph"]) if a.shape == b.shape]
    m["gen_graph_vs_persist_agree"] = sum(same) / N
    P.assert_within(m, MODEL_BOUNDS, MODEL_INFO)
