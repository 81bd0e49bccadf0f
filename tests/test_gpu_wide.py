"""GPU tests (`pytest -m gpu`) of the persistent generate kernel's per-request mode at up to 32 slots and of the sampler's
fast path at top_k <= 128:
- the phase sampler at top_k 65 ... 128 against decode_reference.logits_sample, and against its general path;
- the `_queue_rows` kernel at 17 ... 32 rows (two row groups of at most 16) against the same rows run as launches of at
  most 16 rows, whose draws are held to the restated sampler, and one 3-event launch against three 1-event launches;
- generate_many_requests with 40 requests through 32 slots and a 32-slot GenerateServer against each request generated
  alone, on tv2o-medium."""
import threading
import time

import numpy as np
import pytest
import torch

import decode_reference as DR
import gpu_checks as GC
import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF, _same
from midi_b200 import lib
from test_gpu_generate_many import _mode
from test_gpu_serve import _Env

pytestmark = pytest.mark.gpu

WIDE_K = (65, 96, 127, 128, 20)              # the new fast-path range and a k <= 64 control


def _logit_rows(V, ld, Rn, seed):
    """Rn rows of bf16 logits: random, rows with exact ties at the top (so at the k-th value), and whole rows tied."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    lg = torch.full((Rn, ld), 30.0, device=DEV, dtype=BF)
    lg[:, :V] = (torch.randn(Rn, V, generator=g, device=DEV) * 2.5).to(BF)
    lg[8:16, :V] = lg[8:16, :V].float().clamp(max=1.0).to(BF)
    lg[16:20, :V] = 0.5
    return lg


def test_sampler_fast_path_up_to_top_k_128():
    from midi_b200 import decode as dec
    from midi_b200.tokenizer_tables import TokenizerTables
    tokz = TokenizerTables("v2")
    glut = dec.GrammarLUT(tokz, DEV)
    lut = glut.lut.cpu().numpy()
    V, ld, Rn = 3406, 3408, 40
    logits = _logit_rows(V, ld, Rn, seed=5)
    lg_np = logits[:, :V].float().cpu().numpy()
    ev_types = sorted(tokz.event_ids.values())
    ev = [ev_types[r % len(ev_types)] for r in range(Rn)]
    ev_d = torch.tensor(ev, dtype=torch.long, device=DEV)
    gm = torch.Generator(device=DEV).manual_seed(6)
    mask = (torch.rand(Rn, V, generator=gm, device=DEV) > 0.1).to(torch.uint8)
    mask[3] = 0
    mask_np = mask.cpu().numpy()
    small = torch.zeros(Rn, V, dtype=torch.uint8, device=DEV)          # <= 60 candidates: top_k >= 65 keeps them all
    for r in range(Rn):
        small[r, torch.randperm(V, generator=gm, device=DEV)[:60]] = 1
    small[16:20, :] = 0
    small[16:20, 100:160] = 1

    def rng(step, r):
        if step == 0:
            return glut.eos, glut.eos + 1 + glut.n_event_types
        e = ev[r] - (glut.eos + 1)
        lo, hi = (int(v) for v in lut[e, step - 1])
        return (lo, hi) if hi > lo else (glut.pad, glut.pad + 1)

    def rows_call(top_ks, temp, top_p, step, m, u):
        o = torch.full((Rn,), -7, dtype=torch.long, device=DEV)
        tk = torch.tensor(top_ks, dtype=torch.int32, device=DEV)
        tt = torch.full((Rn,), temp, device=DEV)
        tp = torch.full((Rn,), top_p, device=DEV)
        lib.call("b200_sample_from_logits_rows", logits.data_ptr(), Rn, V, ld, tt.data_ptr(), tp.data_ptr(), tk.data_ptr(),
                 step, ev_d.data_ptr(), glut.lut.data_ptr(), glut.n_event_types, glut.eos, glut.pad,
                 m.data_ptr() if m is not None else None, u.data_ptr(), o.data_ptr(), 1, lib.stream())
        return o

    m = {"sw_logits_mismatch": 0.0, "sw_fast_vs_general_mismatch": 0.0}
    n = amb = wide = per_k = 0
    widest = 0
    for step in range(8):
        for temp in (1.0, 0.7):
            for top_p in (0.5, 0.98, 1.0):
                for use_mask in (False, True):
                    u = DR.uniforms(Rn, seed=100 * step + 7)
                    ud = torch.from_numpy(u).to(DEV)
                    top_ks = [WIDE_K[(r + step) % len(WIDE_K)] for r in range(Rn)]
                    oc = rows_call(top_ks, temp, top_p, step, mask if use_mask else None, ud).cpu().numpy()
                    for r in range(Rn):
                        lo, hi = rng(step, r)
                        widest = max(widest, hi - lo)
                        want, a = DR.logits_sample(lg_np[r], temp, top_p, top_ks[r], lo, hi,
                                                   mask_np[r] if use_mask else None, float(u[r]))
                        n += 1
                        amb += int(a)
                        wide += int(top_ks[r] > 64 and not a)
                        m["sw_logits_mismatch"] += int((not a) and oc[r] != want)
                # fast path (every k of WIDE_K) against the general path (top_k 4096) on rows of <= 60 candidates
                u = DR.uniforms(Rn, seed=step + 31)
                ud = torch.from_numpy(u).to(DEV)
                sm = None if step in (0, 2) else small
                general = rows_call([4096] * Rn, temp, top_p, step, sm, ud)
                for k in WIDE_K[:4]:
                    fast = rows_call([k] * Rn, temp, top_p, step, sm, ud)
                    m["sw_fast_vs_general_mismatch"] += float((fast != general).sum())
                    per_k += Rn
    m["sw_ambiguous_frac"] = amb / n
    m["sw_unambiguous_wide_draws"] = float(wide)
    m["sw_fast_general_rows"] = float(per_k)
    m["sw_widest_range"] = float(widest)
    print(m)
    P.assert_within(m, [("sw_logits_mismatch", 0.0), ("sw_fast_vs_general_mismatch", 0.0), ("sw_ambiguous_frac", 0.25),
                        ("min:sw_unambiguous_wide_draws", 2000.0), ("min:sw_fast_general_rows", 1000.0),
                        ("min:sw_widest_range", 2048.0)])


WIDE_B = (17, 24, 31, 32)
WIDE_POS = (65, 700)
ROW_TOP_K = (1, 20, 65, 100, 128)


def _rows_settings(gg, B, pos, ctx, live, vi):
    temps = [GC.PT_ROW_TEMP[(b + vi) % 3] for b in range(B)]
    top_ps = [GC.PT_ROW_TOP_P[(b + pos) % 4] for b in range(B)]
    top_ks = [ROW_TOP_K[(b + vi) % len(ROW_TOP_K)] for b in range(B)]
    first = [max(0, ctx[b] - (3 * b + pos) % 11) for b in range(B)]
    seeds = [(1000003 * (b + 1) + 7919 * pos + vi) & ((1 << 62) - 1) for b in range(B)]
    row_end = [ctx[b] + 1 if b % 4 == 1 else GC.PT_MAX_LEN - 1 for b in range(B)]
    row_last = [-1 if live[b] else (-2 if b % 2 else ctx[b]) for b in range(B)]
    gg.row_temp.copy_(torch.tensor(temps))
    gg.row_top_p.copy_(torch.tensor(top_ps))
    gg.row_top_k.copy_(torch.tensor(top_ks, dtype=torch.int32))
    gg.row_seed.copy_(torch.tensor(seeds, dtype=torch.int64))
    gg.row_first.copy_(torch.tensor(first, dtype=torch.int32))
    gg.row_end.copy_(torch.tensor(row_end, dtype=torch.int32))
    gg.row_last.copy_(torch.tensor(row_last, dtype=torch.int32))
    return list(zip(temps, top_ps, top_ks)), first, seeds


def _copy_rows(src, dst, b0, n):
    """Rows b0 .. b0 + n - 1 of loop `src` become rows 0 .. n - 1 of loop `dst` (same max_len and page size): the pools of
    those rows, the event-level state, the per-row arrays and the mask rows."""
    mp, page = src.kv1.max_pages, src.kv1.page
    for ps, pd in zip(src.kv1.k + src.kv1.v, dst.kv1.k + dst.kv1.v):
        nh, D = src.kv1.cfg.n_head, src.kv1.cfg.head_dim
        pd.view(n, mp, nh, page, D).copy_(ps.view(src.B, mp, nh, page, D)[b0:b0 + n])
    dst.pos.copy_(src.pos)
    dst.counter.copy_(src.counter)
    for name in ("ev_in", "seq", "row_off", "row_end", "row_last", "row_temp", "row_top_p", "row_top_k", "row_seed",
                 "row_first", "mask"):
        getattr(dst, name).copy_(getattr(src, name)[b0:b0 + n])


def test_rows_kernel_at_17_to_32_rows_equals_launches_of_at_most_16():
    import ctypes
    model = GC._pt_models(("peaked",))["peaked"]
    V = model.tokenizer.vocab_size
    m = {k: 0.0 for k in ("wr_seq_mismatch", "wr_ev_in_mismatch", "wr_row_last_mismatch", "wr_pos_error", "wr_pools_mismatch",
                          "wr_x_mismatch", "wr_k2_mismatch", "wr_v2_mismatch", "wr_ev_t_mismatch", "wr_logits_mismatch",
                          "wr_draw_mismatch", "wr_ws_layout_error", "wr_one_vs_three_mismatch", "wr_not_live_changed")}
    n_rows = n_logits = n_clear = n_wide = 0
    subs = {}
    try:
        for n in (16, 1, 8, 15):                        # the group launches of 17, 24, 31 and 32 rows
            k, h = model._checkout_generator(n, GC.PT_MAX_LEN, 1.0, 0.98, 20, None)
            h.alloc_rows()
            subs[n] = (k, h)
        for B in WIDE_B:
            key, gg = model._checkout_generator(B, GC.PT_MAX_LEN, 1.0, 0.98, 20, None)
            try:
                gg.alloc_rows()
                gg.queue, gg.rows, gg.lengths = True, True, None
                gg.req_top_k = list(ROW_TOP_K)
                assert gg.persistent_ok()
                d, ws, _ = gg._persistent()
                L = DR.decode_ws_layout(d.batch, d.H, d.I_outer, d.I_inner, d.pitch, d.nh_outer, d.n_inner)
                m["wr_ws_layout_error"] += abs(L["total"] - lib.load().b200_decode_events_workspace_bytes(ctypes.byref(d)))
                H, n_in = d.H, d.n_inner
                kv = gg.kv1
                for pos in WIDE_POS:
                    gen = torch.Generator(device=DEV).manual_seed(pos * 17 + B)
                    prompt = torch.randint(0, V, (B, pos + 1, 8), generator=gen, device=DEV)
                    gg._set_lengths(prompt, None)
                    gg._set_state(prompt)
                    pools0 = [t.clone() for t in kv.k + kv.v]
                    vi = pos % 5
                    offs = GC._ragged_offsets(B, pos)
                    live = [not (b % 3 == 2 or b == 31) for b in range(B)]
                    ctx = [pos + o for o in offs]
                    GC._pt_state(gg, pools0, prompt, pos, offs, live, c0=3 + pos)
                    GC._pt_masks(gg, [(b + vi + pos) % 4 for b in range(B)], seed=pos + B)
                    settings, first, seeds = _rows_settings(gg, B, pos, ctx, live, vi)
                    state = kv.k + kv.v + [gg.seq, gg.ev_in, gg.pos, gg.counter, gg.row_last]
                    snap = [t.clone() for t in state]
                    # ---- the 32-row launch
                    ws.fill_(255)
                    GC._pt_launch(gg, "rows", 1)
                    torch.cuda.synchronize()
                    big = {"x": GC._pt_ws(ws, L, "x", BF, (B, H)),
                           "logits": GC._pt_ws(ws, L, "logits", BF, (B, d.pitch))[:, :V],
                           "ev_t": GC._pt_ws(ws, L, "ev_t", torch.int64, (8, B)),
                           "k2": GC._pt_ws(ws, L, "k2", BF, (n_in, B, 8, H)), "v2": GC._pt_ws(ws, L, "v2", BF, (n_in, B, 8, H))}
                    after = [t.clone() for t in state]
                    # ---- the same rows as launches of at most 16 rows, from the same state
                    for t, s in zip(state, snap):
                        t.copy_(s)
                    lv = torch.tensor(live, device=DEV)
                    for b0, nb in ((0, 16), (16, B - 16)):
                        h = subs[nb][1]
                        _copy_rows(gg, h, b0, nb)
                        h.queue, h.rows, h.lengths = True, True, None
                        hd, hws, _ = h._persistent()
                        hL = DR.decode_ws_layout(nb, hd.H, hd.I_outer, hd.I_inner, hd.pitch, hd.nh_outer, hd.n_inner)
                        ev_in0, mask_np = h.ev_in.clone(), h.mask.cpu().numpy()
                        h_pre = [t.clone() for t in h.kv1.k + h.kv1.v]
                        hws.fill_(255)
                        GC._pt_launch(h, "rows", 1)
                        torch.cuda.synchronize()
                        sl = slice(b0, b0 + nb)
                        hl = lv[sl]
                        x = GC._pt_ws(hws, hL, "x", BF, (nb, H))
                        evt = GC._pt_ws(hws, hL, "ev_t", torch.int64, (8, nb))
                        evt_np, bevt_np = evt.cpu().numpy(), big["ev_t"][:, sl].cpu().numpy()
                        n_h = sum(1 for i in range(8) if (evt_np[i] != -1).all())
                        n_b = sum(1 for i in range(8) if (big["ev_t"][i].cpu().numpy() != -1).all())
                        nn = min(n_h, n_b)
                        m["wr_x_mismatch"] += GC._ne(big["x"][sl][hl], x[hl])
                        m["wr_ev_t_mismatch"] += float((bevt_np[:nn][:, live[sl]] != evt_np[:nn][:, live[sl]]).sum())
                        for nm in ("k2", "v2"):
                            got = GC._pt_ws(hws, hL, nm, BF, (n_in, nb, 8, H))
                            m[f"wr_{nm}_mismatch"] += GC._ne(big[nm][:, sl][:, hl, :nn], got[:, hl, :nn])
                        if n_h == n_b:                      # the last step's logits: the same step in both launches
                            lg = GC._pt_ws(hws, hL, "logits", BF, (nb, hd.pitch))[:, :V]
                            m["wr_logits_mismatch"] += GC._ne(big["logits"][sl][hl], lg[hl])
                            n_logits += 1
                        sub_after = [h.seq, h.ev_in, h.row_last]
                        m["wr_seq_mismatch"] += float((after[-5][sl] != sub_after[0]).sum())
                        m["wr_ev_in_mismatch"] += float((after[-4][sl] != sub_after[1]).sum())
                        m["wr_row_last_mismatch"] += float((after[-1][sl] != sub_after[2]).sum())
                        m["wr_pos_error"] += abs(int(after[-3]) - int(h.pos))
                        mp, page = kv.max_pages, kv.page
                        nh, D = kv.cfg.n_head, kv.cfg.head_dim
                        for pb, ph, p0 in zip(after[:2 * len(kv.k)], h.kv1.k + h.kv1.v, h_pre):
                            bv = pb.view(B, mp, nh, page, D)[sl]
                            m["wr_pools_mismatch"] += float((~_same(bv, ph.view(nb, mp, nh, page, D))).sum())
                            dead = ~hl.view(nb, 1, 1, 1, 1).expand_as(bv)
                            m["wr_not_live_changed"] += float((~_same(bv, p0.view(nb, mp, nh, page, D)) & dead).sum())
                        # every draw of the group launch against the restated sampler (from the phase loop's logits)
                        kv2, llog = GC._pt_loop(h, x, evt, max(n_h, 1))
                        u = DR.event_uniforms("rows", nb, max(n_h, 1), pos=pos, row_off=offs[sl], row_first=first[sl],
                                              row_seed=seeds[sl])
                        dec_ = DR.event_decisions(llog.float().cpu().numpy(), evt_np, n_h, live[sl], settings[sl], mask_np,
                                                  u, h.g.lut.cpu().numpy(), h.g.eos, h.g.pad, h.g.n_event_types)
                        clear = (dec_["id"] >= 0) & ~dec_["amb"]
                        m["wr_draw_mismatch"] += float((clear & (dec_["id"] != evt_np[:n_h])).sum())
                        n_clear += int(clear.sum())
                        n_wide += int(clear[:, [s[2] > 64 for s in settings[sl]]].sum())
                        n_rows += nb
                    # ---- one launch of 3 events against three launches of one
                    runs = []
                    for split in (False, True):
                        for t, s in zip(state, snap):
                            t.copy_(s)
                        gg.mask[0, gg.g.eos] = 0
                        for _ in range(3 if split else 1):
                            GC._pt_launch(gg, "rows", 1 if split else 3)
                        torch.cuda.synchronize()
                        runs.append([t.clone() for t in state])
                    m["wr_one_vs_three_mismatch"] += sum(float((~_same(a, b_)).sum()) for a, b_ in zip(*runs))
            finally:
                gg.queue, gg.rows = False, False
                gg.set_deny(())
                model._return_generator(key, gg)
    finally:
        for k, h in subs.values():
            h.queue, h.rows = False, False
            h.set_deny(())
    m["wr_rows_compared"], m["wr_logits_compared"] = float(n_rows), float(n_logits)
    m["wr_clear_draws"], m["wr_wide_top_k_draws"] = float(n_clear), float(n_wide)
    print(m)
    P.assert_within(m, [(k, 0.0) for k in m if not k.endswith(("compared", "draws"))] +
                    [("min:wr_rows_compared", 200.0), ("min:wr_logits_compared", 4.0), ("min:wr_clear_draws", 500.0),
                     ("min:wr_wide_top_k_draws", 150.0)])


def test_32_slots_end_to_end_on_tv2o_medium(monkeypatch):
    from midi_b200 import decode as dec
    from midi_b200.serve import GenerateServer
    torch.manual_seed(0)
    model = GM.cpu_model(GM.config("tv2o-medium")).to(DEV, dtype=BF).eval()
    model._rt()                                     # the weight store outside inference mode, as a served model has it
    tok = model.tokenizer
    songs = GC._song_batch(tok, 40, 14, seed=995).numpy()
    N = 40
    lengths = [1 + (5 * i) % 14 for i in range(N)]
    budgets = [4 + (7 * i) % 13 for i in range(N)]
    prompts = [songs[i, :lengths[i]] for i in range(N)]
    top_k = [(20, 100, 128)[i % 3] for i in range(N)]
    temp = [(1.0, 1.3, 0.8)[i % 3] for i in range(N)]
    top_p = [(0.98, 1.0, 0.9)[i % 3] for i in range(N)]
    patch = [i % 4 == 1 for i in range(N)]
    chans = [[0, 1] if i % 7 == 2 else None for i in range(N)]
    seeds = [int(torch.randint(0, 2 ** 62, (1,), generator=torch.Generator().manual_seed(3000 + i))) for i in range(N)]

    def solo(i):
        return np.stack([e[0] for e in _mode("persist", lambda: list(model.generate_stream(
            prompt=prompts[i], batch_size=1, max_len=lengths[i] + budgets[i], temp=temp[i], top_p=top_p[i], top_k=top_k[i],
            disable_patch_change=patch[i], disable_channels=chans[i], generator=torch.Generator().manual_seed(3000 + i))))])

    ref = [solo(i) for i in range(N)]
    host_events = []
    real_event = dec.GraphGenerator._event
    monkeypatch.setattr(dec.GraphGenerator, "_event", lambda self: (host_events.append(self.B), real_event(self))[1])
    m = {"e2e_many_vs_solo_mismatch": 0.0, "e2e_server_vs_solo_mismatch": 0.0, "e2e_cancel_not_prefix": 0.0}
    got = _mode("persist", lambda: model.generate_many_requests(
        prompts, budgets, batch_size=32, temp=temp, top_p=top_p, top_k=top_k, disable_patch_change=patch,
        disable_channels=chans, seeds=seeds))
    for i in range(N):
        new = got[i][lengths[i]:]
        m["e2e_many_vs_solo_mismatch"] += float((new != ref[i]).sum()) if new.shape == ref[i].shape else 1e9
    # the server: four submitting threads, one cancellation, one top_k = 128 request among them
    streamed, errors, cancel = {}, [], 5

    def user(k, server):
        try:
            time.sleep(0.02 * k)
            reqs = {i: server.submit(prompts[i], budgets[i], temp=temp[i], top_p=top_p[i], top_k=top_k[i],
                                     disable_patch_change=patch[i], disable_channels=chans[i], seed=seeds[i])
                    for i in range(k, N, 4)}
            for i, r in reqs.items():
                evs = []
                for ev in r:
                    evs.append(ev)
                    if i == cancel and len(evs) == 2:
                        r.cancel()
                streamed[i] = np.stack(evs) if evs else np.zeros((0, 8), dtype=np.int64)
        except Exception as e:                      # noqa: BLE001  reported below
            errors.append(e)

    with _Env("persist"), GenerateServer(model, batch_size=32, max_len=64) as server:
        threads = [threading.Thread(target=user, args=(k, server)) for k in range(4)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        on_kernel = server._persist
    assert not errors, errors
    for i in range(N):
        s = streamed[i]
        if i == cancel:
            m["e2e_cancel_not_prefix"] += float((s != ref[i][:len(s)]).sum()) if len(s) <= len(ref[i]) else 1e9
        else:
            m["e2e_server_vs_solo_mismatch"] += float((s != ref[i]).sum()) if s.shape == ref[i].shape else 1e9
    m["e2e_host_issued_events"] = float(len(host_events))
    m["e2e_server_on_kernel"] = float(on_kernel)
    m["e2e_wide_top_k_requests"] = float(sum(k > 64 for k in top_k))
    print(m)
    P.assert_within(m, [("e2e_many_vs_solo_mismatch", 0.0), ("e2e_server_vs_solo_mismatch", 0.0),
                        ("e2e_cancel_not_prefix", 0.0), ("e2e_host_issued_events", 0.0), ("min:e2e_server_on_kernel", 1.0),
                        ("min:e2e_wide_top_k_requests", 20.0)])
