"""The restatements of tests/decode_reference.py and the case sets the decode conformance groups (gv_ / da_ / sm_ / pd_ /
pt_ in gpu_checks.py) feed them, on the CPU: each defect a sampler, RNG, paged-KV or persistent kernel could plausibly have
changes the result on some case, and is judged a failure by the bounds the GPU groups use (the tables of gpu_checks.GROUPS)."""
import math

import numpy as np
import pytest
import torch

import decode_reference as R
import gpu_checks as G
import parity_metrics as P

BF = torch.bfloat16


def _fails(group, metrics):
    res = P.check_bounds(metrics, G.GROUPS[group].bounds)
    assert all(b is not None for _, _, b, _ in res), res
    return any(not ok for *_, ok in res)


def _topp_topk_mismatches(bf16_sem, **defect):
    """Rows (over the sm_ group's V / top_p / top_k sweep) where the restatement with `defect` picks another id."""
    bad = 0
    for V in G.SM_VOCABS:
        probs = R.sampler_cases(V, seed=V)
        if bf16_sem:
            probs = torch.from_numpy(probs).to(BF).float().numpy()
        u = R.uniforms(probs.shape[0], seed=V + 1)
        for top_k in G.sm_top_ks(V):
            for top_p in G.SM_TOP_PS:
                good = R.sample_rows(probs, top_p, top_k, u, bf16_sem)
                bad += int((R.sample_rows(probs, top_p, top_k, u, bf16_sem, **defect) != good).sum())
    return bad


@pytest.mark.parametrize("bf16_sem", [False, True])
@pytest.mark.parametrize("defect", [dict(tie_high=True), dict(cut_ge=True), dict(k_off=1), dict(k_off=-1)],
                         ids=["ties_to_highest_id", "top_p_ge", "top_k_plus_1", "top_k_minus_1"])
def test_sampler_cases_catch_defect(bf16_sem, defect):
    n = _topp_topk_mismatches(bf16_sem, **defect)
    assert n > 0
    assert _fails("sampler_exact", {"sm_topp_fp32_mismatch": float(n)})


def test_sampler_cases_catch_unrounded_cumulative_sums():
    n = _topp_topk_mismatches(True, round_cum=False)
    assert n > 0 and _fails("sampler_exact", {"sm_topp_bf16_mismatch": float(n)})


def test_sampler_restatement_reference_semantics():
    # midi_model.py:152-165 on hand-made rows: sort desc, cut where the mass before exceeds top_p, keep top_k, draw
    p = np.array([0.1, 0.4, 0.0, 0.3, 0.2], dtype=np.float32)
    assert R.sample_tail(p, 1.0, 1, 0.99, False) == 1                 # greedy
    assert R.sample_tail(p, 1.0, 2, 0.99, False) == 3                 # last of the top 2
    assert R.sample_tail(p, 0.5, 5, 0.99, False) == 3                 # mass before id 3 is 0.4 <= 0.5, before id 4 0.7
    assert R.sample_tail(p, 0.3, 5, 0.99, False) == 1                 # only the first survives
    assert R.sample_tail(p, 1.0, 5, 0.0, False) == 1
    tie = np.array([0.0, 0.25, 0.5, 0.25, 0.25], dtype=np.float32)
    assert R.sample_tail(tie, 1.0, 2, 0.99, False) == 1               # tie at the 2nd value: lowest id
    assert R.sample_tail(tie, 1.0, 2, 0.99, False, tie_high=True) == 4
    assert R.sample_tail(np.zeros(7, np.float32), 0.9, 3, 0.5, True) == 0
    assert R.sample_tail(np.array([np.nan, -1.0, 0.2], np.float32), 0.9, 3, 0.5, False) == 2


def test_logits_restatement_ambiguity_and_empty_range():
    rng = np.random.default_rng(3)
    l = torch.from_numpy(rng.standard_normal(3406) * 2.5).to(BF).float().numpy()
    amb = 0
    for r in range(200):
        _, a = R.logits_sample(l * (1 + 0.01 * r), 1.0, 0.98, 20, 0, 3406, None, 0.5)
        amb += a
    assert 0 < amb < 200
    mask = np.ones(3406, np.uint8)
    mask[10:30] = 0
    assert R.logits_sample(l, 0.7, 0.98, 20, 10, 30, mask, 0.5) == (10, False)
    # greedy inside the range is the largest logit of the range (ties: lowest id)
    lt = l.copy()
    lt[40:50] = 9.0
    idx, a = R.logits_sample(lt, 1.0, 1.0, 1, 35, 60, None, 0.3)
    assert idx == 40 and not a


def test_uniform_fill_restatement():
    u = R.uniform_fill(1024, seed=12345, counter=7, dev_seed=99)
    assert u.dtype == np.float32 and u.min() >= 0 and u.max() < 1
    assert abs(float(u.mean()) - 0.5) < 0.05
    assert np.all(u * 16777216 == np.floor(u * 16777216))            # 24-bit grid
    assert not np.array_equal(u, R.uniform_fill(1024, seed=12345, counter=8, dev_seed=99))
    for i in range(3):
        consts = list((R._GOLD, R._M1, R._M2))
        consts[i] ^= 1 << 17                                          # one constant changed
        bad = R.uniform_fill(1024, seed=12345, counter=7, dev_seed=99, consts=tuple(consts))
        n = float((bad != u).sum())
        assert n > 0 and _fails("sampler_exact", {"sm_uniform_mismatch": n})


def test_event_commit_restatement():
    B, T, L = 3, 8, 5
    ev_t = np.arange(T * B).reshape(T, B)
    seq = np.full((B, L, T), -5)
    nxt = np.zeros((B, T), np.int64)
    s2, n2, p2 = R.event_commit(ev_t, seq, nxt, 2, L)
    assert p2 == 3 and np.array_equal(s2[:, 3], ev_t.T) and np.array_equal(n2, ev_t.T)
    assert (s2[:, :3] == -5).all() and (s2[:, 4:] == -5).all()
    s3, _, p3 = R.event_commit(ev_t, seq, nxt, L - 1, L)                # pos + 1 == max_len: seq untouched
    assert p3 == L and (s3 == -5).all()


# ------------------------------------------------------------------------------------------ paged KV metrics
def _pool(nh=2, D=16, page=8, Bn=2, max_pages=3, spare=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    n_pages = Bn * max_pages + spare
    bt = torch.randperm(n_pages, generator=g)[:Bn * max_pages].int().view(Bn, max_pages)
    return P.nan_buffer((n_pages, nh, page, D)), P.nan_buffer((n_pages, nh, page, D)), bt


def test_pool_slot_written_one_position_late_fails():
    k, v, bt = _pool()
    page, T = 8, 13
    vals = torch.randn(2, T, 2, 16, generator=torch.Generator().manual_seed(1)).to(BF)
    for late in (0, 1):
        kk = k.clone()
        for b in range(2):
            for t in range(T):
                kk[int(bt[b, (t + late) // page]), :, (t + late) % page] = vals[b, t]
        m = R.slot_mask(kk.shape, bt, page, [(b, t) for b in range(2) for t in range(T)])
        rep = {f"da_append_{k_}": v_ for k_, v_ in P.sentinel_report(kk, m).items()}
        got = torch.stack([R.gather_kv(kk, bt, page, b, T) for b in range(2)]).transpose(1, 2)
        rep["da_append_mismatch"] = float((got != vals).sum())
        assert _fails("decode_attn_edges", rep) == bool(late), rep
        if late:
            assert rep["da_append_sentinels_changed"] > 0 and rep["da_append_nan_in_range"] > 0


def test_key_read_past_context_propagates_nan():
    k, v, bt = _pool(seed=2)
    page, T = 8, 13
    g = torch.Generator().manual_seed(3)
    for b in range(2):
        for t in range(T):
            k[int(bt[b, t // page]), :, t % page] = torch.randn(2, 16, generator=g).to(BF)
            v[int(bt[b, t // page]), :, t % page] = torch.randn(2, 16, generator=g).to(BF)
    q = torch.randn(2, 3, 16, generator=g, dtype=torch.float64)
    ref = R.paged_attention64(q, k, v, bt, page, 0, T, 0.25)
    assert torch.isfinite(ref).all()
    # the same attention rounded to bf16 passes the per-row bound; one key past T (a NaN slot) makes the row +inf
    assert not _fails("decode_attn_edges", {"da_attn_d64_o_row": P.row_worst(ref.to(BF), ref)})
    past = R.paged_attention64(q, k, v, bt, page, 0, T + 1, 0.25)[:, -1:]
    assert math.isinf(P.row_worst(past, ref[:, -1:]))
    assert _fails("decode_attn_edges", {"da_attn_d64_o_row": P.row_worst(past, ref[:, -1:])})
    # reading one slot early (key t-1 for key t) moves a row by far more than the bound
    k_shift = k.clone()
    for t in range(T - 1, 0, -1):
        k_shift[int(bt[0, t // page]), :, t % page] = k[int(bt[0, (t - 1) // page]), :, (t - 1) % page]
    early = R.paged_attention64(q, k_shift, v, bt, page, 0, T, 0.25)
    assert _fails("decode_attn_edges", {"da_attn_d64_o_row": P.row_worst(early.to(BF), ref)})


# ------------------------------------------------------------------------------------------ persistent kernel, token level
_PT_TEMP, _PT_TOP_P, _PT_TOP_K = (0.5, 1.0, 1.7), (1.0, 0.98, 0.5, 0.1), (1, 2, 20, 64)


def _grammar():
    from midi_b200.decode import GrammarLUT
    from midi_b200.tokenizer_tables import TokenizerTables
    g = GrammarLUT(TokenizerTables("v2"), "cpu")
    return g, g.lut.numpy()


def _pt_event(seed, B=8, kind="plain", scale=3.0):
    """A synthetic event of the persistent kernel that follows the restatement exactly: bf16 logits [8, B, V], per-row
    settings as check_persist_token_exact mixes them, rows b % 4 == 3 not live, every fourth row masked, and the tokens
    ev_t [8, B] the restated draws give (pad for rows that are not live and past n_steps)."""
    g, lut = _grammar()
    V = 3406
    rng = np.random.default_rng(seed)
    logits = torch.from_numpy(rng.standard_normal((8, B, V)) * scale).to(BF).float().numpy()
    settings = [(_PT_TEMP[b % 3], _PT_TOP_P[(b + seed) % 4], _PT_TOP_K[(b + 1) % 4]) for b in range(B)]
    live = [b % 4 != 3 for b in range(B)]
    masks = np.ones((B, V), np.uint8)
    masks[0::4, g.eos + 1 + g.n_event_types:] = rng.random(V - g.eos - 1 - g.n_event_types) > 0.4
    rows = dict(pos=70 + seed, row_off=[-(b % 3) for b in range(B)], row_first=[40 + b for b in range(B)],
                row_seed=[1000003 * (b + 1) + seed for b in range(B)])
    u = (R.event_uniforms("rows", B, 8, **rows) if kind == "rows" else
         R.event_uniforms(kind, B, 8, c0=5 + seed, seed=0x5EED + seed))
    ev_t = np.full((8, B), g.pad, np.int64)
    ev_t[0] = R.event_decisions(logits[:1], ev_t, 1, live, settings, masks, u, lut, g.eos, g.pad, g.n_event_types)["id"][0]
    ev_t[0][~np.array(live)] = g.pad
    n = R.event_n_steps(ev_t[0], live, lut, g.eos, g.n_event_types)
    dec = R.event_decisions(logits[:n], ev_t, n, live, settings, masks, u, lut, g.eos, g.pad, g.n_event_types)
    ev_t[:n] = np.where(dec["id"] >= 0, dec["id"], g.pad)
    return dict(g=g, lut=lut, logits=logits, settings=settings, live=live, masks=masks, u=u, ev_t=ev_t, n=n, rows=rows,
                kind=kind, dec=dec)


def _pt_mismatches(ev, u=None, **defect):
    """Unambiguous decisions of the synthetic event where the restatement with `defect` (or with uniforms `u`) draws
    another id than the event's tokens."""
    g = ev["g"]
    d = R.event_decisions(ev["logits"][:ev["n"]], ev["ev_t"], ev["n"], ev["live"], ev["settings"], ev["masks"],
                          ev["u"] if u is None else u, ev["lut"], g.eos, g.pad, g.n_event_types, **defect)
    clear = (d["id"] >= 0) & ~d["amb"]
    return int((clear & (d["id"] != ev["ev_t"][:ev["n"]])).sum())


def test_counter_uniform_is_uniform_fill():
    seed, dev_seed, c = 987654321, 0x1234567890ABCDE, 5
    u = R.uniform_fill(1024, seed, c, dev_seed)
    assert np.array_equal(R.counter_uniform(seed ^ dev_seed, c, np.arange(1024)), u)
    assert R.counter_uniform(seed ^ dev_seed, c, 7) == u[7]
    assert not np.array_equal(R.counter_uniform(seed ^ dev_seed, c + 1, np.arange(1024)), u)


def test_token_event_restatement_is_self_consistent():
    # the synthetic events draw what the restatement draws, in ranges that follow the grammar, with every counter hit
    evs = [_pt_event(s, kind=k) for s in range(4) for k in ("plain", "rows")]
    for ev in evs:
        assert _pt_mismatches(ev) == 0
        g = ev["g"]
        for b in range(len(ev["live"])):
            if ev["live"][b]:
                assert g.eos <= ev["ev_t"][0, b] <= g.eos + g.n_event_types
    dec = [ev["dec"] for ev in evs]
    clear = [(d["id"] >= 0) & ~d["amb"] for d in dec]
    assert sum(int((c & d["cut"]).sum()) for c, d in zip(clear, dec)) > 0
    assert sum(int(c.sum()) for c in clear) > 0.5 * sum(int((d["id"] >= 0).sum()) for d in dec)


@pytest.mark.parametrize("defect", ["next_row_uniform", "temperature_twice", "previous_step_range",
                                    "rows_index_without_row_first"])
def test_token_decisions_catch_defect(defect):
    n = 0
    for s in range(4):
        ev = _pt_event(s, kind="rows" if defect == "rows_index_without_row_first" else "plain")
        B = len(ev["live"])
        if defect == "next_row_uniform":
            n += _pt_mismatches(ev, u=R.event_uniforms("plain", B, 8, c0=5 + s, seed=0x5EED + s, row_shift=1))
        elif defect == "temperature_twice":
            n += _pt_mismatches(ev, temp_twice=True)
        elif defect == "previous_step_range":
            n += _pt_mismatches(ev, range_lag=1)
        else:
            n += _pt_mismatches(ev, u=R.event_uniforms("rows", B, 8, use_first=False, **ev["rows"]))
    assert n > 0
    assert _fails("persist_token_exact", {"pt_draw_mismatch": float(n)})


def test_token_bookkeeping_catches_defects():
    g, lut = _grammar()
    bad_steps = bad_commit = 0
    for s in range(4):
        ev = _pt_event(s, kind="plain")
        ev0, live = ev["ev_t"][0], ev["live"]
        n = R.event_n_steps(ev0, live, lut, g.eos, g.n_event_types)
        assert n == ev["n"] and 2 <= n <= 8
        for off in (-1, 1):
            bad_steps += abs(R.event_n_steps(ev0, live, lut, g.eos, g.n_event_types, off=off) - n)
        B, pos = len(live), 50
        seq, ev_in = np.full((B, 60, 8), -5), np.arange(B * 8).reshape(B, 8)
        offs = [-(b % 3) for b in range(B)]
        tok, want, want_in = R.event_commit_rows(ev["ev_t"], n, live, seq, ev_in, pos, offs, g.pad)
        assert (tok[:, n:] == g.pad).all()
        for b in range(B):
            changed = np.nonzero((want[b] != -5).any(-1))[0].tolist()
            assert changed == ([pos + offs[b] + 1] if live[b] else [])
            assert np.array_equal(want_in[b], tok[b] if live[b] else ev_in[b])
        _, wrong, _ = R.event_commit_rows(ev["ev_t"], n, live, seq, ev_in, pos, offs, g.pad, commit_all=True)
        bad_commit += int((wrong != want).sum())
    assert bad_steps > 0 and _fails("persist_token_exact", {"pt_n_steps_error": float(bad_steps)})
    assert bad_commit > 0 and _fails("persist_token_exact", {"pt_seq_mismatch": float(bad_commit)})


def test_token_steps64_is_the_oracle_forward_token_and_catches_a_rope_lag():
    from types import SimpleNamespace
    from oracle import midi_oracle as O
    cfg = O.ModelCfg(vocab=50, n_layer=8, n_head=8, n_embd=64, n_inner=128)     # token level: 2 layers, 2 heads of 32
    tc, V, H = cfg.net_token, cfg.vocab, cfg.n_embd
    gen = torch.Generator().manual_seed(0)

    def r(*shape, scale=1.0):
        return torch.randn(*shape, generator=gen, dtype=torch.float64) * scale

    sd, layers = {}, []
    for li in range(tc.n_layer):
        p = f"net_token.layers.{li}."
        for n_, shape in (("self_attn.q_proj", (H, H)), ("self_attn.k_proj", (H, H)), ("self_attn.v_proj", (H, H)),
                          ("self_attn.o_proj", (H, H)), ("mlp.gate_proj", (tc.inner, H)), ("mlp.up_proj", (tc.inner, H)),
                          ("mlp.down_proj", (H, tc.inner))):
            sd[p + n_ + ".weight"] = r(*shape, scale=shape[1] ** -0.5)
        sd[p + "input_layernorm.weight"] = 1 + 0.1 * r(H)
        sd[p + "post_attention_layernorm.weight"] = 1 + 0.1 * r(H)
        w = lambda n_: sd[p + n_ + ".weight"]                                          # noqa: E731
        layers.append(SimpleNamespace(
            qkv=torch.cat([w("self_attn.q_proj"), w("self_attn.k_proj"), w("self_attn.v_proj")]), o=w("self_attn.o_proj"),
            gu=torch.cat([w("mlp.gate_proj"), w("mlp.up_proj")]), down=w("mlp.down_proj"), ln1=w("input_layernorm"),
            ln2=w("post_attention_layernorm")))
    sd["net_token.norm.weight"], sd["net_token.embed_tokens.weight"] = 1 + 0.1 * r(H), r(V, H)
    sd["lm_head.weight"] = r(V, H, scale=H ** -0.5)
    eng = SimpleNamespace(cfg=SimpleNamespace(n_head=tc.n_head, head_dim=tc.head_dim, hidden=H, eps=tc.eps), layers=layers,
                          norm=sd["net_token.norm.weight"], embed=sd["net_token.embed_tokens.weight"])
    B, n = 3, 8
    x, outer_norm = r(B, H), 1 + 0.1 * r(H)
    tokens = torch.randint(0, V, (8, B), generator=gen)
    tokens[2, 1], tokens[4, 0] = V + 5, -1                                            # outside [0, V): row 0
    inv = O.default_inv_freq(tc.head_dim)
    cos, sin = (t[:, :tc.head_dim // 2] for t in O.rope_cos_sin(inv, torch.arange(8), torch.float64))
    k, v, logits = G._token_steps64(eng, sd["lm_head.weight"], outer_norm, x, tokens, n, cos, sin)
    ids = tokens[:n - 1].T.clone()
    ids[(ids < 0) | (ids >= V)] = 0
    cache = O.KV()
    ref = O.forward_token(sd, cfg, O.rmsnorm(x, outer_norm, tc.eps), ids, cache=cache, inv_freq=inv)
    # the oracle normalises and forms attention scores in fp32 (hf's RMSNorm and sdpa semantics), the rest in fp64
    for got, want in [(logits, ref)] + [(k[li], cache.k[li].transpose(1, 2)) for li in range(tc.n_layer)] + \
            [(v[li], cache.v[li].transpose(1, 2)) for li in range(tc.n_layer)]:
        assert float((got - want).abs().max()) < 1e-5 * float(want.abs().max())
    # the same steps with step i rotated at position i - 1: far outside the fp64 bounds of the pt_ group
    k_lag, _, lg_lag = G._token_steps64(eng, sd["lm_head.weight"], outer_norm, x, tokens, n, cos, sin, rope_lag=1)
    assert torch.equal(k_lag[:, :, 0], k[:, :, 0])
    assert _fails("persist_token_exact", {"pt_f64_k_row": P.row_worst(k_lag, k)})
    assert _fails("persist_token_exact", {"pt_f64_logits_row": P.row_worst(lg_lag[:, -1], logits[:, -1])})
