"""The restatements of tests/decode_reference.py and the case sets the decode conformance groups (gv_ / da_ / sm_ / pd_ in
gpu_checks.py) feed them, on the CPU: each defect a sampler, RNG or paged-KV kernel could plausibly have changes the
result on some case, and is judged a failure by the bounds the GPU groups use (the tables of gpu_checks.GROUPS)."""
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
