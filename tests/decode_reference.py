"""Exact restatements of the generate-path kernels that are not a product of bf16 operands: the samplers
(csrc/sampler.cuh), the counter-based RNG and the event commit (csrc/decode.cu), the token-level bookkeeping of the
persistent generate kernel (csrc/decode_persist.cu: grammar ranges, uniforms, step count, commit, workspace layout), plus
an fp64 paged-KV attention that reads keys through the block table.  NumPy / PyTorch on the CPU, so
tests/test_decode_reference.py can show that each one, and the case sets the decode conformance groups of gpu_checks.py
feed it, catches the defects a kernel could plausibly have.

The sampler tail is single-thread fp32 arithmetic (sort by (p desc, id asc), top-k, top-p on bf16-rounded cumulative
sums, a renormalised draw with u), so NumPy float32 scalars reproduce it bit for bit."""
from __future__ import annotations

import numpy as np
import torch

F32 = np.float32


# ------------------------------------------------------------------------------------------ bf16 rounding in NumPy
def bf16_np(x) -> np.ndarray:
    """fp32 values rounded to the nearest bf16 (ties to even), returned as fp32 (finite inputs)."""
    b = np.asarray(x, dtype=F32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(F32)


def _bf16s(x) -> F32:
    return F32(bf16_np(F32(x)).reshape(()))


# ------------------------------------------------------------------------------------------ sampler tail
def sample_tail(p, top_p: float, top_k: int, u: float, bf16_sem: bool, *, tie_high=False, cut_ge=False, k_off=0,
                round_cum=True) -> int:
    """smp::sample_tail (and the fast path of smp::sample_logits_row, which gives the same id) over one row of
    probabilities `p` (fp32 values as the kernel reads them, indexed by id).  Entries that are not > 0 (NaN, negative,
    zero) are not candidates; a row without candidates returns 0.

    The keyword-only switches plant the defects tests/test_decode_reference.py shows the case sets catch: ties broken
    towards the highest id, the top-p test with >= instead of >, top-k off by k_off, cumulative sums not rounded to bf16."""
    p = np.asarray(p, dtype=F32)
    p = np.where(p > 0, p, F32(0))                       # NaN > 0 is False
    ids = np.nonzero(p > 0)[0]
    if ids.size == 0:
        return 0
    order = np.lexsort((-ids if tie_high else ids, -p[ids].astype(np.float64)))
    ids = ids[order]
    ps = p[ids]
    kk = max(0, min(ids.size, max(1, top_k) + k_off))
    sem = bf16_sem and round_cum
    pth = _bf16s(top_p) if bf16_sem else F32(top_p)
    # the kernel's loops are sequential fp32 sums; np.cumsum in float32 adds in the same order
    ps = ps[:kk]
    cum = np.cumsum(ps, dtype=F32)
    cs = bf16_np(cum) if sem else cum
    before = bf16_np(cs - ps) if sem else (cs - ps).astype(F32)
    cut = (before >= pth) if cut_ge else (before > pth)
    w = np.where(cut, F32(0), ps).astype(F32)
    run = np.cumsum(w, dtype=F32)
    total = run[-1] if kk else F32(0)
    choice = 0
    if total > 0:
        last = int(np.nonzero(w > 0)[0][-1])
        target = F32(F32(u) * total)
        hit = np.nonzero((w[:last + 1] > 0) & (run[:last + 1] > target))[0]
        choice = int(hit[0]) if hit.size else last
    return int(ids[choice])


def sample_rows(probs: np.ndarray, top_p: float, top_k: int, u: np.ndarray, bf16_sem: bool, **defect) -> np.ndarray:
    """b200_sample_topp_topk restated: one id per row of probs [R, V]."""
    return np.array([sample_tail(probs[r], top_p, top_k, float(u[r]), bf16_sem, **defect) for r in range(probs.shape[0])],
                    dtype=np.int64)


def sampler_cases(V: int, seed: int) -> np.ndarray:
    """Rows of probabilities [R, V] (fp32) for b200_sample_topp_topk: softmax rows of several temperatures, exact ties
    straddling ranks 1, 20, 64 and 65 with the tied ids scattered, dyadic rows whose cumulative sums land exactly on
    top_p = 0.5 / 0.75, rows with NaN and negative entries, all-zero rows and one-candidate rows."""
    rng = np.random.default_rng(seed)
    rows = []
    for scale in (0.5, 2.0, 4.0):
        for _ in range(6):
            z = rng.standard_normal(V) * scale
            e = np.exp(z - z.max())
            rows.append(e / e.sum())
    for k in (1, 20, 64, 65):
        if V < 2:
            break
        for n_tie in (2, 7):
            r = rng.random(V) * 1e-3
            perm = rng.permutation(V)
            lead = min(k - 1, V - 1)
            r[perm[:lead]] = 0.5 + rng.random(lead)              # strictly above the tie
            tie = perm[lead:lead + n_tie]
            r[tie] = 0.25                                         # ties across the k-th value
            rows.append(r / r.sum() if n_tie == 7 else r)         # one normalised, one not: the tail renormalises
    if V >= 4:
        for vals in ((0.5, 0.25, 0.125, 0.125), (0.25, 0.25, 0.25, 0.125, 0.125)):
            r = np.zeros(V)
            pos = rng.permutation(V)[:len(vals)]
            r[pos] = vals[:len(pos)]
            rows.append(r)
    r = rng.random(V)
    r[rng.permutation(V)[:max(1, V // 3)]] = np.nan
    r[rng.permutation(V)[:max(1, V // 4)]] *= -1
    rows.append(r)
    rows.append(np.zeros(V))
    r = np.zeros(V)
    r[rng.integers(0, V)] = 0.3
    rows.append(r)
    r = np.full(V, -1.0)
    r[0] = np.nan
    rows.append(r)
    return np.stack(rows).astype(F32)


def uniforms(n: int, seed: int) -> np.ndarray:
    """u per row: the edges 0, 0.5 and 1 - 2^-24 cycled with random values."""
    rng = np.random.default_rng(seed)
    u = rng.random(n).astype(F32)
    u[0::4] = 0.0
    u[1::4] = 0.5
    u[2::4] = F32(1 - 2.0 ** -24)
    return u


# ------------------------------------------------------------------------------------------ logits sampler
def _near_bf16_midpoint(p64: np.ndarray, rel_tol: float) -> np.ndarray:
    """True where p64 lies within rel_tol (relative) of a rounding midpoint between two bf16 values."""
    lo = (p64.astype(F32).view(np.uint32) & np.uint32(0xFFFF0000)).view(F32).astype(np.float64)
    mid = ((lo.astype(F32).view(np.uint32) | np.uint32(0x8000)).view(F32)).astype(np.float64)
    return np.abs(p64 - mid) <= rel_tol * np.abs(p64)


def _logits_probs(l, temp: float, lo: int, hi: int, mask):
    """(fp64 p of the allowed ids, 0 elsewhere; allowed; p rounded to bf16) of one logits row, as logits_sample forms them."""
    l = np.asarray(l, dtype=F32)
    x = l if temp == 1.0 else bf16_np(l / F32(temp))
    x64 = x.astype(np.float64)
    e = np.exp(x64 - x64.max())
    p64 = e / e.sum()
    allowed = np.zeros(l.shape[0], dtype=bool)
    allowed[lo:hi] = True
    if mask is not None:
        allowed &= np.asarray(mask) != 0
    p64 = np.where(allowed, p64, 0.0)
    return p64, allowed, bf16_np(p64.astype(F32))


def logits_sample(l, temp: float, top_p: float, top_k: int, lo: int, hi: int, mask, u: float,
                  rel_tol: float = 2.0 ** -17):
    """b200_sample_from_logits for one row restated from fp64 probabilities rounded to bf16.  Returns (id, ambiguous).

    x = bf16(l / temp) (fp32 division), p = bf16(exp(x - max) / sum over the whole vocabulary), ids outside [lo, hi) or
    masked out are not candidates, then the sampler tail.  The kernel's p comes from __expf and an fp32 sum, which can
    sit about one fp32 ulp per unit of |x - max| from the fp64 value; where a candidate that could reach the top k lies
    within rel_tol of a bf16 rounding midpoint, its bf16 p (and so the id) is not determined and the row is ambiguous.
    With every such p determined, the tail is exact fp32 arithmetic on the same values, so u * total needs no margin.
    No candidate (every allowed p rounds to 0): the kernel returns lo."""
    p64, allowed, pb = _logits_probs(l, temp, lo, hi, mask)
    cand = pb > 0
    if not cand.any():
        return lo, bool(_near_bf16_midpoint(p64[allowed], rel_tol).any()) if allowed.any() else False
    kk = min(int(cand.sum()), max(1, top_k))
    kth = np.sort(p64[cand])[::-1][kk - 1]
    # a one-ulp flip moves a bf16 value by at most 2^-7 relative: candidates below 0.98 of the k-th value cannot enter
    relevant = allowed & (p64 >= 0.98 * kth)
    amb = bool(_near_bf16_midpoint(p64[relevant], rel_tol).any())
    return sample_tail(pb, top_p, top_k, u, True), amb


# ------------------------------------------------------------------------------------------ RNG and commit
_GOLD, _M1, _M2 = 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9, 0x94D049BB133111EB


def uniform_fill(n: int, seed: int, counter: int, dev_seed: int, consts=(_GOLD, _M1, _M2)) -> np.ndarray:
    """b200_uniform_fill: u[i] = top 24 bits of splitmix64(seed ^ dev_seed + GOLD (counter * 4096 + i + 1)) * 2^-24.
    `consts` is there so that the CPU test can show one changed constant is caught."""
    g, m1, m2 = (np.uint64(c) for c in consts)
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64((seed ^ dev_seed) & (2 ** 64 - 1)) + g * (np.uint64(counter) * np.uint64(4096) + i + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * m1
        z = (z ^ (z >> np.uint64(27))) * m2
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(F32) * F32(1.0 / 16777216.0)


def event_commit(ev_t: np.ndarray, seq: np.ndarray, ev_next: np.ndarray, pos: int, max_len: int):
    """b200_event_commit: ev_t [T, B] -> seq[b, pos + 1] (only when pos + 1 < max_len) and ev_next [B, T]; pos + 1."""
    seq, ev_next = seq.copy(), ev_next.copy()
    if pos + 1 < max_len:
        seq[:, pos + 1] = ev_t.T
    ev_next[:] = ev_t.T
    return seq, ev_next, pos + 1


def counter_uniform(seed, c, i, consts=(_GOLD, _M1, _M2)) -> np.ndarray:
    """smp::counter_uniform (csrc/sampler.cuh): draw i of counter value c under `seed`, element-wise over broadcast
    integer arrays.  uniform_fill(n, seed, counter, dev_seed)[i] is counter_uniform(seed ^ dev_seed, counter, i)."""
    g, m1, m2 = (np.uint64(k) for k in consts)
    s, c, i = (np.asarray(v, dtype=np.int64).astype(np.uint64) for v in (seed, c, i))
    with np.errstate(over="ignore"):
        z = s + g * (c * np.uint64(4096) + i + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * m1
        z = (z ^ (z >> np.uint64(27))) * m2
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(F32) * F32(1.0 / 16777216.0)


# ------------------------------------------------------------------------------------------ persistent generate kernel
# The token-level half of one event of decode_events_kernel (csrc/decode_persist.cu): which ids each row may draw at each
# step, which uniform it draws with, how many steps the event runs and what it commits.  The keyword-only switches plant
# the defects tests/test_decode_reference.py shows the pt_ scores of gpu_checks.check_persist_token_exact catch.
PD_T, PD_MAXC = 8, 160


def grammar_range(step: int, ev0: int, lut: np.ndarray, eos: int, pad: int, n_event_types: int, *, lag=0):
    """(lo, hi) of the ids a row may draw at token step `step` of an event whose step-0 token is ev0 (sample_row): step 0
    EOS and the event types; step i the range of the event type's parameter i - 1 (lut [n_event_types, 8, 2]); pad alone
    after EOS, for an id that is no event type, or past the type's last parameter.  `lag`: the range of step - lag."""
    step = max(0, step - lag)
    if step == 0:
        return eos, eos + 1 + n_event_types
    e = int(ev0) - (eos + 1)
    if ev0 == eos or e < 0 or e >= n_event_types:
        return pad, pad + 1
    lo, hi = (int(v) for v in lut[e, step - 1])
    return (lo, hi) if hi > lo else (pad, pad + 1)


def event_n_steps(ev0, live, lut: np.ndarray, eos: int, n_event_types: int, *, off=0) -> int:
    """Token steps of the event (midi_model.py:234-237): two at least, else one past the last parameter of every live
    row's event type, at most PD_T.  ev0 [B]: each row's step-0 token; live [B] bool.  `off` plants an off-by-one."""
    need = 2
    for b in range(len(ev0)):
        e = int(ev0[b]) - (eos + 1)
        if not live[b] or ev0[b] == eos or e < 0 or e >= n_event_types:
            continue
        n_par = max([s + 1 for s in range(PD_T - 1) if lut[e, s, 1] > lut[e, s, 0]], default=0)
        need = max(need, n_par + 1)
    return min(PD_T, need) + off


def event_uniforms(kind: str, B: int, n: int, *, c0=0, seed=0, events_done=0, pos=0, row_off=None, row_first=None,
                   row_seed=None, row_shift=0, use_first=True) -> np.ndarray:
    """u [n, B] of the event's steps 0 .. n-1.  kind "rows" (b200_decode_events_queue_rows): row b draws
    counter_uniform(row_seed[b], 8 j + i, 0) at its new event j = pos + row_off[b] - row_first[b], the draw of generating
    the request alone.  Any other kind: counter_uniform(seed, c0 + 8 events_done + i, b), seed and c0 the descriptor's
    rng_state.  `row_shift` draws with row b + row_shift's uniform; use_first=False leaves row_first out of j."""
    u = np.zeros((n, B), dtype=F32)
    for b in range(B):
        bb = (b + row_shift) % B if kind == "rows" else b + row_shift
        for i in range(n):
            if kind == "rows":
                j = pos + int(row_off[bb]) - (int(row_first[bb]) if use_first else 0)
                u[i, b] = counter_uniform(int(row_seed[bb]), PD_T * j + i, 0)
            else:
                u[i, b] = counter_uniform(seed, c0 + PD_T * events_done + i, bb)
    return u


def event_decisions(logits, ev_t, n_steps: int, live, settings, masks, u, lut, eos: int, pad: int, n_event_types: int, *,
                    range_lag=0, temp_twice=False) -> dict:
    """Every sampling decision of one event restated: row b live, step i < n_steps, drawn from logits [n_steps, B, V] (the
    step's bf16 logits as fp32) in the grammar range of step i under ev_t[0][b] (the kernel's own step-0 tokens), with
    the row's settings[b] = (temp, top_p, top_k), mask row masks[b] (or None) and uniform u[i, b].  Returns arrays
    [n_steps, B]: "id" (-1 where no decision), "amb" (logits_sample's ambiguity), "cut" (top-p removed a top-k
    candidate), "tie" (two of the top k + 1 candidates have the same bf16 probability).  `temp_twice` divides by the
    temperature twice; `range_lag` draws in the range of an earlier step."""
    n, B = n_steps, len(live)
    out = {"id": np.full((n, B), -1, np.int64), "amb": np.zeros((n, B), bool), "cut": np.zeros((n, B), bool),
           "tie": np.zeros((n, B), bool)}
    for b in range(B):
        if not live[b]:
            continue
        temp, top_p, top_k = settings[b]
        mrow = None if masks is None else masks[b]
        for i in range(n):
            lo, hi = grammar_range(i, int(ev_t[0][b]), lut, eos, pad, n_event_types, lag=range_lag)
            l = np.asarray(logits[i][b], dtype=F32)
            if temp_twice and temp != 1.0:
                l = bf16_np(l / F32(temp))
            out["id"][i, b], out["amb"][i, b] = logits_sample(l, temp, top_p, top_k, lo, hi, mrow, float(u[i, b]))
            _, _, pb = _logits_probs(l, temp, lo, hi, mrow)
            cand = np.nonzero(pb > 0)[0]
            if cand.size == 0:
                continue
            p = np.sort(pb[cand])[::-1]
            kk = min(cand.size, max(1, top_k))
            before = bf16_np(bf16_np(np.cumsum(p[:kk], dtype=F32)) - p[:kk])
            out["cut"][i, b] = bool((before > _bf16s(top_p)).any())
            out["tie"][i, b] = bool(np.unique(p[:kk + 1]).size < p[:kk + 1].size)
    return out


def event_commit_rows(ev_t, n_steps: int, live, seq, ev_in, pos: int, row_off, pad: int, *, commit_all=False):
    """The commit of decode_events_kernel: row b's tokens are ev_t[t][b] for t < n_steps and pad after; a live row writes
    them to seq[b, pos + row_off[b] + 1] and ev_in[b], a row that is not live writes nothing.  Returns (tokens [B, PD_T],
    seq, ev_in).  `commit_all` lets the rows that are not live commit."""
    B = len(live)
    tok = np.full((B, PD_T), pad, dtype=np.int64)
    tok[:, :n_steps] = np.asarray(ev_t)[:n_steps].T
    seq, ev_in = np.array(seq, copy=True), np.array(ev_in, copy=True)
    for b in range(B):
        if live[b] or commit_all:
            seq[b, pos + int(row_off[b]) + 1] = tok[b]
            ev_in[b] = tok[b]
    return tok, seq, ev_in


def decode_ws_layout(batch: int, H: int, I_outer: int, I_inner: int, pitch: int, nh_outer: int, n_inner: int) -> dict:
    """decode_persist.cu:ws_layout restated: byte offset of each region of the persistent kernel's workspace, and "total".
    Each region starts on a 256-byte boundary; x / h / x2 / h2 / attn are [B, H] bf16, qkv [B, 3H], act [B, max(I)],
    logits [B, pitch], ev_t [PD_T, B] int64, partial [B nh_outer, PD_MAXC, 66] fp32, k2 / v2 [n_inner, B, PD_T, H]."""
    L, o = {}, 0
    B = batch
    for name, nbytes in (("bar", 256), ("x", B * H * 2), ("h", B * H * 2), ("x2", B * H * 2), ("h2", B * H * 2),
                         ("qkv", B * 3 * H * 2), ("attn", B * H * 2), ("act", B * max(I_outer, I_inner) * 2),
                         ("logits", B * pitch * 2), ("ev_t", PD_T * B * 8), ("partial", B * nh_outer * PD_MAXC * 66 * 4),
                         ("k2", n_inner * B * PD_T * H * 2), ("v2", n_inner * B * PD_T * H * 2)):
        L[name] = o
        o = (o + nbytes + 255) // 256 * 256
    L["total"] = o
    return L


# ------------------------------------------------------------------------------------------ paged KV
def slot_mask(pool_shape, block_table: torch.Tensor, page: int, rows_pos) -> torch.Tensor:
    """Boolean mask over a [n_pages, n_heads, page, D] pool of the slots of (batch row, position) pairs `rows_pos`."""
    m = torch.zeros(pool_shape, dtype=torch.bool, device=block_table.device)
    if len(rows_pos):
        b, t = (torch.tensor(c, dtype=torch.long, device=block_table.device) for c in zip(*rows_pos))
        m[block_table.long()[b, t // page], :, t % page] = True
    return m


def gather_kv(pool: torch.Tensor, block_table: torch.Tensor, page: int, b: int, T: int) -> torch.Tensor:
    """Positions 0 .. T-1 of batch row b, read through the block table: [n_heads, T, D] (pool dtype)."""
    t = torch.arange(T, device=pool.device)
    pg = block_table[b].long()[t // page]
    return pool[pg, :, t % page].transpose(0, 1)


def paged_attention64(q: torch.Tensor, k_pool, v_pool, block_table, page: int, b: int, T: int, scale: float):
    """fp64 attention of q [n_heads, Sq, D] over positions 0 .. T-1 of row b, query i seeing keys <= T - Sq + i."""
    k = gather_kv(k_pool, block_table, page, b, T).double()
    v = gather_kv(v_pool, block_table, page, b, T).double()
    Sq = q.shape[1]
    s = (q.double() @ k.transpose(-1, -2)) * scale
    off = T - Sq
    m = torch.arange(T, device=q.device)[None] > (torch.arange(Sq, device=q.device)[:, None] + off)
    return torch.softmax(s.masked_fill(m, float("-inf")), -1) @ v
