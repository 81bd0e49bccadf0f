"""Exact restatements of the generate-path kernels that are not a product of bf16 operands: the samplers
(csrc/sampler.cuh), the counter-based RNG and the event commit (csrc/decode.cu), plus an fp64 paged-KV attention that reads
keys through the block table.  NumPy / PyTorch on the CPU, so tests/test_decode_reference.py can show that each one, and
the case sets the decode conformance groups of gpu_checks.py feed it, catches the defects a kernel could plausibly have.

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


def logits_sample(l, temp: float, top_p: float, top_k: int, lo: int, hi: int, mask, u: float,
                  rel_tol: float = 2.0 ** -17):
    """b200_sample_from_logits for one row restated from fp64 probabilities rounded to bf16.  Returns (id, ambiguous).

    x = bf16(l / temp) (fp32 division), p = bf16(exp(x - max) / sum over the whole vocabulary), ids outside [lo, hi) or
    masked out are not candidates, then the sampler tail.  The kernel's p comes from __expf and an fp32 sum, which can
    sit about one fp32 ulp per unit of |x - max| from the fp64 value; where a candidate that could reach the top k lies
    within rel_tol of a bf16 rounding midpoint, its bf16 p (and so the id) is not determined and the row is ambiguous.
    With every such p determined, the tail is exact fp32 arithmetic on the same values, so u * total needs no margin.
    No candidate (every allowed p rounds to 0): the kernel returns lo."""
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
    pb = bf16_np(p64.astype(F32))
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
