"""The conformance metrics of tests/parity_metrics.py, judged by the bounds the GPU groups use (the tables of
gpu_checks.GROUPS), on the CPU: each corruption a kernel could plausibly make fails, while the same references
recomputed in fp32 with another summation order (and rounded to bf16 as a kernel would) pass.  Also the bound check
itself, and the bound tables of every GPU test."""
import importlib
import math

import pytest
import torch

import gpu_checks as G
import parity_metrics as P

BF = torch.bfloat16


def _fails(group, metrics):
    res = P.check_bounds(metrics, G.GROUPS[group].bounds)
    assert all(b is not None for _, _, b, _ in res), res
    return any(not ok for *_, ok in res)


# ------------------------------------------------------------------------------------------ the bound check
def _oks(metrics, bounds, info=()):
    return {k: ok for k, _, _, ok in P.check_bounds(metrics, bounds, info)}


def test_check_bounds_rules():
    bounds = [("a_long", 1.0), ("a", 2.0), ("min:c", 3.0)]
    res = P.check_bounds({"a_long_x": 1.5, "a_x": 1.5, "c": 3.0, "c_low": 2.9, "nan": math.nan, "t": 9.0},
                         bounds, info=("t",))
    assert res == [("a_long_x", 1.5, 1.0, False),      # the longer prefix, placed first, wins
                   ("a_x", 1.5, 2.0, True),
                   ("c", 3.0, 3.0, True),              # min: a lower bound
                   ("c_low", 2.9, 3.0, False),
                   ("nan", math.nan, None, False),     # matches no bound and is not informational
                   ("t", 9.0, None, True)]             # informational: reported with bound None
    assert _oks({"a": math.nan, "a_inf": math.inf}, bounds) == {"a": False, "a_inf": False}
    assert _oks({"a": 2.0, "c": math.inf}, bounds) == {"a": True, "c": True}


def test_renamed_metric_of_a_group_fails():
    """A metric whose name matches no bound of its group fails instead of dropping out of the check."""
    g = G.GROUPS["model_train"]
    good = {"loss_abs": 1e-3, "loss_ref": 8.0, "grad_global_rel": 1e-2, "grad_worst_rel": 3e-2}
    assert all(_oks(good, g.bounds, g.info).values())
    renamed = {("los_abs" if k == "loss_abs" else k): v for k, v in good.items()}
    assert _oks(renamed, g.bounds, g.info) == {"los_abs": False, "loss_ref": True, "grad_global_rel": True,
                                                "grad_worst_rel": True}


def _bound_tables():
    for name, g in G.GROUPS.items():
        yield name, g.bounds, g.info
    for mod in ("test_gpu_ragged", "test_gpu_recompute", "test_gpu_sample_seq"):
        yield mod, importlib.import_module(mod).BOUNDS, ()


def test_bound_tables_have_no_dead_or_doubled_entries():
    """No entry sits behind an earlier prefix of itself (it could never match), and no informational metric also has
    a bound."""
    problems = []
    for name, bounds, info in _bound_tables():
        prefixes = [p.removeprefix("min:") for p, _ in bounds]
        problems += [(name, "shadowed", b, a) for i, b in enumerate(prefixes) for a in prefixes[:i] if b.startswith(a)]
        problems += [(name, "bounded and informational", n) for n in info if any(n.startswith(p) for p in prefixes)]
    assert not problems, problems


# ------------------------------------------------------------------------------------------ attention rows


def _randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _attn32_reordered(q, k, v):
    """fp32 causal attention with the keys summed in reverse order."""
    q, k, v = q.float(), k.float(), v.float()
    S = q.shape[-2]
    s = (q @ k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool), 1), float("-inf"))
    p = torch.softmax(s, -1)
    return p.flip(-1) @ v.flip(-2)


@pytest.fixture(scope="module")
def attn_ref():
    # eight heads at S = 2047: the last 64-row tile is ragged (63 rows)
    q, k, v, do = (_randn(1, 8, 2047, 64, seed=i) for i in range(4))
    o64, _, dq64, _, _ = P.attn_ref64(q, k, v, do, 0, 0.125)
    return q, k, v, o64, dq64


def test_attention_rows_pass_when_only_rounding_differs(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    o32 = _attn32_reordered(q, k, v)
    assert not _fails("attn_edges", {"ae_wg_o_row": P.row_worst(o32, o64),
                                     "ae_wg_dq_row": P.row_worst(dq64.float(), dq64)})
    # bf16 outputs, as the kernels store them
    assert not _fails("attn_edges", {"ae_wg_o_row": P.row_worst(o32.to(BF), o64),
                                     "ae_wg_dq_row": P.row_worst(dq64.to(BF), dq64)})


def test_attention_zeroed_last_row_of_ragged_tile_fails(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    y = _attn32_reordered(q, k, v).to(BF)
    y[0, 1, 2046] = 0          # the last row of the ragged tile, one head
    # a global relative norm barely moves ...
    glob = float((y.double() - o64).norm() / o64.norm())
    assert glob < 6e-3
    # ... the per-row score does not
    assert _fails("attn_edges", {"ae_wg_o_row": P.row_worst(y, o64)})
    g = dq64.to(BF)
    g[0, 0, 2046] = 0
    assert _fails("attn_edges", {"ae_wg_dq_row": P.row_worst(g, dq64)})


def test_attention_nan_fails(attn_ref):
    q, k, v, o64, dq64 = attn_ref
    y = o64.to(BF)
    y[0, 0, 1000, 7] = float("nan")
    assert P.row_worst(y, o64) == math.inf
    assert _fails("attn_edges", {"ae_wg_o_row": P.row_worst(y, o64)})


def test_zero_reference_rows_use_the_input_scale_floor():
    ref = torch.zeros(2, 4, 64, dtype=torch.float64)
    noise = torch.full_like(ref, 1e-7)
    assert P.row_worst(noise, ref, atol=8e-3) < 1e-4
    assert P.row_worst(noise + 1.0, ref, atol=8e-3) > 1.0


@pytest.fixture(scope="module")
def gemm_ref():
    a = _randn(257, 300, seed=10).to(BF)
    b = (_randn(520, 300, seed=11) * 0.05).to(BF)
    return a, b, a.double() @ b.double().T


def _gm(y, ref, family="store", **kw):
    return {f"gm_{family}_{k}": v for k, v in P.exact_metrics(y, ref, **kw).items()}


def test_gemm_reordered_fp32_passes(gemm_ref):
    a, b, ref = gemm_ref
    y = (a.float().flip(1) @ b.float().flip(1).T).to(BF)
    m = _gm(y, ref)
    assert m["gm_store_maxulp"] <= 1 and not _fails("gemm_matrix", m)


def test_gemm_group_moved_by_4_ulp_fails(gemm_ref):
    a, b, ref = gemm_ref
    y = (a.float() @ b.float().T).to(BF)
    # an 8-column group whose references are all well above the noise floor
    rms = float(ref.pow(2).mean().sqrt())
    big = (ref.abs() > 0.5 * rms).view(257, -1, 8).all(-1)
    r, g = (int(i) for i in torch.nonzero(big)[0])
    bits = y.view(torch.int16)
    bits[r, 8 * g:8 * g + 8] += 4          # 4 ulp away from zero (sign-magnitude bits)
    m = _gm(y, ref)
    assert m["gm_store_maxulp"] >= 4
    assert _fails("gemm_matrix", m)


def test_chained_epilogue_flip_passes_but_3_ulp_fails(gemm_ref):
    a, b, ref = gemm_ref
    r = (_randn(257, 520, seed=12)).to(BF)
    acc = P.round_bf16(ref)
    want = (acc + r.double()).float().to(BF)
    y = ((a.float().flip(1) @ b.float().flip(1).T).to(BF).float() + r.float()).to(BF)
    m = _gm(y, acc + r.double(), "residual", want=want, inter=ref)
    assert not _fails("gemm_matrix", m)
    y.view(torch.int16)[5, 16:24] += 3
    assert _fails("gemm_matrix", _gm(y, acc + r.double(), "residual", want=want, inter=ref))


def test_gemm_nan_fails(gemm_ref):
    a, b, ref = gemm_ref
    y = ref.to(BF)
    y[100, 200] = float("nan")
    assert _fails("gemm_matrix", _gm(y, ref))


def test_sentinels():
    M, N, ldc = 5, 13, 32
    buf = P.nan_buffer((M + 3, ldc))
    buf[:M, :N] = 1.0
    buf[:M, N:16] = 0.0
    inside, pad = (slice(0, M), slice(0, N)), (slice(0, M), slice(N, 16))
    rep = P.sentinel_report(buf, inside, pad)
    assert rep == {"sentinels_changed": 0.0, "nan_in_range": 0.0, "padcols_nonzero": 0.0}
    assert not _fails("gemm_matrix", {f"gm_{k}": v for k, v in rep.items()})
    # one sentinel overwritten (a store past the row, or into the next row's pitch)
    bad = buf.clone()
    bad[M, 0] = 0.0
    assert P.sentinel_report(bad, inside, pad)["sentinels_changed"] == 1
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})
    # one output never written
    bad = buf.clone()
    bad[M - 1, N - 1] = float("nan")
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})
    # a padding column not zeroed
    bad = buf.clone()
    bad[0, 15] = float("nan")
    assert _fails("gemm_matrix", {f"gm_{k}": v for k, v in P.sentinel_report(bad, inside, pad).items()})


def test_poisoned_operand_keeps_values_and_pads_with_nan():
    v = _randn(3, 5, seed=1).to(BF)
    t = P.poisoned(v, 4, 8)
    assert torch.equal(t[:3, :5], v)
    assert bool(torch.isnan(t[:3, 5:].float()).all()) and bool(torch.isnan(t[3].float()).all())
