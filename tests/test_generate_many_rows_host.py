"""Per-request mode of the request queue (`generate_many_requests`, and `generate_many` with per-request settings): the host
side -- each slot's settings, RNG key and mask row written at admission, the `_rows` entries issued, the scalar call left
as it was, input checks -- over the CPU stand-in for the kernel layer (tests/mock_kernels.py), on the host-issued loop
(B200_GENERATE=nograph) and on the persistent kernel's launch protocol.  The kernels themselves are checked on the GPU
(tests/test_gpu_generate_many_rows.py)."""
import inspect

import numpy as np
import pytest
import torch

import host_model
import mock_decode
import mock_kernels
from decode_reference import counter_uniform

LENGTHS, BUDGETS = [5, 2, 9, 3, 7, 4, 1], [6, 4, 4, 8, 5, 5, 4]      # >= 4: generate runs its device loop
TEMPS, TOP_PS, TOP_KS = [1.3, 0.7, 1.0, 1.0, 0.9, 1.2, 1.0], [0.9, 1.0, 0.5, 0.98, 1.0, 0.8, 1.0], [64, 5, 20, 1, 3, 8, 2]
SEEDS = [11, 2 ** 62 - 1, 0, 7, 123456789, 99, 5]
PATCH = [True, False, False, True, False, False, False]
CHANNELS = [None, [0, 9], None, [3], None, None, list(range(16))]


def test_generate_many_requests_signature():
    import midi_model as mm
    params = inspect.signature(mm.MIDIModel.generate_many_requests).parameters
    assert list(params)[1:] == ["prompts", "max_new", "batch_size", "temp", "top_p", "top_k", "generator",
                                "disable_patch_change", "disable_control_change", "disable_channels", "seeds"]
    assert [params[k].default for k in list(params)[3:]] == [8, 1.0, 0.98, 20, None, False, False, None, None]
    assert all(params[k].kind is inspect.Parameter.KEYWORD_ONLY for k in list(params)[8:])


@pytest.fixture(params=["nograph", "persist"])
def model(request, monkeypatch):
    return host_model.generate_model(monkeypatch, request.param)


def _deny(model, i):
    return sorted(model._deny_ids(PATCH[i], False, CHANNELS[i]))


def _kwargs(order):
    return dict(temp=[TEMPS[i] for i in order], top_p=[TOP_PS[i] for i in order], top_k=[TOP_KS[i] for i in order],
                seeds=[SEEDS[i] for i in order], disable_patch_change=[PATCH[i] for i in order],
                disable_channels=[CHANNELS[i] for i in order])


def _solo(model, p, n, i):
    """Request i alone: generate at batch 1 with its settings and a generator whose first draw is SEEDS[i] (greedy mock
    layer: its own loop, nograph)."""
    from midi_b200 import decode
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200_GENERATE", "nograph")
        g = torch.Generator()
        orig = torch.randint
        mp.setattr(torch, "randint", lambda lo, hi, size, generator=None, device=None:
                   torch.tensor([SEEDS[i]]) if generator is g else orig(lo, hi, size, generator=generator, device=device))
        deny = _deny(model, i)
        mp.setattr(decode.GraphGenerator, "set_deny", lambda self, ids, _f=decode.GraphGenerator.set_deny: _f(self, deny))
        return model.generate(prompt=p, batch_size=1, max_len=p.shape[0] + n, temp=TEMPS[i], top_p=TOP_PS[i],
                              top_k=TOP_KS[i], generator=g)[0]


@pytest.mark.parametrize("batch_size", [1, 2, 3, 8])
def test_every_draw_is_the_requests_own(model, batch_size):
    """Each sampler call of request i gets hash(seeds[i], 8 j + t, 0), its own settings and its own mask row, whatever
    slot holds it; the same request set permuted gives each request the same events."""
    prompts = host_model.prompts(model, LENGTHS, seed=21)
    order = list(range(len(prompts)))
    got = model.generate_many_requests(prompts, BUDGETS, batch_size=batch_size, **_kwargs(order))
    by_seed = {SEEDS[i]: i for i in order}
    seen = {i: set() for i in order}
    n_new = [got[i].shape[0] - LENGTHS[i] for i in order]
    for d in mock_decode.DRAWS:
        i = by_seed.get(d["seed"])
        if i is None or not 0 <= d["j"] < n_new[i]:
            continue                                               # an empty slot's row: its draw is never committed
        assert d["u"] == counter_uniform(SEEDS[i], 8 * d["j"] + d["step"], 0), d
        assert (d["temp"], d["top_k"]) == (np.float32(TEMPS[i]), TOP_KS[i]) and d["top_p"] == np.float32(TOP_PS[i]), d
        assert d["deny"] == _deny(model, i), d
        seen[i].add((d["j"], d["step"]))
    for i in order:
        assert {(j, t) for j in range(n_new[i]) for t in (0, 1)} <= seen[i], i
    perm = [3, 6, 0, 5, 1, 4, 2]
    again = model.generate_many_requests([prompts[i] for i in perm], [BUDGETS[i] for i in perm], batch_size=batch_size,
                                **_kwargs(perm))
    for k, i in enumerate(perm):
        assert again[k].shape == got[i].shape and (again[k] == got[i]).all(), i


def test_one_slot_equals_generate_seeded_as_specified(model):
    prompts = host_model.prompts(model, LENGTHS, seed=22)
    order = list(range(len(prompts)))
    got = model.generate_many_requests(prompts, BUDGETS, batch_size=1, **_kwargs(order))
    for i, (p, n) in enumerate(zip(prompts, BUDGETS)):
        solo = _solo(model, p, n, i)
        assert got[i].shape == solo.shape and (got[i] == solo).all(), i
    sampled = [i for i in order if TOP_KS[i] > 1 and got[i].shape[0] > LENGTHS[i] + 1]
    assert len(sampled) >= 3


def test_greedy_requests_in_a_mixed_queue_equal_generating_alone(model):
    prompts = host_model.prompts(model, LENGTHS, seed=23)
    top_k = [1 if i % 2 == 0 else 20 for i in range(len(prompts))]
    got = model.generate_many(prompts, BUDGETS, batch_size=3, top_k=top_k, temp=1.3, top_p=0.9)   # per-request top_k
    for i in range(0, len(prompts), 2):
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200_GENERATE", "nograph")
            solo = model.generate(prompt=prompts[i], batch_size=1, max_len=LENGTHS[i] + BUDGETS[i], top_k=1)[0]
        assert got[i].shape == solo.shape and (got[i] == solo).all(), i


def test_scalar_call_issues_no_rows_entry(model, monkeypatch):
    """Scalar settings without seeds keep the scalar queue: the same kernel calls, none of the `_rows` entries, and scalar
    grammar options only in every row's mask."""
    prompts = host_model.prompts(model, [4, 2, 6], seed=24)
    model.generate_many_requests(prompts[:1], 1, top_k=1)                     # runtime set-up outside the trace
    def trace(**kw):
        with pytest.MonkeyPatch.context() as mp:
            return mock_kernels.trace(mp, lambda: model.generate_many_requests(prompts, [3, 2, 4], batch_size=2, top_k=1, **kw))

    plain = trace()
    assert plain and plain == trace(disable_patch_change=True, disable_channels=[2, 3])
    assert not [n for n in plain if n.endswith("_rows")]
    assert [n for n in trace(seeds=[1, 2, 3]) if n.endswith("_rows")]


def test_per_request_input_errors_raise(model):
    from midi_b200.lib import B200Error
    good = host_model.prompts(model, [3, 4], seed=25)
    bad = [dict(temp=[1.0]), dict(temp=[1.0, 0.0]), dict(temp=[1.0, -1.0]), dict(temp=[1.0, float("nan")]),
           dict(top_p=[0.9, 0.0]), dict(top_p=[0.9, 1.5]), dict(top_k=[1, 0]), dict(top_k=[1, 2.5]), dict(top_k=[1, 2, 3]),
           dict(seeds=[1]), dict(seeds=[1, 2, 3]), dict(seeds=[1, -1]), dict(seeds=[1, 2 ** 62]), dict(seeds=[1, 2.0]),
           dict(seeds=[1, True]), dict(seeds=5), dict(disable_patch_change=[True]), dict(disable_control_change=[1, 2, 3]),
           dict(disable_channels=[16]), dict(disable_channels=[-1]), dict(disable_channels=[None, [16]]),
           dict(disable_channels=[[1], None, None]), dict(disable_channels=[1, None]), dict(disable_channels=[[1], 2]),
           dict(disable_channels=3), dict(disable_channels=[[True], None])]
    for kw in bad:
        with pytest.raises(B200Error):
            model.generate_many_requests(good, 2, **{"top_k": 1, **kw})
    got = model.generate_many_requests(good, 2, top_k=[1, 1], disable_channels=[None, []], seeds=np.array([3, 4]))
    assert len(got) == 2
