"""Request queue (`generate_many`): the host scheduler -- admission with a batch-1 prefill into a slot, the rebase of the
shared counter, per-row stop, refill and output order -- over the CPU stand-in for the kernel layer (tests/mock_kernels.py),
on the host-issued loop (B200_GENERATE=nograph) and on the persistent kernel's launch protocol.  The kernels themselves
are checked on the GPU (tests/test_gpu_generate_many.py)."""
import inspect

import numpy as np
import pytest
import torch

import host_model


def test_generate_many_signature():
    import midi_model as mm
    params = inspect.signature(mm.MIDIModel.generate_many).parameters
    assert list(params)[1:] == ["prompts", "max_new", "batch_size", "temp", "top_p", "top_k", "generator"]
    assert [params[k].default for k in list(params)[3:]] == [8, 1.0, 0.98, 20, None]


@pytest.fixture(params=["nograph", "persist"])
def model(request, monkeypatch):
    return host_model.generate_model(monkeypatch, request.param)


def _bos(model):
    tok = model.tokenizer
    p = np.full((1, tok.max_token_seq), tok.pad_id, dtype=np.int64)
    p[0, 0] = tok.bos_id
    return p


def _check_solo(model, prompts, budgets, got):
    """Request i against generating its prompt alone at batch 1 with max_len = L_i + max_new_i (greedy)."""
    assert isinstance(got, list) and len(got) == len(prompts)
    eos = model.tokenizer.eos_id
    for i, (p, n) in enumerate(zip(prompts, budgets)):
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200_GENERATE", "nograph")                  # the mock layer has no rectangular persistent kernel
            solo = model.generate(prompt=p, batch_size=1, max_len=p.shape[0] + n, top_k=1)[0]
        assert got[i].dtype == np.int64 and got[i].shape == solo.shape, (i, got[i].shape, solo.shape)
        assert (got[i] == solo).all(), i
        k = got[i].shape[0] - p.shape[0]
        assert 1 <= k <= n and (k == n or got[i][-1, 0] == eos), (i, k, n)


def test_more_requests_than_slots_with_mixed_budgets(model):
    lengths, budgets = [5, 2, 9, 3, 7, 4, 2], [6, 1, 3, 8, 2, 5, 4]
    prompts = host_model.prompts(model, lengths, seed=11)
    got = model.generate_many(prompts, budgets, batch_size=3, top_k=1)
    _check_solo(model, prompts, budgets, got)


def test_fewer_requests_than_slots_and_one_request(model):
    prompts = host_model.prompts(model, [4, 6], seed=12)
    _check_solo(model, prompts, [5, 3], model.generate_many(prompts, [5, 3], batch_size=8, top_k=1))
    one = prompts[:1]
    _check_solo(model, one, [4], model.generate_many(one, 4, batch_size=1, top_k=1))


def test_one_new_event_and_bos_only_prompts(model):
    prompts = [_bos(model)] + host_model.prompts(model, [3, 5], seed=13) + [_bos(model)]
    _check_solo(model, prompts, [1] * 4, model.generate_many(prompts, 1, batch_size=2, top_k=1))
    _check_solo(model, prompts, [5, 2, 1, 3], model.generate_many(prompts, [5, 2, 1, 3], batch_size=2, top_k=1))


def test_request_filling_the_pools(model):
    """L + max_new = 64 = the capacity of one 64-position page: the longest request uses its last KV slot."""
    prompts = host_model.prompts(model, [52, 3, 6], seed=14)
    budgets = [12, 4, 2]
    from midi_b200 import decode
    seen = []
    orig = decode.GraphGenerator.run_queue

    def spy(self, *a, **k):
        seen.append((self.max_len, self.kv1.capacity))
        return orig(self, *a, **k)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(decode.GraphGenerator, "run_queue", spy)
        got = model.generate_many(prompts, budgets, batch_size=2, top_k=1)
    assert seen == [(64, 64)]
    _check_solo(model, prompts, budgets, got)


def test_one_batch1_prefill_per_request_in_input_order(model, monkeypatch):
    """Every request's prompt is prefilled once, alone, into one slot's pages; a one-event prompt prefills nothing."""
    from midi_b200 import decode
    prefills = []
    orig = decode.CachedStack.step

    def spy(self, x, kv, s_new, pos_dev=None, *a, **k):
        if pos_dev is None and self is model._b200_rt.cached_outer:
            prefills.append((kv.batch, s_new))
        return orig(self, x, kv, s_new, pos_dev, *a, **k)

    lengths = [4, 7, 2, 5, 3]
    prompts = host_model.prompts(model, lengths, seed=15)
    model.generate_many(prompts[:1], 1, top_k=1)                    # runtime set-up outside the count
    monkeypatch.setattr(decode.CachedStack, "step", spy)
    model.generate_many(prompts, [3, 1, 4, 2, 2], batch_size=2, top_k=1)
    assert prefills == [(1, L - 1) for L in lengths]
    prefills.clear()
    model.generate_many([_bos(model), _bos(model)], 2, batch_size=2, top_k=1)
    assert prefills == []


def test_input_errors_raise(model, monkeypatch):
    from midi_b200.lib import B200Error
    good = host_model.prompts(model, [3, 4], seed=16)
    bad_prompts = [[], (), "ab", [good[0][:0]], [good[0][0]], [good[0][None]], [good[0].astype(np.float32)],
                   [torch.from_numpy(good[0]).to("meta")], [None], good[0]]
    for prompts in bad_prompts:
        with pytest.raises(B200Error):
            model.generate_many(prompts, 2, top_k=1)
    for max_new in [0, -1, [2], [2, 0], [2, 2, 2], 2.0, [2.0, 1], True, torch.tensor([[1, 2]])]:
        with pytest.raises(B200Error):
            model.generate_many(good, max_new, top_k=1)
    for batch_size in [0, -2, 1.5, None]:
        with pytest.raises(B200Error):
            model.generate_many(good, 2, batch_size=batch_size, top_k=1)
    monkeypatch.setenv("B200_GENERATE", "eager")
    with pytest.raises(B200Error):
        model.generate_many(good, 2, top_k=1)


def test_cpu_tensor_prompts_and_budgets(model):
    prompts = host_model.prompts(model, [3, 6, 2], seed=17)
    ref = model.generate_many(prompts, [2, 3, 4], batch_size=2, top_k=1)
    got = model.generate_many([torch.from_numpy(p) for p in prompts], torch.tensor([2, 3, 4]), batch_size=2, top_k=1)
    assert all((a == b).all() and a.shape == b.shape for a, b in zip(ref, got))
