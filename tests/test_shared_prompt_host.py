"""Shared prompts in the request queue (`generate_many`, `generate_many_requests`): requests with equal prompts of at least
65 events prefill once and read the prompt's whole pages from the same KV pages (decode.SharedPages).  Over the CPU
stand-in for the kernel layer (tests/mock_kernels.py), on the host-issued loop and on the persistent kernel's launch
protocol, greedy and per-request sampled.  Every call is compared with the same call with sharing off, and spies check
the page assignment at every launch."""
import numpy as np
import pytest
import torch

import host_model
import mock_kernels

LAUNCHES = ("b200_event_commit_queue", "b200_decode_events_queue", "b200_decode_events_queue_rows")


@pytest.fixture(params=["nograph", "persist"])
def model(request, monkeypatch):
    return host_model.generate_model(monkeypatch, request.param)


class Spy:
    """Checks every launch's block table, counts the outer prefills and the launch names, and keeps the generator and the
    SharedPages (None: the call shared nothing) of the last call."""

    def __init__(self, model, mp):
        from midi_b200 import decode, lib
        self.prefills, self.launches, self.shared_launches, self.gg, self.pages = [], 0, 0, None, None
        self.names = []
        run_queue, step, call = decode.GraphGenerator.run_queue, decode.CachedStack.step, lib.call
        pages_init = decode.SharedPages.__init__

        def spy_pages(pages, *a, **k):
            pages_init(pages, *a, **k)
            self.pages = pages

        def spy_run_queue(gg, *a, **k):
            self.gg = gg
            return run_queue(gg, *a, **k)

        def spy_step(stack, x, kv, s_new, pos_dev=None, *a, **k):
            if pos_dev is None and stack is model._b200_rt.cached_outer:
                self.prefills.append(s_new + 1)
            return step(stack, x, kv, s_new, pos_dev, *a, **k)

        def spy_call(name, *a):
            if name in LAUNCHES:
                self.names.append(name)
                self.check(self.gg)
            return call(name, *a)

        mp.setattr(decode.GraphGenerator, "run_queue", spy_run_queue)
        mp.setattr(decode.CachedStack, "step", spy_step)
        mp.setattr(lib, "call", spy_call)
        mp.setattr(decode.SharedPages, "__init__", spy_pages)

    def check(self, gg):
        self.launches += 1
        table = gg.kv1.block_table.tolist()
        last = gg.row_last.tolist()
        pages = self.pages
        if pages is None:                                   # no shared prompt: the identity table
            assert table == torch.arange(gg.B * gg.kv1.max_pages).view(gg.B, -1).tolist()
            return
        page = gg.kv1.page
        live = [b for b in range(gg.B) if last[b] == -1]
        owner, lead = {}, {}
        for b in live:
            k, S = pages.key[b], pages.shared[b]
            n_sh = S // page
            assert (k is None) == (S == 0) and S % page == 0
            if k is not None and k in lead:                 # a sharer: the same pages below S as its group's first row
                assert table[b][:n_sh] == table[lead[k]][:n_sh], (b, lead[k])
                self.shared_launches += 1
                own = table[b][n_sh:]
            else:
                lead.setdefault(k, b)
                own = table[b]
            for p in own:                                   # no other page is held by two live rows
                assert p not in owner or owner[p] == b, (p, b, owner.get(p))
                owner[p] = b
            assert len(set(own)) == len(own)
        for b in range(gg.B):
            if last[b] == -2:                               # an empty slot: one page of its own, no live row's
                assert len(set(table[b])) == 1 and table[b][0] not in owner, (b, table[b])


def _run(model, prompts, budgets, batch_size, sampled, share=True):
    from midi_b200 import decode
    with pytest.MonkeyPatch.context() as mp:
        if not share:
            mp.setattr(decode, "_share_keys", lambda prompts, page: [None] * len(prompts))
        spy = Spy(model, mp)
        if sampled:
            n = len(prompts)
            got = model.generate_many_requests(prompts, budgets, batch_size=batch_size, temp=1.2, top_p=0.95,
                                               top_k=[5] * n, seeds=[101 + 7 * i for i in range(n)])
        else:
            got = model.generate_many(prompts, budgets, batch_size=batch_size, top_k=1)
    gg, pages = spy.gg, spy.pages
    if pages is not None:                                   # every page is free at the end of the call
        assert sorted(pages.free) == list(range(pages.n_pages)) and not pages.groups
    assert share or pages is None
    assert gg.kv1.block_table.tolist() == torch.arange(gg.B * gg.kv1.max_pages).view(gg.B, -1).tolist()
    return got, spy


def _same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and (x == y).all(), i


def _check(model, prompts, budgets, batch_size, sampled):
    """The call with and without sharing: equal results; returns the sharing call's spy."""
    got, spy = _run(model, prompts, budgets, batch_size, sampled)
    off, spy_off = _run(model, prompts, budgets, batch_size, sampled, share=False)
    _same(got, off)
    assert spy_off.prefills == [p.shape[0] for p in prompts if p.shape[0] > 1]
    assert spy.launches > 0 and spy_off.launches > 0
    return got, spy


@pytest.mark.parametrize("sampled", [False, True])
def test_duplicates_admitted_together(model, sampled):
    a, c = host_model.prompts(model, [70, 90], seed=31)
    prompts = [a, a, c, a]
    got, spy = _check(model, prompts, [5, 3, 4, 6], 4, sampled)
    assert sorted(spy.prefills) == [70, 90]                 # one prefill of the shared prompt
    assert spy.shared_launches > 0


@pytest.mark.parametrize("sampled", [False, True])
def test_duplicates_admitted_apart_and_finishing_at_different_events(model, sampled):
    """Two slots: the second copy of `a` joins the first while it is live, at its own position; the later copies join the
    second; after the last sharer finishes, `a` is prefilled again."""
    a, c, d, e = host_model.prompts(model, [80, 66, 75, 68], seed=32)
    prompts = [a, c, a, a, d, a, e]
    budgets = [9, 2, 3, 8, 9, 1, 2]
    got, spy = _check(model, prompts, budgets, 2, sampled)
    assert spy.prefills.count(80) < 4
    assert spy.shared_launches > 0


@pytest.mark.parametrize("L", [64, 65, 66, 129])
def test_page_boundaries(model, L):
    """L - 1 = 63 shares nothing (no whole page).  L - 1 = 64 and 128 share one and two pages, and their tail pages hold no
    prompt position; L - 1 = 65 shares one page and copies a tail page holding one prompt position."""
    a, c = host_model.prompts(model, [L, 67], seed=33)
    prompts = [a, c, a, a]
    got, spy = _check(model, prompts, [4, 2, 5, 3], 3, False)
    if L - 1 < 64:
        assert spy.prefills.count(L) == 3 and spy.shared_launches == 0
    else:
        assert spy.prefills.count(L) == 1 and spy.shared_launches > 0


@pytest.mark.parametrize("sampled", [False, True])
def test_empty_slot_while_sharers_are_live(model, sampled):
    """The distinct request finishes first and no request waits: its slot stays empty (and, on the host-issued loop, keeps
    appending) while the sharers run on."""
    a, c = host_model.prompts(model, [72, 5], seed=34)
    got, spy = _check(model, [a, c, a], [7, 1, 6], 3, sampled)
    assert spy.shared_launches > 0


@pytest.mark.parametrize("sampled", [False, True])
def test_refilled_slot_prefills_beside_shared_pages(model, sampled):
    """Slot 1 is refilled with distinct prompts while the sharers of `a` are live: their prefills go to free pages."""
    a, c, d, e = host_model.prompts(model, [100, 3, 70, 90], seed=35)
    got, spy = _check(model, [a, c, d, a, e], [10, 1, 2, 9, 2], 3, sampled)
    assert spy.prefills.count(100) == 1 and spy.shared_launches > 0


def test_call_without_a_shared_prompt_keeps_its_trace(model):
    """No shareable duplicate (distinct prompts, or equal ones of fewer than 65 events): no SharedPages is made, every
    launch sees the identity block table, every prefill goes through the slot's own pages (PagedKV.row), and the kernel
    calls are those of the call with sharing patched off."""
    from midi_b200 import decode
    prompts = host_model.prompts(model, [64, 70, 5], seed=36)
    prompts = [prompts[0], prompts[1], prompts[0], prompts[2]]
    model.generate_many(prompts[:1], 1, top_k=1)                        # runtime set-up outside the trace

    def trace(share):
        with pytest.MonkeyPatch.context() as mp:
            if not share:
                mp.setattr(decode, "_share_keys", lambda prompts, page: [None] * len(prompts))
            mp.setattr(decode.PagedKV, "table_row", lambda *a: pytest.fail("a prefill through the block table"))
            spy = Spy(model, mp)
            names = mock_kernels.trace(mp, lambda: model.generate_many(prompts, [3, 2, 4, 2], batch_size=2, top_k=1))
        assert spy.pages is None and spy.launches > 0
        return names

    on = trace(True)
    assert on and on == trace(False)


def test_share_keys():
    from midi_b200 import decode
    rng = np.random.default_rng(0)
    a, b = (torch.from_numpy(rng.integers(0, 50, (70, 8))) for _ in range(2))
    short = torch.from_numpy(rng.integers(0, 50, (64, 8)))
    a2 = a.clone()
    a2[69, 7] += 1                                          # differs in the last token only
    assert decode._share_keys([a, b, a.clone(), short, short.clone(), a2, b], 64) == [0, 1, 0, None, None, None, 1]
    assert decode._share_keys([a, b, a2], 64) == [None] * 3
