"""GPU tests (`pytest -m gpu`) of shared prompts in the request queue: requests with equal prompts prefill once and read the
prompt's whole pages from the same KV pages.  Every request of a sharing call must be bit for bit the same request with
sharing off, on every loop (persist, graph, nograph), in scalar and per-request mode, at 4, 8 and 16 slots; on the
persistent kernel a per-request result must also be generate() of its prompt alone; and each shared prompt must be
prefilled once per stretch in which one of its requests is resident."""
import pytest
import torch

import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF
from test_gpu_generate_many import _mode

pytestmark = pytest.mark.gpu

BOUNDS = [
    ("sh_vs_sharing_off_mismatch", 0.0), ("sh_rows_persist_vs_generate_mismatch", 0.0), ("sh_prefill_count_error", 0.0),
    ("sh_pages_left_held", 0.0), ("sh_sharing_state_error", 0.0), ("min:sh_requests_compared", 300.0), ("min:sh_sharer_admissions", 40.0),
    ("min:sh_generate_compared", 6.0),
]

SHARED = [100, 129, 2300, 3900]          # four samples of each
DISTINCT = [40, 700, 3100]


def _requests(tok):
    from midi_b200.synth import synth_batch
    songs = synth_batch(tok, len(SHARED) + len(DISTINCT), max(SHARED + DISTINCT), seed=77).numpy()
    pieces = [songs[i, :L] for i, L in enumerate(SHARED)]
    others = [songs[len(SHARED) + i, :L] for i, L in enumerate(DISTINCT)]
    prompts = []
    for i, p in enumerate(pieces):                    # samples of a piece interleaved with the distinct requests
        prompts += [p, p]
        if i < len(others):
            prompts.append(others[i])
        prompts += [p, p]
    budgets = [6 + (5 * i) % 13 for i in range(len(prompts))]
    return prompts, budgets


def _expected_prefills(keys, lengths, n_new, B):
    """Outer prefills of the queue's schedule: request i runs n_new[i] events from its admission; finished slots are
    refilled in slot order; a request is prefilled unless a live request has its share key."""
    N = len(keys)
    slot, end = [None] * B, [0] * B
    t, nxt, count, free = 0, 0, 0, list(range(B))
    while True:
        for b in free:
            slot[b] = None
        for b in free:
            if nxt < N:
                live_keys = {keys[slot[x]] for x in range(B) if slot[x] is not None}
                if lengths[nxt] > 1 and (keys[nxt] is None or keys[nxt] not in live_keys):
                    count += 1
                slot[b], end[b] = nxt, t + n_new[nxt]
                nxt += 1
        live = [b for b in range(B) if slot[b] is not None]
        if not live:
            return count
        t = min(end[b] for b in live)
        free = [b for b in live if end[b] == t]


def test_shared_prompts_are_bitwise_sharing_off():
    from midi_b200 import decode
    m = {k: 0.0 for k, _ in BOUNDS}
    m = {k.removeprefix("min:"): v for k, v in m.items()}
    model = GM.cpu_model().to(DEV, dtype=BF).eval()
    prompts, budgets = _requests(model.tokenizer)
    N = len(prompts)
    seeds = [int(torch.randint(0, 2 ** 62, (1,), generator=torch.Generator().manual_seed(500 + i))) for i in range(N)]
    keys = decode._share_keys([torch.from_numpy(p) for p in prompts], 64)
    assert sum(k is not None for k in keys) == 4 * len(SHARED)
    prefills, admissions, made = [], [], []
    step, admit, pages_init = decode.CachedStack.step, decode.SharedPages.admit, decode.SharedPages.__init__

    def spy_step(stack, x, kv, s_new, pos_dev=None, *a, **k):
        if pos_dev is None and stack is model._b200_rt.cached_outer:
            prefills.append(s_new)
        return step(stack, x, kv, s_new, pos_dev, *a, **k)

    def spy_admit(pages, b, L, key):
        src = admit(pages, b, L, key)
        admissions.append(src is not None)
        return src

    def spy_pages(pages, *a, **k):
        pages_init(pages, *a, **k)
        made.append(pages)

    def call(mode, B, per_request, share):
        kw = dict(temp=1.1, top_p=0.95, top_k=[40] * N, seeds=seeds) if per_request else dict(
            temp=1.1, top_p=0.95, top_k=40, generator=torch.Generator().manual_seed(9))
        prefills.clear()
        admissions.clear()
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(decode.CachedStack, "step", spy_step)
            mp.setattr(decode.SharedPages, "admit", spy_admit)
            mp.setattr(decode.SharedPages, "__init__", spy_pages)
            if not share:
                mp.setattr(decode, "_share_keys", lambda prompts, page: [None] * len(prompts))
            out = _mode(mode, lambda: model.generate_many_requests(prompts, budgets, batch_size=B, **kw))
        pages = made.pop() if made else None
        m["sh_sharing_state_error"] += (pages is None) == share
        if pages is not None:
            free = pages.free
            m["sh_pages_left_held"] += abs(len(free) - pages.n_pages) + pages.n_pages - len(set(free)) + len(pages.groups)
        return out, list(prefills), sum(admissions)

    for mode in ("persist", "graph", "nograph"):
        for per_request in (False, True):
            for B in (4, 8, 16):
                got, n_pre, n_join = call(mode, B, per_request, True)
                off, n_pre_off, _ = call(mode, B, per_request, False)
                assert len(n_pre_off) == N
                for a, b in zip(got, off):
                    m["sh_vs_sharing_off_mismatch"] += float((a != b).sum()) if a.shape == b.shape else 1e9
                m["sh_requests_compared"] += N
                m["sh_sharer_admissions"] += n_join
                n_new = [o.shape[0] - p.shape[0] for o, p in zip(off, prompts)]
                want = _expected_prefills(keys, [p.shape[0] for p in prompts], n_new, B)
                m["sh_prefill_count_error"] += abs(len(n_pre) - want) + abs(len(n_pre) + n_join - N)
                if mode == "persist" and per_request and B == 8:
                    for i in [0, 2, 6, 7, 11, 13, 17]:
                        p = prompts[i]
                        solo = _mode("persist", lambda: model.generate(
                            prompt=p, batch_size=1, max_len=p.shape[0] + budgets[i], temp=1.1, top_p=0.95, top_k=40,
                            generator=torch.Generator().manual_seed(500 + i)))[0]
                        m["sh_rows_persist_vs_generate_mismatch"] += (float((solo != got[i]).sum())
                                                                       if solo.shape == got[i].shape else 1e9)
                        m["sh_generate_compared"] += 1
    P.assert_within(m, BOUNDS)
