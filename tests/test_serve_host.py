"""The serving queue (midi_b200/serve.py: GenerateServer) over the CPU stand-in for the kernel layer (tests/mock_kernels.py),
on the host-issued loop (B200_GENERATE=nograph) and on the streaming persistent kernel's launch protocol: requests
submitted from several threads while the server runs, cancellations, the stream against result(), the budget and EOS,
input errors, a worker failure, the app-shaped helper, and generate_many's kernel calls left as they were.  The kernel
itself is checked on the GPU (tests/test_gpu_serve.py)."""
import os
import shutil
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

import host_model
import mock_decode
import mock_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENGTHS = [5, 2, 9, 3, 7, 4, 1, 6, 3, 8, 2, 5]
BUDGETS = [6, 4, 3, 8, 5, 5, 4, 7, 2, 6, 5, 3]
TOP_KS = [1, 20, 1, 3, 1, 1, 8, 1, 1, 64, 1, 2]
TEMPS = [1.0, 1.3, 1.0, 0.9, 1.0, 1.0, 1.2, 1.0, 1.0, 0.8, 1.0, 1.1]
SEEDS = [11, 2 ** 62 - 1, 0, 7, 123456789, 99, 5, 42, 8, 77, 3, 1000]
CHANNELS = [None, [0, 9], None, None, None, [3], None, None, None, None, None, [1]]


@pytest.fixture(params=["nograph", "persist"])
def model(request, monkeypatch):
    m = host_model.generate_model(monkeypatch, request.param)
    m.loop = request.param
    return m


def _kw(i):
    return dict(temp=TEMPS[i], top_p=0.9, top_k=TOP_KS[i], disable_channels=CHANNELS[i], seed=SEEDS[i])


def _many(model, prompts, idx):
    """generate_many_requests of requests idx, each with its settings and seed, through one slot."""
    return model.generate_many_requests([prompts[i] for i in idx], [BUDGETS[i] for i in idx], batch_size=1,
                                        temp=[TEMPS[i] for i in idx], top_p=[0.9] * len(idx),
                                        top_k=[TOP_KS[i] for i in idx], disable_channels=[CHANNELS[i] for i in idx],
                                        seeds=[SEEDS[i] for i in idx])


def _solo_greedy(model, p, n):
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200_GENERATE", "nograph")
        return model.generate(prompt=p, batch_size=1, max_len=p.shape[0] + n, top_k=1)[0]


@pytest.mark.parametrize("slots", [2, 4])
def test_requests_from_three_threads_with_cancellations(model, slots):
    from midi_b200.serve import GenerateServer
    prompts = host_model.prompts(model, LENGTHS, seed=31)
    cancel = {3, 7}
    streamed, results, errors = {}, {}, []

    def user(k, idx, delay):
        try:
            time.sleep(delay)
            reqs = {}
            for i in idx:
                reqs[i] = server.submit(prompts[i], BUDGETS[i], **_kw(i))
                time.sleep(0.02)
            for i, r in reqs.items():
                evs = []
                for ev in r:
                    evs.append(ev)
                    if i in cancel and len(evs) == 2:
                        r.cancel()
                streamed[i], results[i] = evs, r.result()
        except Exception as e:                    # noqa: BLE001  reported by the main thread
            errors.append(e)

    with GenerateServer(model, batch_size=slots, max_len=32) as server:
        threads = [threading.Thread(target=user, args=(k, list(range(k, len(LENGTHS), 3)), 0.05 * k)) for k in range(3)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    assert not errors, errors
    assert not server._thread.is_alive()
    eos = model.tokenizer.eos_id
    ref = _many(model, prompts, list(range(len(LENGTHS))))
    for i, p in enumerate(prompts):
        L, got = p.shape[0], results[i]
        new = np.stack(streamed[i]) if streamed[i] else np.zeros((0, 8), dtype=np.int64)
        assert got.dtype == np.int64 and got.shape[0] == L + len(new), i
        assert (got[:L] == p).all() and (got[L:] == new).all(), i                 # the stream is result()[L:], in order
        assert 1 <= len(new) <= BUDGETS[i], i
        if i in cancel:
            assert (ref[i][L:L + len(new)] == new).all(), i                         # a prefix of the uncancelled request
            continue
        assert got.shape == ref[i].shape and (got == ref[i]).all(), i
        assert len(new) == BUDGETS[i] or new[-1, 0] == eos, i
        if TOP_KS[i] == 1:
            solo = _solo_greedy(model, p, BUDGETS[i])
            assert got.shape == solo.shape and (got == solo).all(), i
        deny = set(model._deny_ids(False, False, CHANNELS[i]))
        assert not any(deny & set(row.tolist()) for row in new), i
    if model.loop == "persist":
        assert mock_decode.LAUNCHES and all(n <= 64 for n, _, _, _ in mock_decode.LAUNCHES)


def test_cancel_ends_a_running_launch(model):
    """A cancellation while a launch runs ends it after the event in which ctl is seen; the slot then serves the next
    request, whose result is unchanged."""
    from midi_b200.serve import GenerateServer
    prompts = host_model.prompts(model, [4, 3], seed=32)
    with GenerateServer(model, batch_size=1, max_len=64) as server:
        seen = []
        long = server.submit(prompts[0], 40, top_k=1, seed=1)
        if model.loop == "persist":
            mock_decode.ON_EVENT.append(lambda k: seen.append(k) if k == 3 and not long.cancelled and long.cancel() is None
                                        else None)
        else:
            it = iter(long)
            for _ in range(3):
                next(it)
            long.cancel()
        nxt = server.submit(prompts[1], 5, top_k=1, seed=2)
        got_long, got_next = long.result(), nxt.result()
    assert prompts[0].shape[0] + 3 <= got_long.shape[0] < prompts[0].shape[0] + 40
    if model.loop == "persist":
        first = mock_decode.LAUNCHES[0]
        assert first[3] and first[2] == 3                                    # left after the event that saw ctl
    solo = _solo_greedy(model, prompts[1], 5)
    assert got_next.shape == solo.shape and (got_next == solo).all()
    solo_long = _solo_greedy(model, prompts[0], 40)
    assert (solo_long[:got_long.shape[0]] == got_long).all()


def test_submit_checks_raise_in_the_callers_thread(model):
    from midi_b200.lib import B200Error
    from midi_b200.serve import GenerateServer
    p = host_model.prompts(model, [4], seed=33)[0]
    bad = [dict(max_new=0), dict(max_new=2.0), dict(max_new=True), dict(max_new=13), dict(temp=0.0), dict(temp=-1.0),
           dict(temp=float("nan")), dict(top_p=0.0), dict(top_p=1.5), dict(top_k=0), dict(top_k=2.5), dict(seed=-1),
           dict(seed=2 ** 62), dict(seed=2.0), dict(seed=True), dict(disable_channels=[16]), dict(disable_channels=[-1]),
           dict(disable_channels=3), dict(disable_channels=[True]), dict(disable_channels="9")]
    with GenerateServer(model, batch_size=2, max_len=16) as server:
        for kw in bad:
            with pytest.raises(B200Error):
                server.submit(p, **{"max_new": 2, "top_k": 1, **kw})
        for prompt in (p[:0], p[0], p.astype(np.float32), torch.from_numpy(p).to(torch.float32), "x"):
            with pytest.raises(B200Error):
                server.submit(prompt, 2, top_k=1)
        ok = server.submit(p, 12, top_k=1, seed=4)               # L - 1 + max_new = 15 < 16
        assert ok.result().shape[0] <= 16
    with pytest.raises(B200Error):
        server.submit(p, 2)
    # seeds of requests without one come from the server's generator, in submission order
    g = torch.Generator().manual_seed(9)
    want = [int(torch.randint(0, 2 ** 62, (1,), generator=torch.Generator().manual_seed(9)).item())]
    with GenerateServer(model, batch_size=1, max_len=16, generator=g) as server:
        r = server.submit(p, 2)
        r.result()
    assert r.seed == want[0]


def test_weights_changed_since_start_raise(model):
    from midi_b200.lib import B200Error
    from midi_b200.serve import GenerateServer
    p = host_model.prompts(model, [3], seed=34)[0]
    with GenerateServer(model, batch_size=1, max_len=16) as server:
        server.submit(p, 2, top_k=1).result()
        with torch.no_grad():
            model.lm_head.weight.mul_(1.0)
        with pytest.raises(B200Error):
            server.submit(p, 2, top_k=1)


def test_worker_error_reaches_every_iterator(model, monkeypatch):
    from midi_b200 import lib
    from midi_b200.lib import B200Error
    from midi_b200.serve import GenerateServer
    prompts = host_model.prompts(model, [3, 4, 5, 2, 6], seed=35)
    call = lib.call

    def failing(name, *a):                # the first event fails, with two requests resident and three waiting
        if name in ("b200_decode_events_queue_stream", "b200_event_commit_queue") and len(server._pending) == 3:
            raise B200Error("injected launch failure")
        return call(name, *a)

    monkeypatch.setattr(lib, "call", failing)
    server = GenerateServer(model, batch_size=2, max_len=32)
    with server._lock:                    # all five queued before the worker admits any
        reqs = [server.submit(p, 20, top_k=1) for p in prompts]
    for r in reqs:
        with pytest.raises(B200Error, match="injected"):
            list(r)
        with pytest.raises(B200Error, match="injected"):
            r.result()
    server._thread.join(5)
    assert not server._thread.is_alive()
    with pytest.raises(B200Error):
        server.submit(prompts[0], 2, top_k=1)
    server.close()


def test_helper_rows_and_pad_layout(model):
    """server.generate_stream: [B, 8] per event, pad events after a row ends, row i = generate_stream at batch 1 seeded with
    the i-th draw of the generator."""
    from midi_b200.serve import GenerateServer
    tok = model.tokenizer
    prompt = host_model.prompts(model, [5], seed=36)[0]
    B, max_len = 3, 12
    with GenerateServer(model, batch_size=2, max_len=64) as server:
        # EOS is likely for some rows with a sampled step 0: check the pad layout whenever a row ends early
        out = list(server.generate_stream(prompt, batch_size=B, max_len=max_len, top_k=3, temp=1.5,
                                          generator=torch.Generator().manual_seed(5)))
    assert out and all(e.shape == (B, 8) and e.dtype == np.int64 for e in out)
    assert len(out) <= max_len - prompt.shape[0]
    seeds = torch.Generator().manual_seed(5)
    for b in range(B):
        s = int(torch.randint(0, 2 ** 62, (1,), generator=seeds).item())
        g = torch.Generator()
        orig = torch.randint
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200_GENERATE", "nograph")                  # the mock layer has no rectangular persistent kernel
            mp.setattr(torch, "randint", lambda lo, hi, size, generator=None, device=None:
                       torch.tensor([s]) if generator is g else orig(lo, hi, size, generator=generator, device=device))
            solo = list(model.generate_stream(prompt, batch_size=1, max_len=max_len, top_k=3, temp=1.5, generator=g))
        row = np.stack([e[b] for e in out])
        k = len(solo)
        assert (row[:k] == np.stack([e[0] for e in solo])).all(), b
        assert (row[k:] == tok.pad_id).all(), b
        assert k == max_len - prompt.shape[0] or solo[-1][0, 0] == tok.eos_id, b
    assert any((row == tok.pad_id).all() for row in out[-1]) or len(out) == max_len - prompt.shape[0]


def test_generate_many_trace_is_unchanged_by_a_server(model):
    from midi_b200.serve import GenerateServer
    prompts = host_model.prompts(model, [4, 2, 6], seed=37)
    model.generate_many_requests(prompts[:1], 1, top_k=1)

    def trace():
        with pytest.MonkeyPatch.context() as mp:
            return mock_kernels.trace(mp, lambda: model.generate_many_requests(prompts, [3, 2, 4], batch_size=2, top_k=1,
                                                                             seeds=[1, 2, 3]))

    before = trace()
    with GenerateServer(model, batch_size=2, max_len=10) as server:       # the loop generate_many then reuses
        server.submit(prompts[0], 3, top_k=1).result()
    assert before and trace() == before
    assert "b200_decode_events_queue_stream" not in before


def test_stream_entry_checks_its_buffers_without_a_gpu():
    """A plain-C program (tests/abi/abi_stream.c) calls b200_decode_events_queue_stream without its host buffers: the
    entry refuses with B200_ERR_ARG before any CUDA call."""
    from midi_b200 import lib
    if not os.path.exists(lib.LIB_PATH):
        import sys
        subprocess.check_call([sys.executable, os.path.join(ROOT, "midi-model_b200", "build_ext.py")])
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"abi_stream_{os.getpid()}")
    libdir = os.path.dirname(lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "abi", "abi_stream.c"), "-L", libdir, "-lmidi_b200",
                           f"-Wl,-rpath,{libdir}", "-o", exe])
    try:
        r = subprocess.run([exe], capture_output=True, text=True)
    finally:
        os.remove(exe)
    assert r.returncode == 0 and "abi stream ok" in r.stdout, r.stdout + r.stderr
