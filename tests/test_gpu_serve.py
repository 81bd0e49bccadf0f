"""GPU tests (`pytest -m gpu`) of the serving queue (midi_b200/serve.py): the STREAM persistent kernel against the per-request
queue kernel over the same launches (state, host mirror, `committed`, the `ctl` exit and its bound, continuing after it), and
a trained model's requests submitted from three threads, some cancelled, against generating each alone."""
import threading
import time

import numpy as np
import pytest
import torch

import gpu_checks as GC
import gpu_model as GM
import parity_metrics as P
from gpu_checks import DEV, BF, _same
from oracle import midi_oracle as O
from test_gpu_generate_many import _mode, _restore, _snapshot, _tiny, _vs_oracle
from test_gpu_generate_many_rows import _set_rows

pytestmark = pytest.mark.gpu

KERNEL_BOUNDS = [
    ("st_state_vs_rows_mismatch", 0.0), ("st_mirror_vs_seq_mismatch", 0.0), ("st_committed_error", 0.0),
    ("st_ctl_before_events_error", 0.0), ("st_ctl_exit_past_bound", 0.0), ("st_after_ctl_vs_uninterrupted_mismatch", 0.0),
    ("min:st_ctl_launches_ended_early", 2.0), ("min:st_events_mirrored", 100.0),
]
MODEL_BOUNDS = [
    ("sv_loss_last", 1.5), ("sv_persist_vs_solo_stream_mismatch", 0.0), ("sv_cancelled_not_prefix", 0.0),
    ("sv_stream_vs_result_mismatch", 0.0), ("sv_grammar_option_violations", 0.0), ("sv_helper_vs_solo_mismatch", 0.0),
    ("sv_graph_greedy_vs_oracle_mismatch", 0.0), ("sv_nograph_greedy_vs_oracle_mismatch", 0.0),
    ("sv_graph_repeat_mismatch", 0.0), ("sv_nograph_repeat_mismatch", 0.0), ("min:sv_requests_compared", 20.0),
    ("min:sv_sampled_events_compared", 100.0), ("min:sv_cancelled", 4.0),
]


def _pinned(shape, dtype):
    return torch.zeros(shape, dtype=dtype, pin_memory=True)


def _stream_launch(gg, n, exit_on_done, out, committed, ctl):
    import ctypes
    from midi_b200 import lib
    d, ws, _ = gg._persistent()
    lib.call("b200_decode_events_queue_stream", ctypes.byref(d), gg.row_off.data_ptr(), gg.row_end.data_ptr(),
             gg.row_last.data_ptr(), int(exit_on_done), int(n), ws.data_ptr(), ws.numel(), gg.row_temp.data_ptr(),
             gg.row_top_p.data_ptr(), gg.row_top_k.data_ptr(), gg.row_seed.data_ptr(), gg.row_first.data_ptr(),
             out.data_ptr(), committed.data_ptr(), ctl.data_ptr(), lib.stream())


def test_stream_kernel_equals_the_rows_kernel():
    m = {k: 0.0 for k, _ in KERNEL_BOUNDS if not k.startswith("min:")}
    model = _tiny()
    max_len, launches = 4104, (3, 1, 4)
    mirrored = early = 0
    for B in (5, 16):
        key, gg = model._checkout_generator(B, max_len, 1.0, 1.0, 1, None, per_row=True)
        try:
            out = _pinned((B, max_len, 8), torch.int64)
            committed = _pinned((B,), torch.int32)
            ctl = _pinned((1,), torch.int32)
            for pos in (65, 4000):
                offs, state, snap = _snapshot(gg, B, pos, seed=pos + 3 * B)
                _set_rows(gg, B, pos, offs, seed=pos + B)
                gg.lengths, gg.queue, gg.rows = None, True, True
                base = [t.clone() for t in state]
                n_all = sum(launches)
                # ---- ctl never set: the same launches on both kernels
                for n in launches:
                    gg._events_queue(n, exit_on_done=False)
                ref = [t.clone() for t in state]
                _restore(state, base)
                out.fill_(-1)
                committed.fill_(-1)
                for n in launches:
                    _stream_launch(gg, n, False, out, committed, ctl)
                torch.cuda.synchronize()
                m["st_state_vs_rows_mismatch"] += sum(float((~_same(a, b)).sum()) for a, b in zip(state, ref))
                seq = gg.seq.cpu()
                for b in range(B):
                    r = pos + offs[b]
                    m["st_committed_error"] += abs(int(committed[b]) - (r + n_all))
                    m["st_mirror_vs_seq_mismatch"] += float((out[b, r + 1:r + 1 + n_all] != seq[b, r + 1:r + 1 + n_all]).sum())
                    m["st_mirror_vs_seq_mismatch"] += float((out[b, :r + 1] != -1).sum() + (out[b, r + 1 + n_all:] != -1).sum())
                    mirrored += n_all
                # ---- ctl set before a launch: it ends after its first event
                _restore(state, base)
                ctl.fill_(1)
                _stream_launch(gg, 10, False, out, committed, ctl)
                torch.cuda.synchronize()
                m["st_ctl_before_events_error"] += abs(int(gg.pos) - pos - 1)
                early += int(gg.pos) - pos < 10
                # ---- ctl set while a launch runs: it ends within one more event, and a launch without ctl continues
                ctl.fill_(0)
                committed.fill_(-1)
                _stream_launch(gg, 200, False, out, committed, ctl)
                b0 = 0
                t0 = time.time()
                while int(committed[b0]) < pos + offs[b0] + 5 and time.time() - t0 < 20:
                    time.sleep(0.0005)
                seen = int(committed[b0]) - (pos + offs[b0] + 1)      # events of this launch committed before the store
                ctl.fill_(1)
                torch.cuda.synchronize()
                ran = int(gg.pos) - pos - 1
                m["st_ctl_exit_past_bound"] += max(0, ran - (seen + 2))
                early += ran < 200
                ctl.fill_(0)
                rest = n_all + 20 - 1 - ran
                if rest > 0:
                    _stream_launch(gg, rest, False, out, committed, ctl)
                interrupted = [t.clone() for t in state]
                _restore(state, base)
                gg._events_queue(n_all + 20, exit_on_done=False)
                torch.cuda.synchronize()
                m["st_after_ctl_vs_uninterrupted_mismatch"] += sum(
                    float((~_same(a, b)).sum()) for a, b in zip(state, interrupted))
        finally:
            gg.lengths, gg.queue, gg.rows = None, False, False
            gg.set_deny(())
            model._return_generator(key, gg)
    m["st_events_mirrored"] = float(mirrored)
    m["st_ctl_launches_ended_early"] = float(early)
    P.assert_within(m, KERNEL_BOUNDS)


def _trained():
    model = GM.cpu_model()
    ocfg = O.cfg_from_hf(model.config)
    model = model.to(DEV, dtype=BF).train()
    tok = model.tokenizer
    for step in range(1, 241):                              # check_model_peaked_greedy's training
        batch = GC._song_batch(tok, 16, 66, seed=step).to(DEV)
        loss = model.training_loss(batch)
        model.fused_optimizer_step(lr=3e-4 * min(1.0, step / 20), step=step, weight_decay=0.01)
    model.eval()
    return model, ocfg, float(loss)


def test_serving_a_trained_model():
    from midi_b200.serve import GenerateServer
    model, ocfg, loss = _trained()
    m = {"sv_loss_last": loss}
    tok = model.tokenizer
    sd16 = GC._sd(model, BF)
    songs = GC._song_batch(tok, 12, 14, seed=991).numpy()
    lengths = [1, 14, 3, 9, 6, 12, 2, 14, 5, 8, 11, 4]
    budgets = [24, 6, 17, 30, 24, 5, 12, 20, 30, 10, 16, 9]
    N = len(lengths)
    prompts = [songs[i, :L] for i, L in enumerate(lengths)]
    greedy = {0, 5, 9}
    top_k = [1 if i in greedy else (20, 64, 8)[i % 3] for i in range(N)]
    temp = [1.0 if i in greedy else (1.3, 0.8, 1.0)[i % 3] for i in range(N)]
    top_p = [0.98 if i in greedy else (0.9, 1.0, 0.95)[i % 3] for i in range(N)]
    patch = [i % 4 == 1 for i in range(N)]
    ctrl = [i % 5 == 2 for i in range(N)]
    chans = [[0, 1] if i in (2, 7) else None for i in range(N)]
    seeds = [int(torch.randint(0, 2 ** 62, (1,), generator=torch.Generator().manual_seed(2000 + i))) for i in range(N)]
    cancel = {3, 8}

    def kw(i):
        return dict(temp=temp[i], top_p=top_p[i], top_k=top_k[i], disable_patch_change=patch[i],
                    disable_control_change=ctrl[i], disable_channels=chans[i], seed=seeds[i])

    solo = []
    for i in range(N):
        evs = _mode("persist", lambda: list(model.generate_stream(
            prompt=prompts[i], batch_size=1, max_len=lengths[i] + budgets[i], temp=temp[i], top_p=top_p[i], top_k=top_k[i],
            disable_patch_change=patch[i], disable_control_change=ctrl[i], disable_channels=chans[i],
            generator=torch.Generator().manual_seed(2000 + i))))
        solo.append(np.stack([e[0] for e in evs]))

    bad = not_prefix = stream_bad = viol = 0.0
    compared = sampled = n_cancel = 0
    for slots in (4, 8):
        streamed, results, errors = {}, {}, []

        def user(k, server):
            try:
                time.sleep(0.03 * k)
                reqs = {}
                for i in range(k, N, 3):
                    reqs[i] = server.submit(prompts[i], budgets[i], **kw(i))
                    time.sleep(0.01 * (1 + i % 3))
                for i, r in reqs.items():
                    evs = []
                    for ev in r:
                        evs.append(ev)
                        if i in cancel and len(evs) == 4:
                            r.cancel()
                    streamed[i], results[i] = evs, r.result()
            except Exception as e:                    # noqa: BLE001  reported below
                errors.append(e)

        with _Env("persist"), GenerateServer(model, batch_size=slots, max_len=64) as server:
            threads = [threading.Thread(target=user, args=(k, server)) for k in range(3)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
        assert not errors, errors
        for i in range(N):
            new = np.stack(streamed[i]) if streamed[i] else np.zeros((0, 8), dtype=np.int64)
            stream_bad += float((results[i][lengths[i]:] != new).sum()) if results[i].shape[0] == lengths[i] + len(
                new) else 1e9
            deny = set(model._deny_ids(patch[i], ctrl[i], chans[i]))
            viol += sum(1 for row in new if deny & set(row.tolist()))
            if i in cancel:
                n_cancel += 1
                not_prefix += float((solo[i][:len(new)] != new).sum()) if len(new) <= len(solo[i]) else 1e9
                continue
            bad += float((solo[i] != new).sum()) if solo[i].shape == new.shape else 1e9
            compared += 1
            sampled += len(new) if i not in greedy else 0
    # the app-shaped helper: row b is generate_stream at batch 1 seeded with the b-th draw of the generator
    piece = prompts[1]
    with _Env("persist"), GenerateServer(model, batch_size=4, max_len=64) as server:
        rows = list(server.generate_stream(piece, batch_size=3, max_len=40, temp=1.0, top_p=0.98, top_k=20,
                                           disable_channels=[9], generator=torch.Generator().manual_seed(77)))
    g = torch.Generator().manual_seed(77)
    hbad = 0.0
    for b in range(3):
        s = int(torch.randint(0, 2 ** 62, (1,), generator=g).item())
        ref = _mode("persist", lambda: list(model.generate_stream(piece, batch_size=1, max_len=40, temp=1.0, top_p=0.98,
                                                                  top_k=20, disable_channels=[9], generator=_First(s))))
        ref = np.stack([e[0] for e in ref])
        row = np.stack([e[b] for e in rows])
        hbad += float((row[:len(ref)] != ref).sum()) + float((row[len(ref):] != tok.pad_id).sum())
    # graph and host-issued loops: greedy requests equal the oracle, sampled ones repeat for the same submission order
    for mode in ("graph", "nograph"):
        runs = []
        for _ in range(2):
            with _Env(mode), GenerateServer(model, batch_size=4, max_len=64) as server:
                reqs = [server.submit(prompts[i], budgets[i], **kw(i)) for i in range(N)]
                runs.append([r.result() for r in reqs])
        gi = sorted(greedy)
        m[f"sv_{mode}_greedy_vs_oracle_mismatch"] = _vs_oracle(model, sd16, ocfg, [prompts[i] for i in gi],
                                                               [budgets[i] for i in gi], [runs[0][i] for i in gi])
        m[f"sv_{mode}_repeat_mismatch"] = sum(float((a != b).sum()) if a.shape == b.shape else 1e9
                                              for a, b in zip(*runs))
    m.update({"sv_persist_vs_solo_stream_mismatch": bad, "sv_cancelled_not_prefix": not_prefix,
              "sv_stream_vs_result_mismatch": stream_bad, "sv_grammar_option_violations": float(viol),
              "sv_helper_vs_solo_mismatch": hbad, "sv_requests_compared": float(compared),
              "sv_sampled_events_compared": float(sampled), "sv_cancelled": float(n_cancel)})
    P.assert_within(m, MODEL_BOUNDS)


class _Env:
    """B200_GENERATE=mode for a with block."""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        import os
        self.old = os.environ.get("B200_GENERATE")
        os.environ["B200_GENERATE"] = self.mode

    def __exit__(self, *exc):
        import os
        if self.old is None:
            os.environ.pop("B200_GENERATE", None)
        else:
            os.environ["B200_GENERATE"] = self.old


class _First(torch.Generator):
    """A CPU generator whose first torch.randint(0, 2**62, (1,)) draw is `seed`."""

    def __init__(self, seed):
        super().__init__()
        self.first = seed


_randint = torch.randint


def _randint_first(lo, hi, size, generator=None, device=None, **k):
    if isinstance(generator, _First) and generator.first is not None:
        s, generator.first = generator.first, None
        return torch.tensor([s])
    return _randint(lo, hi, size, generator=generator, device=device, **k)


@pytest.fixture(autouse=True)
def _first_draw(monkeypatch):
    monkeypatch.setattr(torch, "randint", _randint_first)
