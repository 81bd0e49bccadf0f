"""TEST INFRASTRUCTURE: a CPU stand-in for the streaming queue entry (`b200_decode_events_queue_stream`), on top of
tests/mock_shared.py (and so tests/mock_rows.py and tests/mock_queue.py), so that the serving queue (midi_b200/serve.py)
runs in the CPU suite on the host-issued loop and on the persistent kernel's launch protocol.  Semantics follow
include/midi_b200.h.

The stand-in runs the per-request queue stand-in one event at a time.  After each event it writes every committed event of
a live row to the host mirror `out_events`, then `committed[b]`, and then samples `ctl`: when it is nonzero the launch ends
after that event, which is the kernel's bound (a store seen in event e ends the launch after event e).  Every hook in
ON_EVENT is called after each event with the number of events this launch has run, so a test can act while a launch runs.
LAUNCHES records (n_events, exit_on_done, events run, ended by ctl) per launch.
"""
import torch

import mock_rows
import mock_shared
from mock_kernels import _from_ptr

PD_T = 8
ON_EVENT = []
LAUNCHES = []


def _decode_events_queue_stream(desc, row_off, row_end, row_last, exit_on_done, n_events, ws, wsb, row_temp, row_top_p,
                                row_top_k, row_seed, row_first, out_events, committed, ctl, s):
    d = desc._obj
    B = d.batch
    pos = _from_ptr(d.pos, 1, torch.int32)
    seq = _from_ptr(d.seq, B * d.max_len * PD_T, torch.int64).view(B, d.max_len, PD_T)
    out = _from_ptr(out_events, B * d.max_len * PD_T, torch.int64).view(B, d.max_len, PD_T)
    done = _from_ptr(committed, B, torch.int32)
    flag = _from_ptr(ctl, 1, torch.int32)
    last = _from_ptr(row_last, B, torch.int32)
    offs = _from_ptr(row_off, B, torch.int32).tolist()
    ran, by_ctl = 0, False
    for e in range(n_events):
        p = int(pos[0])
        live = [b for b in range(B) if int(last[b]) == -1]
        if not live or p + 1 >= d.max_len:
            break
        mock_rows._decode_events_queue_rows(desc, row_off, row_end, row_last, exit_on_done, 1, ws, wsb, row_temp,
                                            row_top_p, row_top_k, row_seed, row_first, s)
        ran += 1
        for b in live:
            q = p + offs[b] + 1
            out[b, q] = seq[b, q]
            done[b] = q
        for hook in ON_EVENT:
            hook(ran)
        fin = any(int(last[b]) != -1 for b in live)
        if int(flag[0]) != 0:
            by_ctl = True
            break
        if fin and exit_on_done:
            break
    LAUNCHES.append((n_events, exit_on_done, ran, by_ctl))


class _Event:
    """torch.cuda.Event stand-in: the mock kernels have finished when their call returns."""

    def __init__(self, *a, **k):
        pass

    def record(self, stream=None):
        pass

    def query(self):
        return True


def _call(name, *args):
    if name == "b200_decode_events_queue_stream":
        return _decode_events_queue_stream(*args)
    return mock_rows._call(name, *args)


def install(monkeypatch, persist=False):
    """mock_shared.install plus the streaming entry, host memory in place of pinned memory and a finished-at-once event,
    for the duration of one test."""
    from midi_b200 import lib, serve
    mock_shared.install(monkeypatch, persist=persist)
    monkeypatch.setattr(lib, "call", _call)
    monkeypatch.setattr(serve, "_pinned", lambda shape, dtype: torch.zeros(shape, dtype=dtype))
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    ON_EVENT.clear()
    LAUNCHES.clear()
