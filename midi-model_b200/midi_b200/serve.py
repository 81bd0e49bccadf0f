"""A serving queue over one per-request generate loop: requests are submitted from any thread while it runs, each request's
events are streamed as the device commits them, and a request can be cancelled.

    with GenerateServer(model, batch_size=8, max_len=8192) as server:
        req = server.submit(prompt, max_new=512, temp=1.0, top_p=0.98, top_k=20, disable_channels=[9], seed=1234)
        for ev in req:            # int64 numpy [8] per new event, in order; ends after an EOS event or the budget
            ...
        req.result()              # int64 [L + n, 8]: the prompt and the new events, as generate_many returns them
        req.cancel()              # ends the stream; the slot is freed within the kernel's exit bound

One worker thread owns the device side: a per-request GraphGenerator (checked out from the model's pool, returned on close),
its CUDA stream and a SharedPages pool.  Submitting threads only append to a locked FIFO and set the kernel's `ctl` flag.

The scheduler is GraphGenerator.run_queue's, run online: between launches finished and cancelled requests leave their
slots, waiting requests are admitted (`_admit`: batch-1 prefill, or a copy of the prompt's tail page when a resident request
has the same prompt), and the rows are rebased (pos = the largest live position, row_off[b] = r_b - pos).  On the
persistent kernel each launch is `b200_decode_events_queue_stream` over at most 64 events, with exit_on_done while requests
wait; the worker polls the pinned `committed` array about every millisecond and hands each new event to its request.  The
launch also ends when the host sets `ctl`: a request submitted while a slot is free, a cancellation, or close.  Where the
persistent kernel does not apply (more than 32 slots, a live request with top_k > 128, or a model it is not built for) the
server runs the graph loop (or the host-issued one, B200_GENERATE=nograph), one event per step, and streams after every
event.

Guarantee: on the persistent kernel (batch_size <= 32, every top_k <= 128), a request that is not cancelled streams bit for
bit the events of generate_stream(prompt, batch_size=1, max_len=L + max_new, temp, top_p, top_k, grammar options,
generator=g), g being a generator whose first draw is the request's seed, for prompts of at most 4096 events; whatever the
arrival times, submitting threads, slots, cancellations and other requests.  A cancelled request streams a prefix of those
events.  Every request's stream equals result()[L:].
"""
from __future__ import annotations

import atexit
import collections
import numbers
import os
import threading
import time
import weakref

import numpy as np
import torch

from . import lib
from .decode import SharedPages, _share_keys

BLOCK = 64                  # events per persistent launch at most: the worker also notices close and errors between them
POLL_S = 0.001              # sleep between two polls of `committed` (an event takes milliseconds)


def _pinned(shape, dtype) -> torch.Tensor:
    """Zeroed page-locked host memory, which the streaming kernel writes and reads through its device mapping."""
    return torch.zeros(shape, dtype=dtype, pin_memory=True)


class Request:
    """One submitted request: iterate it for its new events, `result()` for the whole sequence, `cancel()` to stop it."""

    def __init__(self, server, prompt: np.ndarray, max_new: int, setting):
        self._server = server
        self.prompt, self.max_new, self.setting = prompt, max_new, setting      # setting: (temp, top_p, top_k, seed, deny)
        self.seed = setting[3]
        self._events = []
        self._cond = threading.Condition()
        self._done = False
        self._error = None
        self._result = None
        self.cancelled = False

    def __iter__(self):
        i = 0
        while True:
            with self._cond:
                while i >= len(self._events) and not self._done:
                    self._cond.wait()
                if i < len(self._events):
                    ev = self._events[i]
                elif self._error is not None:
                    raise self._error
                else:
                    return
            i += 1
            yield ev

    def result(self, timeout=None) -> np.ndarray:
        """The prompt and every new event, int64 [L + n, 8], once the request has ended (raises the worker's error)."""
        with self._cond:
            if not self._cond.wait_for(lambda: self._done, timeout):
                raise TimeoutError("request still running")
            if self._error is not None:
                raise self._error
            return self._result

    def done(self) -> bool:
        with self._cond:
            return self._done

    def cancel(self) -> None:
        """Stop generating: the stream ends after the events already committed."""
        self._server._cancel(self)

    # ---- worker side
    def _push(self, evs) -> None:
        with self._cond:
            self._events.extend(evs)
            self._cond.notify_all()

    def _finish(self, result=None, error=None) -> None:
        with self._cond:
            self._result, self._error, self._done = result, error, True
            self._cond.notify_all()


def _host_prompt(prompt, T: int, pad_id: int, what: str) -> np.ndarray:
    """generate_many's checks of one prompt and MIDIModel._prompt_tensor's token padding, on the host: int64 [L, T]."""
    if isinstance(prompt, torch.Tensor):
        if prompt.device.type != "cpu":
            raise lib.B200Error(f"{what}: the prompt must be a numpy array or a CPU tensor, got {prompt.device}")
        prompt = prompt.numpy()
    if not isinstance(prompt, np.ndarray) or prompt.dtype.kind not in "iu" or prompt.ndim != 2 or prompt.shape[0] < 1:
        raise lib.B200Error(f"{what}: the prompt must be a 2-D integer array with at least one event, got "
                            f"{getattr(prompt, 'dtype', type(prompt).__name__)} {tuple(getattr(prompt, 'shape', ()))}")
    prompt = prompt[:, :T]
    if prompt.shape[1] < T:
        prompt = np.pad(prompt, ((0, 0), (0, T - prompt.shape[1])), mode="constant", constant_values=pad_id)
    return np.ascontiguousarray(prompt, dtype=np.int64)


class GenerateServer:
    """Continuous batching for requests that arrive while it runs (see the module docstring).  `batch_size` slots,
    `max_len` events per request at most (prompt and new events), seeds of requests submitted without one drawn from
    `generator` in submission order.  Use it as a context manager, or call close(); the worker thread is also joined at
    interpreter exit."""

    def __init__(self, model, batch_size: int = 8, max_len: int = 8192, generator=None):
        from midi_model import _loop_mode
        if isinstance(batch_size, bool) or not isinstance(batch_size, numbers.Integral) or batch_size < 1:
            raise lib.B200Error(f"GenerateServer: batch_size must be an int >= 1, got {batch_size!r}")
        if isinstance(max_len, bool) or not isinstance(max_len, numbers.Integral) or max_len < 2:
            raise lib.B200Error(f"GenerateServer: max_len must be an int >= 2, got {max_len!r}")
        mode = os.environ.get("B200_GENERATE", "persist")
        if mode == "eager":
            raise lib.B200Error("GenerateServer: the serving queue needs the device-resident loop (B200_GENERATE=eager)")
        self.model, self.B, self.max_len, self.generator = model, int(batch_size), int(max_len), generator
        self._use_graph = _loop_mode(mode)
        self._rt = model._rt()
        self._version = self._rt.param_version()
        tok = model.tokenizer
        self._T, self._pad = tok.max_token_seq, tok.pad_id
        self._lock = threading.Condition()
        self._pending = collections.deque()
        self._n_live = 0
        self._closed = False
        self._error = None
        self._gg = None
        self._ctl = None
        self._ready = threading.Event()
        self._thread = threading.Thread(target=self._worker, name="GenerateServer", daemon=True)
        self._thread.start()
        self._ready.wait()
        if self._error is not None:
            self._thread.join()
            raise self._error
        ref = weakref.ref(self)
        self._atexit = lambda: (lambda s: s is not None and s.close())(ref())
        atexit.register(self._atexit)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ------------------------------------------------------------------ submitting threads
    def submit(self, prompt, max_new: int, temp=1.0, top_p=0.98, top_k=20, disable_patch_change=False,
               disable_control_change=False, disable_channels=None, seed=None) -> Request:
        """Queue one request; returns at once.  The checks of generate_many_requests apply and raise B200Error here, as do
        L - 1 + max_new >= max_len, a closed server and a model whose runtime or weights changed since the server started."""
        what = "GenerateServer.submit"
        p = _host_prompt(prompt, self._T, self._pad, what)
        if isinstance(max_new, bool) or not isinstance(max_new, numbers.Integral) or max_new < 1:
            raise lib.B200Error(f"{what}: max_new must be an int >= 1, got {max_new!r}")
        if p.shape[0] - 1 + int(max_new) >= self.max_len:
            raise lib.B200Error(f"{what}: a request of {p.shape[0]} prompt events and {max_new} new events ends at event "
                                f"{p.shape[0] - 1 + int(max_new)}, past the server's max_len {self.max_len}")
        if disable_channels is not None and (isinstance(disable_channels, (str, bytes)) or not isinstance(
                disable_channels, (collections.abc.Sequence, np.ndarray, torch.Tensor))):
            raise lib.B200Error(f"{what}: disable_channels must be None or a list of channel numbers, got {disable_channels!r}")
        rt = self.model.__dict__.get("_b200_rt")
        if rt is not self._rt or rt.param_version() != self._version or (
                self._gg is not None and self._gg.outer is not rt.cached_outer):
            raise lib.B200Error(f"{what}: the model's runtime or weights changed since the server started")
        with self._lock:
            if self._closed:
                raise self._error if self._error is not None else lib.B200Error(f"{what}: the server is closed")
            # per-request settings as generate_many_requests checks them; a seed of None is drawn here, in submission order
            setting = self.model._request_settings(
                1, [temp], [top_p], [top_k], [disable_patch_change], [disable_control_change], [disable_channels],
                None if seed is None else [seed], self.generator)[0]
            req = Request(self, p, int(max_new), setting)
            self._pending.append(req)
            if self._n_live + len(self._pending) <= self.B:
                self._signal()                     # a slot is free: end the running launch so that the worker admits it
            self._lock.notify_all()
        return req

    def generate_stream(self, prompt=None, batch_size=1, max_len=512, temp=1.0, top_p=0.98, top_k=20,
                        disable_patch_change=False, disable_control_change=False, disable_channels=None, generator=None):
        """MIDIModel.generate_stream's arguments and output, served as batch_size requests: yields int64 [batch_size, 8]
        per event, a pad event for a row that has ended, until every row has ended.  The prompt is normalised and cut
        to its last 4096 events as there.

        Row i is request i, seeded with the i-th draw of `generator` (torch.randint(0, 2**62, (1,))), so it is what
        generate_stream(prompt_i, batch_size=1, ..., generator=g_i) yields, g_i being a generator whose first draw is that
        seed.  It is deliberately not the output of generate_stream(batch_size=k): the rows of one loop share one random
        stream there, and here each row samples on its own.  Closing the iteration early cancels the rows."""
        inp = self._helper_prompt(prompt, batch_size)[:, -4096:]
        L = inp.shape[1]
        if L >= max_len:
            return
        gen_dev = generator.device if generator is not None else torch.device("cpu")
        seeds = [int(torch.randint(0, 2 ** 62, (1,), generator=generator, device=gen_dev).item()) for _ in range(len(inp))]
        reqs = [self.submit(inp[b], max_len - L, temp=temp, top_p=top_p, top_k=top_k,
                            disable_patch_change=disable_patch_change, disable_control_change=disable_control_change,
                            disable_channels=disable_channels, seed=seeds[b]) for b in range(len(inp))]
        its = [iter(r) for r in reqs]
        ended = [False] * len(reqs)
        pad = np.full(self._T, self._pad, dtype=np.int64)
        try:
            while True:
                row = []
                for i, it in enumerate(its):
                    ev = None if ended[i] else next(it, None)
                    ended[i] = ev is None
                    row.append(pad if ev is None else ev)
                if all(ended):
                    return
                yield np.stack(row)
        finally:
            for r in reqs:
                if not r.done():
                    r.cancel()

    def _helper_prompt(self, prompt, batch_size):
        """MIDIModel._prompt_tensor on the host: [batch_size, P, T] int64."""
        T = self._T
        if prompt is None:
            inp = np.full((batch_size, 1, T), self._pad, dtype=np.int64)
            inp[:, 0, 0] = self.model.tokenizer.bos_id
            return inp
        prompt = np.asarray(prompt)
        if prompt.ndim == 2:
            prompt = np.repeat(prompt[None, :], repeats=batch_size, axis=0)
        elif prompt.shape[0] == 1:
            prompt = np.repeat(prompt, repeats=batch_size, axis=0)
        elif prompt.ndim != 3 or prompt.shape[0] != batch_size:
            raise ValueError(f"invalid shape for prompt, {prompt.shape}")
        prompt = prompt[..., :T]
        if prompt.shape[-1] < T:
            prompt = np.pad(prompt, ((0, 0), (0, 0), (0, T - prompt.shape[-1])), mode="constant", constant_values=self._pad)
        return np.ascontiguousarray(prompt, dtype=np.int64)

    def _signal(self) -> None:
        if self._ctl is not None:
            self._ctl[0] = 1

    def _cancel(self, req: Request) -> None:
        with self._lock:
            req.cancelled = True
            self._signal()
            self._lock.notify_all()

    def close(self) -> None:
        """Stop the worker: every request still pending or running ends (as cancelled), the loop goes back to the model's
        pool, and the thread is joined."""
        with self._lock:
            self._closed = True
            self._signal()
            self._lock.notify_all()
        if self._thread is not threading.current_thread():
            self._thread.join()
        if getattr(self, "_atexit", None) is not None:
            atexit.unregister(self._atexit)
            self._atexit = None

    # ------------------------------------------------------------------ worker thread
    def _worker(self) -> None:
        key = gg = None
        clean = False
        try:
            # the loop and its per-request arrays are made outside inference mode: they go back to the pool that
            # generate_many_requests draws from, which updates them in place
            key, gg = self.model._checkout_generator(self.B, self.max_len, 1.0, 1.0, 1, None, per_row=True)
            gg.alloc_rows()
            self._gg = gg
            with torch.inference_mode(), torch.cuda.stream(gg.stream):
                try:
                    self._start(gg)
                    self._ready.set()
                    self._serve(gg)
                    clean = True
                finally:
                    if getattr(self, "_pages", None) is not None:
                        self._pages.close()
                    gg.set_deny(())
                    torch.cuda.current_stream().wait_stream(gg.stream)
        except BaseException as e:           # noqa: BLE001  every request learns of the worker's failure
            err = e if isinstance(e, Exception) else lib.B200Error(f"GenerateServer worker stopped: {e!r}")
            with self._lock:
                self._error, self._closed = err, True
                pending, self._pending = list(self._pending), collections.deque()
            for r in pending + [r for r in getattr(self, "_slot", []) if r is not None]:
                r._finish(error=err)
            self._ready.set()
        finally:
            if clean:
                self.model._return_generator(key, gg)

    def _start(self, gg) -> None:
        """Empty queue state, the per-request arrays, the page pool and, on the persistent kernel, the host mirror.  The
        graph loop's per-event graph is captured now, while no request is resident (capture runs an event)."""
        gg.queue, gg.rows, gg.lengths = True, True, None
        gg.req_top_k = []
        self._persist = self._use_graph == "persist" and gg.persistent_ok()
        self._graph = self._use_graph is True or (self._use_graph == "persist" and not self._persist)
        gg._capture(self._graph, gg._set_queue_state)
        self._pages = SharedPages(gg.kv1)
        B = self.B
        self._slot = [None] * B
        self._posn = [0] * B
        self._offs = [0] * B
        self._groups = {}                          # share group key -> [prompt, resident count]
        self._slot_group = [None] * B
        if self._persist:
            self._out = _pinned((B, self.max_len, self._T), torch.int64)
            self._committed = _pinned((B,), torch.int32)
            ctl = _pinned((1,), torch.int32)
            self._out_np, self._committed_np = self._out.numpy(), self._committed.numpy()
            with self._lock:
                self._ctl_t, self._ctl = ctl, ctl.numpy()

    def _share_key(self, prompt: np.ndarray):
        """Share group of a request being admitted: that of a resident request with an equal prompt, else a new one (a
        prompt of fewer than page + 1 events shares nothing)."""
        page = self._gg.kv1.page
        if prompt.shape[0] - 1 < page:
            return None
        groups = list(self._groups.items())
        keys = _share_keys([torch.from_numpy(prompt)] + [torch.from_numpy(g[0]) for _, g in groups], page)
        for i, (k, _) in enumerate(groups):
            if keys[0] is not None and keys[i + 1] == keys[0]:
                return k
        k = object()
        self._groups[k] = [prompt, 0]
        return k

    def _serve(self, gg) -> None:
        B = self.B
        slot, posn = self._slot, self._posn
        changed = True
        while True:
            if self._ctl is not None:
                self._ctl[0] = 0                   # before the queue is read: a later submission sets it again
            with self._lock:
                closing = self._closed
                cancelled = [r for r in self._pending if r.cancelled]
                for r in cancelled:
                    self._pending.remove(r)
            for r in cancelled:
                r._finish(result=r.prompt.copy())
            freed = [b for b in range(B) if slot[b] is not None and (slot[b].cancelled or closing)]
            for b in freed:
                self._end(gg, b, posn[b])
            changed |= bool(freed)
            if closing:
                with self._lock:
                    pending, self._pending = list(self._pending), collections.deque()
                for r in pending:
                    r._finish(result=r.prompt.copy())
                return
            free = [b for b in range(B) if slot[b] is None]
            with self._lock:
                admit = [self._pending.popleft() for _ in range(min(len(free), len(self._pending)))]
                self._n_live = B - len(free) + len(admit)
            for b in free:
                self._pages.release(b)
            for b, r in zip(free, admit):
                k = self._share_key(r.prompt)
                self._slot_group[b] = k
                if k is not None:
                    self._groups[k][1] += 1
                gg._admit(b, torch.from_numpy(r.prompt).to(gg.seq.device), r.setting, self._pages, k)
                slot[b], posn[b] = r, r.prompt.shape[0] - 1
                if self._ctl is not None:
                    self._committed_np[b] = posn[b]
                changed = True
            live = [b for b in range(B) if slot[b] is not None]
            if not live:
                with self._lock:
                    if not self._pending and not self._closed:
                        self._lock.wait(0.05)
                continue
            if changed:
                for b in range(B):
                    if slot[b] is None and self._slot_group[b] is None:
                        self._pages.park(b)
                pos = max(posn[b] for b in live)
                self._offs = [posn[b] - pos if slot[b] is not None else -pos for b in range(B)]
                gg.pos.fill_(pos)
                gg.row_off.copy_(torch.tensor(self._offs, dtype=torch.int32))
                gg.row_end.copy_(torch.tensor([self._end_at(b) if slot[b] is not None else 0 for b in range(B)],
                                              dtype=torch.int32))
                gg.row_last.copy_(torch.tensor([-1 if slot[b] is not None else -2 for b in range(B)], dtype=torch.int32))
                changed = False
            gg.req_top_k = [slot[b].setting[2] for b in live]
            with self._lock:
                waiting = bool(self._pending)
            if self._persist and gg.persistent_ok():
                n = min(BLOCK, max(self._end_at(b) - posn[b] for b in live))
                self._launch_stream(gg, n, waiting, live)
                state = torch.cat([gg.pos, gg.row_last]).cpu()
            else:
                # the graph loop, or for a persistent server's event with a live top_k > 128 request its launches issued
                # from the host (a graph captured now would have to run an event of its own)
                if self._graph:
                    gg.graph_queue_rows.replay()
                else:
                    gg._event()
                bs = torch.tensor(live, dtype=torch.long)
                qs = torch.tensor([posn[b] + 1 for b in live], dtype=torch.long)
                evs = gg.seq[bs.to(gg.seq.device), qs.to(gg.seq.device)].cpu().numpy()
                state = torch.cat([gg.pos, gg.row_last]).cpu()
                for i, b in enumerate(live):
                    slot[b]._push([evs[i].copy()])
            p_now, last = int(state[0]), state[1:].tolist()
            for b in live:
                if last[b] >= 0:
                    self._end(gg, b, last[b])
                    changed = True
                else:
                    posn[b] = p_now + self._offs[b]

    def _end_at(self, b: int) -> int:
        """Seq index of the last event slot b's request may commit."""
        r = self._slot[b]
        return r.prompt.shape[0] - 1 + r.max_new

    def _launch_stream(self, gg, n: int, exit_on_done: bool, live) -> None:
        """One launch of the streaming kernel; the new events go to their requests while it runs and after it ends."""
        import ctypes
        d, ws, _ = gg._persistent()
        lib.call("b200_decode_events_queue_stream", ctypes.byref(d), gg.row_off.data_ptr(), gg.row_end.data_ptr(),
                 gg.row_last.data_ptr(), int(exit_on_done), int(n), ws.data_ptr(), ws.numel(), gg.row_temp.data_ptr(),
                 gg.row_top_p.data_ptr(), gg.row_top_k.data_ptr(), gg.row_seed.data_ptr(), gg.row_first.data_ptr(),
                 self._out.data_ptr(), self._committed.data_ptr(), self._ctl_t.data_ptr(), lib.stream())
        done = torch.cuda.Event()
        done.record(gg.stream)
        while True:
            finished = done.query()
            self._drain(live)
            if finished:
                return
            time.sleep(POLL_S)

    def _drain(self, live) -> None:
        """Hand every event committed since the last look to its request: committed[b] first, then the events up to it."""
        for b in live:
            r = self._slot[b]
            c = int(self._committed_np[b])
            first = r.prompt.shape[0] + len(r._events)
            if c >= first:
                r._push([ev.copy() for ev in self._out_np[b, first:c + 1]])

    def _end(self, gg, b: int, last: int) -> None:
        """Slot b's request ends with its events up to seq index `last`; the slot is free for the next admission."""
        r = self._slot[b]
        r._finish(result=gg.seq[b, :last + 1].clone().cpu().numpy())
        k = self._slot_group[b]
        if k is not None:
            self._groups[k][1] -= 1
            if self._groups[k][1] == 0:
                del self._groups[k]
        self._slot[b], self._slot_group[b] = None, None
