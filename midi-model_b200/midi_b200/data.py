"""Host data path of the train step (train.py:31-90, 408-425), GPU side.

The reference dataset keeps every tokenised MIDI file as an int16 matrix `[events, max_token_seq]` (train.py:71), widens it
to int64 on the host, pads to the longest sample of the batch with `pad_id` (`collate_fn`, train.py:82-86) and lets the
DataLoader pin and copy int64 batches (8 bytes per token).  Here the batch stays int16 until it is on the GPU:

* `collate(samples, pad_id)`    -- `collate_fn` on int16, straight into pinned memory (one allocation per batch);
* `Prefetcher(batches, device)` -- copies batch i+1 host->device on a copy stream while step i computes (2-deep ring,
                                   event-ordered, allocator-safe);
* `MIDIModel.training_loss(batch_int16)` -- one kernel (`b200_batch_to_xy_i16`) widens and cuts the batch into the
                                   contiguous `x = batch[:, :-1]`, `y = batch[:, 1:]` int64 views the step needs.

That is 2 bytes per token over PCIe instead of 8 and no host-side widening: 0.26 MB per step at batch 8 x 2049 events.
"""
from __future__ import annotations

from typing import Iterable, Iterator, List, Sequence

import numpy as np
import torch


def collate(samples: Sequence, pad_id: int = 0, pin: bool = True) -> torch.Tensor:
    """train.py:82-86 on int16: stack ragged `[L_i, T]` token matrices into `[B, max L_i, T]`, right-padded with `pad_id`.
    `samples` may be numpy arrays or tensors of any integer dtype whose values fit int16 (vocab 3406 does)."""
    mats: List[np.ndarray] = []
    for s in samples:
        a = s.numpy() if isinstance(s, torch.Tensor) else np.asarray(s)
        if a.ndim != 2:
            raise ValueError(f"collate: expected [events, tokens] matrices, got shape {a.shape}")
        mats.append(a)
    if not mats:
        raise ValueError("collate: empty batch")
    T = mats[0].shape[1]
    if any(m.shape[1] != T for m in mats):
        raise ValueError("collate: samples disagree on tokens per event")
    L = max(m.shape[0] for m in mats)
    out = torch.empty((len(mats), L, T), dtype=torch.int16, pin_memory=pin and torch.cuda.is_available())
    o = out.numpy()
    o[...] = pad_id
    for i, m in enumerate(mats):
        if m.size and (m.max() > np.iinfo(np.int16).max or m.min() < np.iinfo(np.int16).min):
            raise ValueError("collate: token id outside int16")
        o[i, :m.shape[0]] = m
    return out


class Prefetcher:
    """Iterate device copies of host batches, keeping `depth` host->device copies in flight on a side stream.

    for batch in Prefetcher(loader, device):         # batch: int16 [B, L, T] on `device`
        loss = model.training_loss(batch)
    """

    def __init__(self, batches: Iterable[torch.Tensor], device, depth: int = 2):
        self.it: Iterator[torch.Tensor] = iter(batches)
        self.device = torch.device(device)
        self.depth = max(1, int(depth))
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.queue: list = []

    def _issue(self) -> bool:
        try:
            host = next(self.it)
        except StopIteration:
            return False
        if not host.is_pinned():
            host = host.pin_memory()
        with torch.cuda.stream(self.copy_stream):
            dev = host.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.queue.append((dev, ev, host))          # `host` stays referenced until its copy has been consumed
        return True

    def __iter__(self):
        while len(self.queue) < self.depth and self._issue():
            pass
        while self.queue:
            dev, ev, _host = self.queue.pop(0)
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ev)
            dev.record_stream(cur)                  # allocated on the copy stream, consumed on the compute stream
            self._issue()
            yield dev
