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

The sample lengths are known here, before padding; passing them trains each sample on its own events only (ragged
batches, `b200_batch_to_xy_packed_i16` packs the rows that have a target):

    lengths = [len(s) for s in samples]
    batch = collate(samples, pad_id)
    loss = model.training_loss(batch.to("cuda"), lengths=lengths)     # lengths stay on the host

A pre-tokenised corpus (midi_b200/corpus.py) yields `(tokens, lengths, aug)` tuples; `augment_(tokens, aug)` then runs
train.py's augmentation on the device batch.
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

    An item may also be a tuple, such as the `(tokens, lengths, aug)` of `Corpus.batches`: each tensor in it is copied,
    everything else (`lengths`, a list that stays on the host) is passed through, and the tuple is yielded.
    """

    def __init__(self, batches: Iterable, device, depth: int = 2):
        self.it: Iterator = iter(batches)
        self.device = torch.device(device)
        self.depth = max(1, int(depth))
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.queue: list = []

    def _issue(self) -> bool:
        try:
            item = next(self.it)
        except StopIteration:
            return False
        parts = item if isinstance(item, tuple) else (item,)
        host = tuple(p.pin_memory() if isinstance(p, torch.Tensor) and not p.is_pinned() else p for p in parts)
        with torch.cuda.stream(self.copy_stream):
            dev = tuple(p.to(self.device, non_blocking=True) if isinstance(p, torch.Tensor) else p for p in host)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.queue.append((dev, ev, host, isinstance(item, tuple)))   # `host` stays referenced until its copy is consumed
        return True

    def __iter__(self):
        while len(self.queue) < self.depth and self._issue():
            pass
        while self.queue:
            dev, ev, _host, is_tuple = self.queue.pop(0)
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ev)
            for p in dev:
                if isinstance(p, torch.Tensor):
                    p.record_stream(cur)            # allocated on the copy stream, consumed on the compute stream
            self._issue()
            yield dev if is_tuple else dev[0]


_AUG_IDS = None


def augment_ids(tok=None):
    """The `lib.AugmentIds` of the v2 token layout (event ids and first parameter ids)."""
    from . import lib
    from .tokenizer_tables import TokenizerTables
    tok = tok or TokenizerTables("v2")
    if tok.version != "v2":
        raise lib.B200Error(f"augment: the {tok.version} tokenizer is not supported (its augment differs); v2 only")
    ev, pid = tok.event_ids, tok.parameter_ids
    return lib.AugmentIds(*(ev[e] for e in ("note", "patch_change", "control_change", "set_tempo", "key_signature")),
                          *(pid[p][0] for p in ("track", "channel", "pitch", "velocity", "controller", "value", "bpm", "sf",
                                                "mi")))


def augment_(batch: torch.Tensor, aug: torch.Tensor) -> torch.Tensor:
    """train.py's `MIDITokenizerV2.augment` of every sample of a device int16 batch `[B, L, T]`, in place, with the draws
    of `aug` (int32 `[B, 10]` on the same device, as `Corpus.batches` yields it).  Returns `batch`.

    The corpus metadata carries the two rules that depend on the whole file (the abort when a pitch shift moves a non-drum
    note out of 0..127, and sf = 0 on drum-only tracks), so augmenting a crop gives, row for row, the crop of the
    reference's augmented file.  Pad, BOS and EOS rows are left alone."""
    global _AUG_IDS
    from . import ops
    if _AUG_IDS is None:
        _AUG_IDS = augment_ids()
    return ops.augment_(batch, aug, _AUG_IDS)
