"""Seeded synthetic, grammar-valid MIDI-event token tensors.

Row 0 of every sequence is `[bos, 0 x 7]`; every later row is one event drawn
with the type mix note .85 / control_change .06 / patch_change .03 / set_tempo
.02 / time_signature .02 / key_signature .02, each parameter uniform in its id
range, padded with 0 to 8 ids -- the layout `event2tokens` produces
(reference `midi_tokenizer.py:920-928`).  Deterministic in (seed, shape).
"""
from __future__ import annotations

import numpy as np
import torch

_MIX = {"note": 0.85, "control_change": 0.06, "patch_change": 0.03, "set_tempo": 0.02,
        "time_signature": 0.02, "key_signature": 0.02}


def synth_batch(tok, batch: int, n_events: int, seed: int = 1234, pad_tail: int = 0) -> torch.Tensor:
    """int64 (batch, n_events, max_token_seq).  `pad_tail` trailing rows are all-pad (ragged sequences)."""
    rng = np.random.default_rng(seed)
    T = tok.max_token_seq
    names = [n for n in tok.events if n in _MIX]
    p = np.array([_MIX[n] for n in names], dtype=np.float64)
    p /= p.sum()
    out = np.zeros((batch, n_events, T), dtype=np.int64)
    out[:, 0, 0] = tok.bos_id
    n_real = n_events - pad_tail
    kinds = rng.choice(len(names), size=(batch, n_events), p=p)
    for ki, name in enumerate(names):
        sel = kinds == ki
        sel[:, 0] = False
        sel[:, n_real:] = False
        cnt = int(sel.sum())
        if cnt == 0:
            continue
        rows = np.zeros((cnt, T), dtype=np.int64)
        rows[:, 0] = tok.event_ids[name]
        for j, pname in enumerate(tok.events[name]):
            ids = tok.parameter_ids[pname]
            rows[:, 1 + j] = rng.integers(ids[0], ids[-1] + 1, size=cnt)
        out[sel] = rows
    return torch.from_numpy(out)


def random_ids(vocab: int, batch: int, n_events: int, T: int = 8, seed: int = 1234) -> torch.Tensor:
    """Uniform random ids in [0, vocab) -- pure kernel-parity variant."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, vocab, (batch, n_events, T), generator=g, dtype=torch.int64)
