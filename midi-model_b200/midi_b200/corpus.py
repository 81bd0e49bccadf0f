"""Pre-tokenised MIDI corpus for the fused trainer: train.py's data path (train.py:31-90, 398-425) with the parsing done once.

train.py's `MidiDataset` re-reads, parses (`MIDI.midi2score`), tokenises, augments and crops every file in every epoch,
about 0.1-0.2 s of CPU per sample.  Here the files are tokenised once into one int16 matrix on disk; per step the host
only crops the memory-mapped rows and copies them into a pinned batch, and the augmentation runs on the GPU, in place,
on the batch already there (`data.augment_`, kernel `b200_augment_i16`):

    build_corpus(train_paths, "corpus/train", model.tokenizer, workers=16)            # once
    corpus = Corpus("corpus/train", model.tokenizer)
    for tokens, lengths, aug in data.Prefetcher(corpus.batches(8, 2048, epoch=epoch), "cuda"):
        data.augment_(tokens, aug)
        loss = model.training_loss(tokens, lengths=lengths)

On disk (`out_dir`):
  tokens.npy    int16 [total_events, T]: every kept file's token rows, BOS and EOS included, one file after another;
  offsets.npy   int64 [n_files + 1]: file i is rows offsets[i]:offsets[i+1];
  meta.npy      int32 [n_files, 6]: what the augmentation needs about the whole file -- the min and max pitch of the notes
                whose original channel is not 9 (128 and -1 when there is none) and the 128-bit mask of its drum-only
                tracks (every note on channel 9, at least one note) as four 32-bit words;
  paths.txt     the source path of each kept file, one per line;
  manifest.json tokenizer version, optimise_midi, T, vocab size, file and event counts, and the skip count per reason.

A file is kept when `MidiDataset.load_midi` would accept it: size within 3000..384000 bytes, a parse, a non-empty track,
a tokenisation and, with `quality=True`, `check_quality`.  Every row must also be well-formed (BOS / EOS, or a known event
id with each parameter token in its range and pads after).  The reference replaces a file that fails with a random other
file; the corpus drops it and counts it in the manifest.  Only the v2 tokenizer is supported: v1's augment differs.
"""
from __future__ import annotations

import json
import os
import queue
import random
import struct
import threading
import time
from concurrent.futures import ProcessPoolExecutor
from functools import partial
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import lib
from .data import collate

FORMAT = 1
MIN_FILE_SIZE, MAX_FILE_SIZE = 3000, 384000                   # MidiDataset defaults (train.py:32-33)
SKIP_REASONS = ("read_error", "too_large", "too_small", "parse_error", "empty_track", "tokenize_error", "bad_quality",
                "malformed")
META_PITCH_MIN, META_PITCH_MAX, META_DRUM = 0, 1, 2           # meta.npy columns; META_DRUM.. META_DRUM + 3: the mask
META_COLS = 6
EXTENSION = (".mid", ".midi")

# augmentation ranges of train.py (MIDITokenizerV2.augment defaults; track shift 0)
PITCH_SHIFT, VEL_SHIFT, CC_VAL_SHIFT, BPM_SHIFT, CHANNEL_SHIFT = 4, 10, 10, 10, 16


def _require_v2(version: str, what: str):
    if version != "v2":
        raise lib.B200Error(f"{what}: a {version} corpus is not supported: only the v2 tokenizer's augmentation runs on "
                            "the device")


# ------------------------------------------------------------------ building
class _RowCheck:
    """Well-formedness of token rows as one lookup: for each possible token 0 (pad, BOS, EOS, the event ids) the allowed
    half-open id range of every position."""

    def __init__(self, tok):
        T = tok.max_token_seq
        n0 = max(tok.event_ids.values()) + 1
        pad = tok.pad_id
        self.lo = np.full((n0, T), pad, np.int64)
        self.hi = np.full((n0, T), pad + 1, np.int64)
        self.ok0 = np.zeros(n0, bool)
        for i in (tok.bos_id, tok.eos_id):
            self.ok0[i] = True
            self.lo[i, 0], self.hi[i, 0] = i, i + 1
        for name, i in tok.event_ids.items():
            self.ok0[i] = True
            self.lo[i, 0], self.hi[i, 0] = i, i + 1
            for j, p in enumerate(tok.events[name]):
                ids = tok.parameter_ids[p]
                self.lo[i, 1 + j], self.hi[i, 1 + j] = ids[0], ids[-1] + 1

    def __call__(self, a: np.ndarray) -> bool:
        t0 = a[:, 0]
        if (t0 < 0).any() or (t0 >= len(self.ok0)).any() or not self.ok0[t0].all():
            return False
        return bool(((a >= self.lo[t0]) & (a < self.hi[t0])).all())


def file_meta(tok, a: np.ndarray) -> np.ndarray:
    """The meta.npy row of one file's token rows `a` [n, T]: non-drum pitch range and drum-only track mask."""
    ev = tok.events["note"]
    c_track, c_ch, c_pitch = (1 + ev.index(p) for p in ("track", "channel", "pitch"))
    notes = a[a[:, 0] == tok.event_ids["note"]].astype(np.int64)
    tr = notes[:, c_track] - tok.parameter_ids["track"][0]
    ch = notes[:, c_ch] - tok.parameter_ids["channel"][0]
    p = notes[:, c_pitch] - tok.parameter_ids["pitch"][0]
    out = np.zeros(META_COLS, np.int32)
    melodic = ch != 9
    out[META_PITCH_MIN] = p[melodic].min() if melodic.any() else 128
    out[META_PITCH_MAX] = p[melodic].max() if melodic.any() else -1
    drum_only = np.zeros(128, bool)
    drum_only[tr] = True
    drum_only[tr[melodic]] = False
    words = np.zeros(4, np.uint32)
    for t in np.flatnonzero(drum_only):
        words[t >> 5] |= np.uint32(1 << (t & 31))
    out[META_DRUM:META_DRUM + 4] = words.view(np.int32)
    return out


def _load_one(path: str, tok, quality: bool, midi2score: Callable):
    """`MidiDataset.load_midi` without the augmentation: (tokens int16 [n, T], meta row) or the reason it is skipped."""
    try:
        with open(path, "rb") as f:
            datas = f.read()
    except OSError:
        return "read_error"
    if len(datas) > MAX_FILE_SIZE:
        return "too_large"
    if len(datas) < MIN_FILE_SIZE:
        return "too_small"
    try:
        mid = midi2score(datas)
        empty = max([0] + [len(track) for track in mid[1:]]) == 0
    except Exception:
        return "parse_error"
    if empty:
        return "empty_track"
    try:
        seq = tok.tokenize(mid)
    except Exception:
        return "tokenize_error"
    if quality:
        try:
            good = tok.check_quality(seq)[0]
        except Exception:
            good = False
        if not good:
            return "bad_quality"
    try:
        a = np.asarray(seq, dtype=np.int64)
    except (ValueError, TypeError, OverflowError):
        return "malformed"
    if a.ndim != 2 or a.shape[0] == 0 or a.shape[1] != tok.max_token_seq or not _RowCheck(tok)(a):
        return "malformed"
    return a.astype(np.int16), file_meta(tok, a)


def _npy_header(shape, total: int = 128) -> bytes:
    """A version-1.0 .npy header for little-endian int16 data of `shape`, padded to `total` bytes, so that the shape can
    be rewritten in place once the streamed row count is known."""
    d = "{'descr': '<i2', 'fortran_order': False, 'shape': %r, }" % (tuple(shape),)
    body = d.ljust(total - 11) + "\n"
    return b"\x93NUMPY\x01\x00" + struct.pack("<H", len(body)) + body.encode("latin1")


def build_corpus(paths: Sequence[str], out_dir: str, tokenizer, quality: bool = False, workers: int = 1,
                 midi2score: Optional[Callable] = None) -> dict:
    """Tokenise `paths` once with the caller's `tokenizer` (the reference's MIDITokenizerV2 in a train.py environment) into
    `out_dir` (see the module docstring).  Files are kept in the order of `paths`.  `workers` > 1 parses in that many
    processes.  `midi2score` parses the bytes of a file; by default it is `MIDI.midi2score`, the parser train.py imports.
    Returns the manifest."""
    _require_v2(tokenizer.version, "build_corpus")
    if midi2score is None:
        try:
            import MIDI                                    # train.py's parser module, on sys.path next to train.py
        except ImportError as e:
            raise lib.B200Error("build_corpus: no midi2score given and the `MIDI` module train.py uses is not "
                                "importable") from e
        midi2score = MIDI.midi2score
    T = tokenizer.max_token_seq
    os.makedirs(out_dir, exist_ok=True)
    skipped = {r: 0 for r in SKIP_REASONS}
    offsets: List[int] = [0]
    metas: List[np.ndarray] = []
    kept: List[str] = []
    load = partial(_load_one, tok=tokenizer, quality=quality, midi2score=midi2score)
    tok_path = os.path.join(out_dir, "tokens.npy")
    with open(tok_path, "wb") as f:
        f.write(_npy_header((0, T)))
        pool = ProcessPoolExecutor(workers) if workers > 1 else None
        try:
            results = pool.map(load, paths, chunksize=16) if pool else map(load, paths)
            for path, r in zip(paths, results):
                if isinstance(r, str):
                    skipped[r] += 1
                    continue
                a, m = r
                f.write(a.astype("<i2").tobytes())
                offsets.append(offsets[-1] + a.shape[0])
                metas.append(m)
                kept.append(str(path))
        finally:
            if pool:
                pool.shutdown()
        f.seek(0)
        f.write(_npy_header((offsets[-1], T)))
    np.save(os.path.join(out_dir, "offsets.npy"), np.asarray(offsets, np.int64))
    np.save(os.path.join(out_dir, "meta.npy"), np.stack(metas) if metas else np.zeros((0, META_COLS), np.int32))
    with open(os.path.join(out_dir, "paths.txt"), "w") as f:
        f.writelines(p.replace("\n", " ") + "\n" for p in kept)
    manifest = {"format": FORMAT, "tokenizer_version": tokenizer.version,
                "optimise_midi": bool(tokenizer.optimise_midi), "T": T, "vocab_size": tokenizer.vocab_size,
                "quality": bool(quality), "n_files": len(kept), "n_events": offsets[-1], "skipped": skipped}
    with open(os.path.join(out_dir, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    return manifest


def get_midi_list(path: str) -> List[str]:
    """train.py:273-283: every .mid / .midi file under `path`, sorted."""
    files = {os.path.join(root, f) for root, _dirs, names in os.walk(path) for f in names}
    return sorted(f for f in files if os.path.splitext(f)[1].lower() in EXTENSION)


def split_midi_list(path: str, data_val_split: int, seed: int = 0):
    """train.py's split (train.py:391-403): `get_midi_list`, `random.seed(seed)` (`pl.seed_everything`), `random.shuffle`;
    the last `data_val_split` files are the validation set.  Returns (train_paths, val_paths)."""
    paths = get_midi_list(path)
    random.Random(seed).shuffle(paths)
    n_train = len(paths) - data_val_split
    return paths[:n_train], paths[n_train:]


# ------------------------------------------------------------------ loading
def _mix(x: np.ndarray) -> np.ndarray:
    """splitmix64's finaliser on uint64 arrays (wrapping arithmetic)."""
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def draws(seed: int, epoch: int, positions: np.ndarray, n: int) -> np.ndarray:
    """Counter-based uint64 draws [len(positions), n], a function of (seed, epoch, position) only."""
    pos = np.asarray(positions, dtype=np.uint64)
    h = _mix(np.full(pos.shape, seed & (2 ** 64 - 1), np.uint64) + np.uint64(0x9E3779B97F4A7C15))
    h = _mix(h ^ np.uint64(epoch & (2 ** 64 - 1)))
    h = _mix(h ^ pos)
    return np.stack([_mix(h ^ np.uint64((j + 1) * 0x9E3779B97F4A7C15 % 2 ** 64)) for j in range(n)], axis=1)


class Corpus:
    """A corpus written by `build_corpus`, memory-mapped.  The manifest must match `tokenizer` (version, optimise_midi,
    tokens per event, vocabulary size); a v1 corpus raises."""

    def __init__(self, path: str, tokenizer):
        with open(os.path.join(path, "manifest.json")) as f:
            m = json.load(f)
        self.manifest = m
        _require_v2(m.get("tokenizer_version"), "Corpus")
        if m.get("format") != FORMAT:
            raise lib.B200Error(f"Corpus: format {m.get('format')} in {path}, expected {FORMAT}")
        want = {"tokenizer_version": tokenizer.version, "optimise_midi": bool(tokenizer.optimise_midi),
                "T": tokenizer.max_token_seq, "vocab_size": tokenizer.vocab_size}
        bad = {k: (m.get(k), v) for k, v in want.items() if m.get(k) != v}
        if bad:
            raise lib.B200Error(f"Corpus: {path} was built for another tokenizer: " +
                                ", ".join(f"{k} {a!r} (tokenizer: {b!r})" for k, (a, b) in bad.items()))
        self.tokens = np.load(os.path.join(path, "tokens.npy"), mmap_mode="r")
        self.offsets = np.load(os.path.join(path, "offsets.npy"))
        self.meta = np.load(os.path.join(path, "meta.npy"))
        n = m["n_files"]
        if self.tokens.shape != (m["n_events"], m["T"]) or self.offsets.shape != (n + 1,) or self.meta.shape != (n, META_COLS) \
                or self.offsets[-1] != m["n_events"]:
            raise lib.B200Error(f"Corpus: the arrays in {path} do not match its manifest")
        self.pad_id = tokenizer.pad_id

    def __len__(self) -> int:
        return len(self.offsets) - 1

    def file(self, i: int) -> np.ndarray:
        """The token rows of file i (a view of the memory map)."""
        return self.tokens[self.offsets[i]:self.offsets[i + 1]]

    def plan(self, max_len: int = 2048, *, train: bool = True, seed: int = 0, epoch: int = 0, rank: int = 0,
             world_size: int = 1):
        """This rank's samples of one epoch, in order: (file int64 [n], start int64 [n], length int64 [n],
        aug int32 [n, lib.AUG_COLS]).

        train=True: the files in a permutation drawn from (seed, epoch); crop start `choice([0, randrange(0, max(1, n_b -
        max_len))])` (train.py's rand_start); augmentation draws in train.py's ranges, the sample skipped when its pitch
        shift would move a non-drum note of the file out of 0..127.  Every draw is a function of (seed, epoch, position
        in the epoch).  train=False (validation): the files in order, start `(i * (max_start // 8)) % max_start` with
        max_start = max(1, n_i - max_len), no augmentation (every sample skipped).  Ranks split the epoch as
        DistributedSampler does: padded by wrap-around to a multiple of world_size, rank r takes positions r, r + ws, ..."""
        if not 0 <= rank < world_size:
            raise lib.B200Error(f"plan: rank {rank} outside world size {world_size}")
        if max_len < 1:
            raise lib.B200Error(f"plan: max_len {max_len} < 1")
        n = len(self)
        if n == 0:
            raise lib.B200Error("plan: the corpus has no files")
        order = np.random.default_rng([seed & (2 ** 63 - 1), epoch]).permutation(n) if train else np.arange(n)
        total = -(-n // world_size) * world_size
        pos = np.arange(rank, total, world_size, dtype=np.int64)
        files = order[pos % n].astype(np.int64)
        n_ev = self.offsets[files + 1] - self.offsets[files]
        aug = np.zeros((len(files), lib.AUG_COLS), np.int32)
        if train:
            u = draws(seed, epoch, pos, 7)
            r = (u[:, 0] % np.maximum(1, n_ev - max_len).astype(np.uint64)).astype(np.int64)
            start = np.where(u[:, 1] & np.uint64(1), r, 0)
            pitch = (u[:, 2] % np.uint64(2 * PITCH_SHIFT + 1)).astype(np.int64) - PITCH_SHIFT
            aug[:, lib.AUG_PITCH] = pitch
            aug[:, lib.AUG_VELOCITY] = (u[:, 3] % np.uint64(2 * VEL_SHIFT + 1)).astype(np.int64) - VEL_SHIFT
            aug[:, lib.AUG_CC_VALUE] = (u[:, 4] % np.uint64(2 * CC_VAL_SHIFT + 1)).astype(np.int64) - CC_VAL_SHIFT
            aug[:, lib.AUG_BPM] = (u[:, 5] % np.uint64(2 * BPM_SHIFT + 1)).astype(np.int64) - BPM_SHIFT
            aug[:, lib.AUG_CHANNEL] = (u[:, 6] % np.uint64(CHANNEL_SHIFT + 1)).astype(np.int64)
            pmin = self.meta[files, META_PITCH_MIN].astype(np.int64)
            pmax = self.meta[files, META_PITCH_MAX].astype(np.int64)
            aug[:, lib.AUG_SKIP] = (pmin <= pmax) & ((pmin + pitch < 0) | (pmax + pitch > 127))
            aug[:, lib.AUG_DRUM:lib.AUG_DRUM + 4] = self.meta[files, META_DRUM:META_DRUM + 4]
        else:
            max_start = np.maximum(1, n_ev - max_len)
            start = (files * (max_start // 8)) % max_start
            aug[:, lib.AUG_SKIP] = 1
        length = np.minimum(max_len, n_ev - start)
        return files, start, length, aug

    def batches(self, batch_size: int, max_len: int = 2048, *, train: bool = True, seed: int = 0, epoch: int = 0,
                rank: int = 0, world_size: int = 1, depth: int = 4) -> "BatchLoader":
        """One epoch of `plan(...)` as batches `(tokens int16 [B, L_max, T] pinned, lengths list of B ints, aug int32
        [B, lib.AUG_COLS] pinned)`, gathered by one background thread up to `depth` batches ahead.  The last batch may be
        smaller.  Feed it to `data.Prefetcher`, then `data.augment_(tokens, aug)` on the device."""
        if batch_size < 1:
            raise lib.B200Error(f"batches: batch_size {batch_size} < 1")
        return BatchLoader(self, self.plan(max_len, train=train, seed=seed, epoch=epoch, rank=rank,
                                           world_size=world_size), batch_size, depth)


_END = object()


def _make_batch(corpus: Corpus, plan, batch_size: int, i: int):
    files, start, length, aug = (a[i * batch_size:(i + 1) * batch_size] for a in plan)
    off = corpus.offsets[files] + start
    tokens = collate([corpus.tokens[o:o + n] for o, n in zip(off, length)], corpus.pad_id)
    a = torch.empty(aug.shape, dtype=torch.int32, pin_memory=torch.cuda.is_available())
    a.numpy()[...] = aug
    return tokens, [int(n) for n in length], a


def _produce(q: queue.Queue, stop: threading.Event, make: Callable, n: int, host_s: List[float]):
    """The loader thread.  It holds no reference to its BatchLoader, so dropping the loader stops it."""
    def put(item) -> bool:
        while not stop.is_set():
            try:
                q.put(item, timeout=0.05)
                return True
            except queue.Full:
                pass
        return False

    try:
        for i in range(n):
            t0 = time.perf_counter()
            item = make(i)
            host_s.append(time.perf_counter() - t0)
            if not put(item):
                return
        put(_END)
    except BaseException as e:                 # re-raised in the consumer's thread
        put(e)


class BatchLoader:
    """Iterator over the batches of a plan, built by one daemon thread (crop from the memory map + `data.collate` into
    pinned memory).  `host_s` records the thread's time per batch.  Exhausting it, `close()` or dropping it stops the
    thread."""

    def __init__(self, corpus: Corpus, plan, batch_size: int, depth: int = 4):
        self.n_batches = -(-len(plan[0]) // batch_size)
        self.batch = partial(_make_batch, corpus, plan, batch_size)     # batch i, built in the calling thread
        self.host_s: List[float] = []
        self._q: queue.Queue = queue.Queue(maxsize=max(1, depth))
        self._stop = threading.Event()
        self._thread = threading.Thread(target=_produce, args=(self._q, self._stop, self.batch, self.n_batches, self.host_s),
                                        name="corpus-loader", daemon=True)
        self._thread.start()

    def __len__(self) -> int:
        return self.n_batches

    def __iter__(self):
        return self

    def __next__(self):
        if self._stop.is_set():
            raise StopIteration
        item = self._q.get()
        if item is _END:
            self.close()
            raise StopIteration
        if isinstance(item, BaseException):
            self.close()
            raise item
        return item

    def close(self):
        self._stop.set()
        self._thread.join()

    def __del__(self):
        self._stop.set()
