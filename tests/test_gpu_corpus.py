"""GPU tests (`pytest -m gpu`) of train.py's augmentation on the device (`data.augment_`, kernel `b200_augment_i16`) and of
the corpus loader feeding the fused trainer.

The kernel must equal `augment_v2` (tests/augment_reference.py) bit for bit: on every case of tests/golden/augment_v2.npz (the reference's
own `augment` with forced draws), and on random sequences for every (pitch, channel) shift pair.  Cropping then augmenting
on the device must equal `augment_v2` of the whole file then cropping; pad, BOS and EOS rows and positions at
or beyond a sample's length must come back unchanged.  End to end, loader -> Prefetcher -> augment_ -> training_loss(batch,
lengths) must see the very batch `augment_v2` augments on the host, so the loss and every GEMM-produced gradient are
bit-identical; RMSNorm-weight and embedding gradients are summed with fp32 atomics in a run-dependent order and get the
1e-3 global relative bound of the other trainer tests."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from parity_metrics import assert_within

BOUNDS = [
    ("aug_mismatch", 0.0),             # elements of the device batch that differ from augment_v2's
    ("batch_mismatch", 0.0),           # device-augmented batch vs the host-augmented one
    ("loss_mismatch", 0.0),
    ("gemm_grad_mismatch", 0.0),
    ("atomic_grad_rel", 1e-3),
]


def _dev_augment(tokens: np.ndarray, aug: np.ndarray) -> np.ndarray:
    import torch
    from midi_b200 import data
    b = torch.from_numpy(np.ascontiguousarray(tokens, np.int16)).cuda()
    a = torch.from_numpy(np.ascontiguousarray(aug, np.int32)).cuda()
    data.augment_(b, a)
    torch.cuda.synchronize()
    return b.cpu().numpy().astype(np.int64)


def _aug_row(meta, shifts, skip=None):
    from midi_b200 import corpus as CO, lib
    from test_corpus_host import _aborted
    a = np.zeros(lib.AUG_COLS, np.int32)
    a[lib.AUG_PITCH:lib.AUG_CHANNEL + 1] = shifts
    a[lib.AUG_SKIP] = _aborted(meta, shifts[0]) if skip is None else skip
    a[lib.AUG_DRUM:] = meta[CO.META_DRUM:]
    return a


@pytest.mark.gpu
def test_kernel_golden_cases():
    from midi_b200 import corpus as CO
    from midi_b200.tokenizer_tables import TokenizerTables
    from test_corpus_host import _oracle_batch
    tok = TokenizerTables("v2")
    g = dict(np.load(os.path.join(GOLDEN, "augment_v2.npz")))
    toks, off, cases, out, oo = g["tokens"], g["offsets"], g["cases"], g["out"], g["out_offsets"]
    L = int(np.diff(off).max()) + 3
    batch = np.full((len(cases), L, toks.shape[1]), tok.pad_id, np.int16)
    aug, lengths, ref = [], [], []
    for i, (f, ps, vs, cs, bs, _ts, ch) in enumerate(cases):
        rows = toks[off[f]:off[f + 1]]
        batch[i, :len(rows)] = rows
        aug.append(_aug_row(CO.file_meta(tok, rows.astype(np.int64)), (ps, vs, cs, bs, ch)))
        lengths.append(len(rows))
        ref.append(out[oo[i]:oo[i + 1]])
    aug = np.stack(aug)
    got = _dev_augment(batch, aug)
    want = _oracle_batch(batch, lengths, aug)
    m = {"aug_mismatch_oracle": float((got != want).sum()),
         "aug_mismatch_reference": float(sum(int((got[i, :n] != r).sum()) for i, (n, r) in enumerate(zip(lengths, ref)))),
         "aug_mismatch_pad_tail": float(sum(int((got[i, n:] != tok.pad_id).sum()) for i, n in enumerate(lengths)))}
    assert aug[:, 0].any() and not aug[:, 0].all()
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_kernel_random_every_shift():
    """Random well-formed rows, BOS / EOS / pad rows among them, for all 153 (pitch, channel) pairs with random velocity /
    cc value / bpm shifts, random skip flags and random drum masks."""
    from midi_b200.tokenizer_tables import TokenizerTables
    from test_corpus_host import _event_rows, _oracle_batch
    tok = TokenizerTables("v2")
    rng = np.random.default_rng(11)
    pairs = [(p, c) for p in range(-4, 5) for c in range(17)]
    B, L = len(pairs) * 2, 257
    batch = np.empty((B, L, tok.max_token_seq), np.int16)
    aug = np.zeros((B, 10), np.int32)
    special = {0: tok.pad_id, 1: tok.bos_id, 2: tok.eos_id}
    for b in range(B):
        rows = np.asarray(_event_rows(rng, L), np.int16)
        for r in rng.choice(L, 12, replace=False):
            rows[r] = special[int(r) % 3]
            rows[r, 1:] = tok.pad_id
        batch[b] = rows
        p, c = pairs[b % len(pairs)]
        aug[b, 0] = b >= len(pairs) and rng.random() < 0.3
        aug[b, 1:6] = (p, rng.integers(-10, 11), rng.integers(-10, 11), rng.integers(-10, 11), c)
        aug[b, 6:] = rng.integers(-2 ** 31, 2 ** 31, 4)
    # pitches in range after any shift, as the host guarantees for a sample it does not skip
    d = tok.parameter_ids["pitch"][0]
    note = batch[..., 0] == tok.event_ids["note"]
    batch[..., 5] = np.where(note, d + 4 + (batch[..., 5] - d) % 120, batch[..., 5])
    got = _dev_augment(batch, aug)
    want = _oracle_batch(batch, [L] * B, aug)
    untouched = ~np.isin(batch[..., 0], list(tok.event_ids.values()))
    m = {"aug_mismatch_random": float((got != want).sum()),
         "aug_mismatch_special_rows": float((got[untouched] != batch[untouched]).sum())}
    assert untouched.sum() >= B * 12 and (got != batch).any()
    assert_within(m, BOUNDS)


def _corpus(tmp_path):
    from midi_b200 import corpus as CO
    from midi_b200.tokenizer_tables import TokenizerTables
    from test_corpus_host import _build
    rng = np.random.default_rng(5)
    lengths = [int(x) for x in rng.integers(1, 1200, 30)]
    return CO.Corpus(_build(tmp_path, lengths), TokenizerTables("v2"))


@pytest.mark.gpu
def test_crop_then_augment_equals_augment_then_crop(tmp_path):
    import torch
    from midi_b200 import data, lib
    import augment_reference as AR
    from test_corpus_host import _drum_bits
    corpus = _corpus(tmp_path)
    pad = corpus.pad_id
    m = {"aug_mismatch_crop": 0.0, "aug_mismatch_tail": 0.0}
    n_skip = n_run = 0
    for epoch in range(3):
        plan = corpus.plan(500, seed=1, epoch=epoch)
        i = 0
        for tokens, lengths, aug in data.Prefetcher(corpus.batches(7, 500, seed=1, epoch=epoch), "cuda"):
            data.augment_(tokens, aug)
            got = tokens.cpu().numpy().astype(np.int64)
            a_np = aug.cpu().numpy()
            for b, n in enumerate(lengths):
                f, s, a = plan[0][i + b], plan[1][i + b], a_np[b]
                whole = AR.augment_v2(corpus.file(f), a[lib.AUG_PITCH:lib.AUG_CHANNEL + 1], bool(a[lib.AUG_SKIP]),
                                     _drum_bits(a[lib.AUG_DRUM:]))
                m["aug_mismatch_crop"] += float((got[b, :n] != whole[s:s + n]).sum())
                m["aug_mismatch_tail"] += float((got[b, n:] != pad).sum())
                n_skip += int(a[lib.AUG_SKIP])
            i += len(lengths)
        assert i == len(corpus)
        n_run += i
    assert 0 < n_skip < n_run
    torch.cuda.synchronize()
    assert_within(m, BOUNDS)


@pytest.mark.gpu
def test_loader_augment_training_loss_end_to_end(tmp_path):
    import torch
    import gpu_model as GM
    from midi_b200 import data
    from test_corpus_host import _oracle_batch
    corpus = _corpus(tmp_path)
    model = GM.cuda_model()
    loader = corpus.batches(4, 700, seed=7, epoch=0)
    host = [loader.batch(i) for i in range(2)]          # the same batches, augmented on the host by augment_v2
    loader.close()
    m = {}
    for i, (tokens, lengths, aug) in enumerate(data.Prefetcher(corpus.batches(4, 700, seed=7, epoch=0), "cuda")):
        if i == 2:
            break
        data.augment_(tokens, aug)
        h_tok, h_len, h_aug = host[i]
        assert h_len == lengths and torch.equal(h_aug, aug.cpu())
        ref = torch.from_numpy(_oracle_batch(h_tok.numpy(), h_len, h_aug.numpy()).astype(np.int16)).cuda()
        m[f"batch_mismatch_{i}"] = float((tokens != ref).sum())
        dev = GM.step(model, lambda gr: model.training_loss(tokens, lengths=lengths, grad_ready=gr))
        hst = GM.step(model, lambda gr: model.training_loss(ref, lengths=h_len, grad_ready=gr))
        m.update(GM.exact(dev, hst, f"e2e_{i}"))
        assert bool(torch.isfinite(dev[0]))
    assert_within(m, BOUNDS)
