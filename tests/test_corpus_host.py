"""Host tests of the pre-tokenised corpus (midi_b200/corpus.py) and of train.py's augmentation restated in
tests/augment_reference.py: `augment_v2` against the reference's own `augment` (tests/golden/augment_v2.npz), the
builder's files, the loader's epoch order, crops, draws, rank shares and abort flags, the manifest checks, and
`data.augment_`'s call of `b200_augment_i16` through a mock of that entry kept in this file."""
import ctypes
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

import augment_reference as AR
from conftest import GOLDEN
from midi_b200 import corpus as CO, data, lib
from midi_b200.tokenizer_tables import TokenizerTables
from oracle import ref_loader

TOK = TokenizerTables("v2")
T = TOK.max_token_seq


def _drum_bits(words) -> np.ndarray:
    w = np.asarray(words, np.int32).view(np.uint32).astype(np.int64)
    return np.array([(w[t >> 5] >> (t & 31)) & 1 for t in range(128)], bool)


def _aborted(meta, pitch) -> bool:
    lo, hi = int(meta[CO.META_PITCH_MIN]), int(meta[CO.META_PITCH_MAX])
    return lo <= hi and (lo + pitch < 0 or hi + pitch > 127)


def _oracle_batch(tokens, lengths, aug):
    """augment_v2 on each sample's first lengths[b] rows of a [B, L, T] batch; the rest unchanged."""
    out = np.array(tokens, np.int64)
    for b, n in enumerate(lengths):
        a = aug[b]
        out[b, :n] = AR.augment_v2(out[b, :n], a[lib.AUG_PITCH:lib.AUG_CHANNEL + 1], bool(a[lib.AUG_SKIP]),
                                  _drum_bits(a[lib.AUG_DRUM:lib.AUG_DRUM + 4]))
    return out


# ------------------------------------------------------------------ the restatement against the reference
@pytest.fixture(scope="module")
def golden_aug():
    return dict(np.load(os.path.join(GOLDEN, "augment_v2.npz")))


def test_augment_v2_equals_reference(golden_aug):
    g = golden_aug
    toks, off, cases, out, oo = g["tokens"], g["offsets"], g["cases"], g["out"], g["out_offsets"]
    seen = set()
    n_abort = n_kept = 0
    for i, (f, ps, vs, cs, bs, ts, ch) in enumerate(cases):
        rows = toks[off[f]:off[f + 1]]
        ref = out[oo[i]:oo[i + 1]]
        meta = CO.file_meta(TOK, rows.astype(np.int64))
        ab = _aborted(meta, ps)
        got = AR.augment_v2(rows, (ps, vs, cs, bs, ch), ab, _drum_bits(meta[CO.META_DRUM:]))
        np.testing.assert_array_equal(got, ref, err_msg=f"case {i}: file {g['names'][f]} shifts {ps, vs, cs, bs, ch}")
        # crop then augment == augment then crop, for every crop boundary pair of a coarse grid
        for s in range(0, len(rows), 97):
            for e in (s + 1, s + 200, len(rows)):
                np.testing.assert_array_equal(AR.augment_v2(rows[s:e], (ps, vs, cs, bs, ch), ab,
                                                           _drum_bits(meta[CO.META_DRUM:])), ref[s:e])
        if ab:
            n_abort += 1
            np.testing.assert_array_equal(ref, rows)
        else:
            n_kept += 1
        seen.add((int(ps), int(ch)))
    assert seen == {(p, c) for p in range(-4, 5) for c in range(17)}
    assert n_abort >= 2 * 2 * 17 and n_kept > n_abort
    assert {-10, 0, 10} <= set(cases[:, 2]) and {-10, 0, 10} <= set(cases[:, 3]) and {-10, 0, 10} <= set(cases[:, 4])


def test_augment_v2_fixture_covers_the_rules(golden_aug):
    """The fixture reaches the traps: velocity / cc value / bpm 0 clamped to 1 under a zero shift, negative sf, drum-only
    key signatures, drum notes beyond 0..127 after the shift in a file that does not abort."""
    g = golden_aug
    d = AR.V2_IDS
    rows = g["tokens"].astype(np.int64)
    ev = rows[:, 0]
    assert (rows[ev == d["note"], 6] == d["velocity"]).any()
    assert ((ev == d["control_change"]) & (rows[:, 6] == d["value"]) & np.isin(rows[:, 5] - d["controller"], [1, 2, 7, 11])).any()
    assert (rows[ev == d["set_tempo"], 4] == d["bpm"]).any()
    assert set(rows[ev == d["key_signature"], 4] - d["sf"]) == set(range(15))
    assert (ev == TOK.bos_id).sum() == 3 and (ev == TOK.eos_id).sum() == 3
    metas = [CO.file_meta(TOK, rows[g["offsets"][f]:g["offsets"][f + 1]]) for f in range(3)]
    assert [int(_drum_bits(m[CO.META_DRUM:]).sum()) for m in metas] == [1, 1, 2]
    assert metas[2][CO.META_PITCH_MIN] == 128 and metas[2][CO.META_PITCH_MAX] == -1   # 'drums': never aborts


def test_augment_v2_zero_shift_is_not_identity():
    d = AR.V2_IDS
    rows = np.array([[d["note"], d["time1"], d["time2"], d["track"], d["channel"] + 2, d["pitch"] + 60, d["velocity"], d["duration"]],
                     [d["set_tempo"], d["time1"], d["time2"], d["track"], d["bpm"], 0, 0, 0],
                     [d["control_change"], d["time1"], d["time2"], d["track"], d["channel"], d["controller"] + 7, d["value"], 0]])
    got = AR.augment_v2(rows, (0, 0, 0, 0, 0), False, np.zeros(128, bool))
    assert got[0, 6] == d["velocity"] + 1 and got[1, 4] == d["bpm"] + 1 and got[2, 6] == d["value"] + 1
    np.testing.assert_array_equal(AR.augment_v2(rows, (0, 0, 0, 0, 0), True, np.zeros(128, bool)), rows)


# ------------------------------------------------------------------ a stub tokenizer and parser for the builder
def _event_rows(rng, n):
    """n random well-formed v2 event rows (notes on channels incl. 9, other events)."""
    names = list(TOK.events)
    rows = []
    for _ in range(n):
        name = names[int(rng.integers(len(names)))]
        vals = [int(rng.integers(TOK.event_parameters[p])) for p in TOK.events[name]]
        if name == "note":
            vals[TOK.events["note"].index("track")] = int(rng.integers(4))
            vals[TOK.events["note"].index("pitch")] = int(rng.integers(2, 126))   # some pitch shifts abort, some not
        rows.append(TOK.event2tokens([name] + vals))
    return rows


def stub_midi2score(datas: bytes):
    """File format of these tests: b'<kind> <seed> <n events>' padded with spaces.  The 'score' carries the rows."""
    kind, seed, n = datas.decode().split()
    if kind == "garbage":
        raise ValueError("not a MIDI file")
    if kind == "empty":
        return [480, []]
    rows = _event_rows(np.random.default_rng(int(seed)), int(n))
    if kind == "malformed":
        rows[len(rows) // 2][1] = TOK.vocab_size + 5
    return [480, [kind] + rows]


class StubTokenizer(TokenizerTables):
    def __init__(self, version="v2"):
        super().__init__(version)

    def tokenize(self, score):
        kind, rows = score[1][0], score[1][1:]
        if kind == "raise":
            raise RuntimeError("tokenize failed")
        bos = [self.bos_id] + [self.pad_id] * (self.max_token_seq - 1)
        eos = [self.eos_id] + [self.pad_id] * (self.max_token_seq - 1)
        return [bos] + rows + [eos]

    def check_quality(self, seq):
        return len(seq) % 2 == 0, "odd"


def _write(path, kind, seed, n, size=3000):
    with open(path, "wb") as f:
        f.write(f"{kind} {seed} {n}".encode().ljust(size))
    return str(path)


def _build(tmp_path, lengths, name="c", seed=0, **kw):
    src = tmp_path / (name + "_src")
    src.mkdir()
    paths = [_write(src / f"{i}.mid", "ok", seed * 100000 + i, n) for i, n in enumerate(lengths)]
    out = str(tmp_path / name)
    CO.build_corpus(paths, out, StubTokenizer(), midi2score=stub_midi2score, **kw)
    return out


def test_builder_files_and_skips(tmp_path):
    src = tmp_path / "src"
    src.mkdir()
    paths = [_write(src / "a.mid", "ok", 1, 40), _write(src / "small.mid", "ok", 2, 5, size=2999),
             _write(src / "large.mid", "ok", 3, 5, size=384001), _write(src / "g.mid", "garbage", 0, 0),
             _write(src / "e.mid", "empty", 0, 0), _write(src / "r.mid", "raise", 4, 3),
             _write(src / "m.mid", "malformed", 5, 9), str(src / "missing.mid"), _write(src / "b.mid", "ok", 6, 1),
             _write(src / "q.mid", "ok", 7, 3), _write(src / "c.mid", "ok", 8, 300, size=384000)]
    tok = StubTokenizer()
    man = CO.build_corpus(paths, str(tmp_path / "out"), tok, midi2score=stub_midi2score)
    assert man["skipped"] == {"read_error": 1, "too_large": 1, "too_small": 1, "parse_error": 1, "empty_track": 1,
                              "tokenize_error": 1, "bad_quality": 0, "malformed": 1}
    kept = [(1, 40), (6, 1), (7, 3), (8, 300)]
    assert man["n_files"] == 4 and man["n_events"] == sum(n + 2 for _, n in kept)
    assert (man["tokenizer_version"], man["T"], man["optimise_midi"], man["vocab_size"]) == ("v2", T, False, TOK.vocab_size)
    c = CO.Corpus(str(tmp_path / "out"), tok)
    np.testing.assert_array_equal(c.offsets, np.cumsum([0] + [n + 2 for _, n in kept]))
    assert c.tokens.dtype == np.int16 and c.tokens.shape == (man["n_events"], T)
    for i, (seed, n) in enumerate(kept):
        want = np.asarray(tok.tokenize(stub_midi2score(f"ok {seed} {n}".encode())), np.int16)
        np.testing.assert_array_equal(c.file(i), want)
        np.testing.assert_array_equal(c.meta[i], CO.file_meta(tok, want.astype(np.int64)))
    with open(tmp_path / "out" / "paths.txt") as f:
        assert f.read().split("\n")[:-1] == [paths[0], paths[8], paths[9], paths[10]]
    man_q = CO.build_corpus(paths, str(tmp_path / "outq"), tok, quality=True, midi2score=stub_midi2score)
    assert man_q["skipped"]["bad_quality"] == 3 and man_q["n_files"] == 2 and man_q["quality"]   # odd row counts
    man_w = CO.build_corpus(paths, str(tmp_path / "outw"), tok, workers=2, midi2score=stub_midi2score)
    assert man_w == man
    for f in ("tokens.npy", "offsets.npy", "meta.npy"):
        np.testing.assert_array_equal(np.load(tmp_path / "outw" / f), np.load(tmp_path / "out" / f))


def test_file_meta():
    d = AR.V2_IDS

    def note(tr, ch, p):
        return TOK.event2tokens(["note", 0, 0, tr, ch, p, 50, 1])
    rows = np.array([note(0, 9, 0), note(0, 9, 127), note(1, 9, 30), note(1, 2, 40), note(2, 5, 70), note(100, 9, 3),
                     note(33, 9, 3), TOK.event2tokens(["key_signature", 0, 0, 7, 3, 0])])
    m = CO.file_meta(TOK, rows)
    assert (m[CO.META_PITCH_MIN], m[CO.META_PITCH_MAX]) == (40, 70)
    assert set(np.flatnonzero(_drum_bits(m[CO.META_DRUM:]))) == {0, 33, 100}
    assert d["note"] == TOK.event_ids["note"]


def test_split_midi_list(tmp_path):
    import random
    for i in range(23):
        (tmp_path / ("d" if i % 3 else "") ).mkdir(exist_ok=True)
        (tmp_path / ("d" if i % 3 else "") / f"f{i}.{'MID' if i % 5 == 0 else 'mid'}").write_bytes(b"")
    (tmp_path / "x.txt").write_bytes(b"")
    tr, va = CO.split_midi_list(str(tmp_path), 4, seed=7)
    lst = sorted(str(p) for p in tmp_path.rglob("*") if p.suffix.lower() in (".mid", ".midi"))
    random.seed(7)
    random.shuffle(lst)
    assert tr == lst[:19] and va == lst[19:]


# ------------------------------------------------------------------ the loader
@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    rng = np.random.default_rng(3)
    lengths = [int(x) for x in rng.integers(1, 700, 37)] + [0, 1, 299, 300, 301]
    return CO.Corpus(_build(tmp_path_factory.mktemp("corpus"), lengths), TOK)


def test_plan_deterministic_and_in_range(corpus):
    a = corpus.plan(300, seed=5, epoch=2)
    b = corpus.plan(300, seed=5, epoch=2)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    c = corpus.plan(300, seed=5, epoch=3)
    assert not np.array_equal(a[0], c[0]) and sorted(a[0]) == sorted(c[0]) == list(range(len(corpus)))
    assert not np.array_equal(corpus.plan(300, seed=6, epoch=2)[0], a[0])
    files, start, length, aug = a
    n = corpus.offsets[files + 1] - corpus.offsets[files]
    assert ((start >= 0) & (start <= np.maximum(0, n - 300 - 1))).all()
    np.testing.assert_array_equal(length, np.minimum(300, n - start))
    many = np.concatenate([corpus.plan(300, seed=1, epoch=e)[3] for e in range(40)])
    for col, lo, hi in ((lib.AUG_PITCH, -4, 4), (lib.AUG_VELOCITY, -10, 10), (lib.AUG_CC_VALUE, -10, 10),
                        (lib.AUG_BPM, -10, 10), (lib.AUG_CHANNEL, 0, 16)):
        assert set(many[:, col]) == set(range(lo, hi + 1))


def test_plan_abort_and_drum_metadata(corpus):
    for e in range(10):
        files, _, _, aug = corpus.plan(128, seed=9, epoch=e)
        for f, a in zip(files, aug):
            m = corpus.meta[f]
            assert a[lib.AUG_SKIP] == _aborted(m, a[lib.AUG_PITCH])
            np.testing.assert_array_equal(a[lib.AUG_DRUM:], m[CO.META_DRUM:])


def test_crop_distribution(tmp_path):
    n, max_len = 300, 100
    c = CO.Corpus(_build(tmp_path, [n - 2] * 50), TOK)
    starts = np.concatenate([c.plan(max_len, seed=0, epoch=e)[1] for e in range(80)])
    m = n - max_len                               # randrange(0, m), then choice([0, r])
    assert starts.max() <= m - 1
    p0 = 0.5 + 0.5 / m
    assert abs((starts == 0).mean() - p0) < 4 * (p0 * (1 - p0) / len(starts)) ** 0.5
    from scipy.stats import chisquare
    nz = starts[starts > 0]
    assert chisquare(np.bincount(nz, minlength=m)[1:]).pvalue > 1e-3
    short = CO.Corpus(_build(tmp_path, [99, 100, 0], name="short"), TOK)    # n <= max_len + 1: always 0
    assert (short.plan(max_len, seed=0, epoch=0)[1] == 0).all()


def test_validation_plan(corpus):
    files, start, length, aug = corpus.plan(300, train=False)
    np.testing.assert_array_equal(files, np.arange(len(corpus)))
    for i in files:
        n = corpus.offsets[i + 1] - corpus.offsets[i]
        max_start = max(1, n - 300)
        assert start[i] == (i * (max_start // 8)) % max_start and length[i] == min(300, n - start[i])
    assert (aug[:, lib.AUG_SKIP] == 1).all() and (aug[:, 1:] == 0).all()


@pytest.mark.parametrize("ws", [1, 2, 3, 4, 7])
@pytest.mark.parametrize("train", [True, False])
def test_rank_shares(corpus, ws, train):
    n = len(corpus)
    shares = [corpus.plan(200, train=train, seed=2, epoch=1, rank=r, world_size=ws) for r in range(ws)]
    assert len({len(s[0]) for s in shares}) == 1 and len(shares[0][0]) == -(-n // ws)
    allf = np.concatenate([s[0] for s in shares])
    assert set(allf) == set(range(n)) and len(allf) - n == (-n) % ws      # only DistributedSampler's wrap-around repeats
    if ws == 1:
        return
    full = corpus.plan(200, train=train, seed=2, epoch=1)                  # the ranks' samples are the 1-rank epoch's
    for r, s in enumerate(shares):
        k = len(range(r, n, ws))
        for x, y in zip(s, full):
            np.testing.assert_array_equal(x[:k], y[r::ws][:k])
    with pytest.raises(lib.B200Error):
        corpus.plan(200, rank=ws, world_size=ws)


def test_batches_match_plan(corpus):
    plan = corpus.plan(256, seed=4, epoch=0)
    loader = corpus.batches(5, 256, seed=4, epoch=0, depth=2)
    got = list(loader)
    assert len(got) == len(loader) == -(-len(plan[0]) // 5) and len(loader.host_s) == len(got)
    i = 0
    for tokens, lengths, aug in got:
        B = tokens.shape[0]
        assert tokens.dtype == torch.int16 and aug.dtype == torch.int32 and isinstance(lengths, list)
        assert tokens.shape[1] == max(lengths) and tokens.shape[2] == T
        assert lengths == [int(x) for x in plan[2][i:i + B]]
        np.testing.assert_array_equal(aug.numpy(), plan[3][i:i + B])
        for b in range(B):
            f, s, n = plan[0][i + b], plan[1][i + b], plan[2][i + b]
            np.testing.assert_array_equal(tokens[b, :n].numpy(), corpus.file(f)[s:s + n])
            assert (tokens[b, n:] == TOK.pad_id).all()
        i += B
    assert i == len(plan[0])
    early = corpus.batches(2, 64, depth=1)
    next(early)
    early.close()
    assert not early._thread.is_alive()


def test_manifest_checks(tmp_path):
    out = _build(tmp_path, [10, 20])
    CO.Corpus(out, TOK)
    man = json.load(open(os.path.join(out, "manifest.json")))
    for key, val in (("T", 9), ("tokenizer_version", "v1"), ("optimise_midi", True), ("vocab_size", 1), ("format", 2),
                     ("n_events", 5)):
        bad = dict(man, **{key: val})
        json.dump(bad, open(os.path.join(out, "manifest.json"), "w"))
        with pytest.raises(lib.B200Error):
            CO.Corpus(out, TOK)
    json.dump(man, open(os.path.join(out, "manifest.json"), "w"))
    t1 = TokenizerTables("v1")
    with pytest.raises(lib.B200Error):
        CO.Corpus(out, t1)
    with pytest.raises(lib.B200Error):
        CO.build_corpus([], str(tmp_path / "v1"), StubTokenizer("v1"), midi2score=stub_midi2score)
    opt = TokenizerTables("v2")
    opt.set_optimise_midi(True)
    with pytest.raises(lib.B200Error):
        CO.Corpus(out, opt)


# ------------------------------------------------------------------ data.augment_ over a mock of b200_augment_i16
def _mock_augment_call(name, batch_p, B, L, T_, aug_p, ids, _stream):
    """b200_augment_i16 as include/midi_b200.h states it, on host memory, through augment_v2."""
    assert name == "b200_augment_i16"
    from mock_kernels import _from_ptr
    d = ids._obj
    assert {f: getattr(d, f) for f, _ in d._fields_} == {**{e: AR.V2_IDS[e] for e in ("note", "patch_change", "control_change",
                                                                                   "set_tempo", "key_signature")},
                                                          **{p: AR.V2_IDS[p] for p in ("track", "channel", "pitch", "velocity",
                                                                                      "controller", "value", "bpm", "sf", "mi")}}
    b = _from_ptr(batch_p, B * L * T_, torch.int16).view(B, L, T_)
    a = _from_ptr(aug_p, B * lib.AUG_COLS, torch.int32).view(B, lib.AUG_COLS).numpy()
    b[...] = torch.from_numpy(_oracle_batch(b.numpy(), [L] * B, a))


def test_augment_wrapper_over_mock(monkeypatch, corpus):
    tokens, lengths, aug = corpus.batches(6, 200, seed=3, epoch=1).batch(0)
    want = _oracle_batch(tokens.numpy(), lengths, aug.numpy())
    monkeypatch.setattr(lib, "call", _mock_augment_call)
    monkeypatch.setattr(lib, "require_cuda", lambda t, what="tensor": None)
    monkeypatch.setattr(lib, "stream", lambda: None)
    assert data.augment_(tokens, aug) is tokens
    np.testing.assert_array_equal(tokens.numpy(), want)
    with pytest.raises(lib.B200Error):
        data.augment_(tokens, aug[:, :5].contiguous())
    with pytest.raises(lib.B200Error):
        data.augment_(tokens.long(), aug)
    with pytest.raises(lib.B200Error):
        data.augment_ids(TokenizerTables("v1"))


def test_augment_entry_declared():
    hdr = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "midi_b200.h")).read()
    assert "int b200_augment_i16(void* batch, int B, int L, int T, const int* aug" in hdr
    assert "#define B200_AUG_COLS 10" in hdr and lib.AUG_COLS == 10
    assert ctypes.sizeof(lib.AugmentIds) == 14 * 4


# ------------------------------------------------------------------ with the reference's own tokenizer and parser
def _ref_modules():
    if not ref_loader.available():
        pytest.skip("the reference tokenizer is not importable (MIDI_REFERENCE_DIR)")
    try:
        _, rt = ref_loader.load()
        spec = importlib.util.spec_from_file_location("_ref_MIDI", os.path.join(ref_loader.REF_DIR, "MIDI.py"))
        midi = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(midi)
    except Exception as e:           # e.g. a dependency of the reference missing here
        pytest.skip(f"the reference tokenizer is not importable: {e}")
    return rt, midi


def _ref_score(seed):
    rng = np.random.default_rng(seed)
    tracks = []
    for tr in range(4):
        ev = [["patch_change", 0, tr, 8 * tr], ["key_signature", 0, int(rng.integers(-7, 8)), int(rng.integers(2))]]
        if tr == 0:
            ev.append(["set_tempo", 0, 500000])
        ch = 9 if tr == 1 else tr
        t = 0
        for _ in range(400):
            t += int(rng.integers(0, 240))
            ev.append(["note", t, int(rng.integers(30, 480)), ch, int(rng.integers(20, 100)), int(rng.integers(1, 128))])
            if rng.random() < 0.1:
                ev.append(["control_change", t, ch, int(rng.choice([1, 7, 11, 64])), int(rng.integers(0, 128))])
        tracks.append(ev)
    return [480] + tracks


def test_reference_tokenizer_corpus(tmp_path):
    import random
    rt, midi = _ref_modules()
    tok = rt.MIDITokenizerV2()
    paths = []
    for i in range(3):
        p = tmp_path / f"{i}.mid"
        p.write_bytes(midi.score2midi(_ref_score(i)))
        paths.append(str(p))
    man = CO.build_corpus(paths, str(tmp_path / "c"), tok, midi2score=midi.midi2score)
    c = CO.Corpus(str(tmp_path / "c"), tok)
    assert man["n_files"] == 3
    for i, p in enumerate(paths):
        seq = np.asarray(tok.tokenize(midi.midi2score(open(p, "rb").read())), np.int16)
        np.testing.assert_array_equal(c.file(i), seq)
        for ps in (-4, 0, 3):
            forced = iter([ps, -10, 5, 10, 0, 7])
            saved = random.randint
            random.randint = lambda a, b: next(forced)
            try:
                ref = np.asarray(tok.augment(seq.tolist()), np.int64)
            finally:
                random.randint = saved
            m = c.meta[i]
            for s, e in ((0, 100), (57, 900), (len(seq) - 50, len(seq))):
                got = AR.augment_v2(seq[s:e], (ps, -10, 5, 10, 7), _aborted(m, ps), _drum_bits(m[CO.META_DRUM:]))
                np.testing.assert_array_equal(got, ref[s:e])
