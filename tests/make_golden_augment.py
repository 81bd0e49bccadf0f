"""Generate tests/golden/augment_v2.npz from the UNMODIFIED reference -- run where a checkout of the reference is present
(MIDI_REFERENCE_DIR, see oracle/ref_loader.py):  python tests/make_golden_augment.py

The fixture is what the reference's MIDITokenizerV2.augment (train.py's augmentation) returns, with its six
`random.randint` draws forced, on token sequences that reach each of its rules, for every pitch and channel shift.
tests/augment_reference.py is checked against it (tests/test_corpus_host.py).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _augment_files(tok):
    """Token sequences (not MIDI files: the reference's `augment` takes rows) that reach every rule of `augment`: BOS / EOS,
    notes on mixed, drum-only and single-channel tracks with velocity 0 / 1 / 127, every patch-change channel, cc 1 / 2 /
    7 / 11 and other controllers at value 0 / 1 / 127, bpm 0 / 1 / 383, time signatures, and every sf / mi on drum-only,
    mixed and note-less tracks.  'mixed' never aborts, 'edge' (non-drum pitches 2 ... 125) aborts for pitch shifts of
    magnitude 3 and 4 and has drum notes at 0 and 127, 'drums' has notes on channel 9 only."""
    rng = np.random.default_rng(2024)
    e2t = tok.event2tokens

    def keysigs(tracks):
        return [e2t(["key_signature", 0, 0, tr, sf, mi]) for tr in tracks for sf in range(15) for mi in range(2)]

    def common(tracks_ks):
        rows = [e2t(["patch_change", 1, 0, 0, c, 5 * c]) for c in range(16)]
        rows += [e2t(["control_change", 2, 1, 0, c % 16, cc, v]) for c, (cc, v) in
                 enumerate((cc, v) for cc in (0, 1, 2, 7, 10, 11, 64, 127) for v in (0, 1, 64, 127))]
        rows += [e2t(["set_tempo", 3, 2, 0, b]) for b in (0, 1, 2, 100, 374, 383)]
        rows += [e2t(["time_signature", 0, 0, 0, 3, 2])]
        return rows + keysigs(tracks_ks)

    def notes(track, chans, pitches, vels=(0, 1, 64, 127)):
        return [e2t(["note", int(rng.integers(128)), int(rng.integers(16)), track, int(c), int(p), int(v), 10])
                for c in chans for p in pitches for v in vels]

    files = {
        "mixed": notes(0, (0, 3, 9), (30, 60, 90)) + notes(1, (9,), (0, 35, 127)) + notes(3, (15,), (40, 41))
                 + common((0, 1, 2, 3)),
        "edge": notes(0, (1,), (2, 125)) + notes(1, (9,), (0, 127)) + notes(2, (9, 4), (50,)) + common((0, 1, 2, 5)),
        "drums": notes(0, (9,), range(0, 128, 9)) + notes(5, (9,), (0, 127)) + common((0, 5, 7)),
    }
    out = {}
    for name, rows in files.items():
        assert all(len(r) == tok.max_token_seq for r in rows), name
        rows = [rows[i] for i in rng.permutation(len(rows))]
        bos = [tok.bos_id] + [tok.pad_id] * (tok.max_token_seq - 1)
        eos = [tok.eos_id] + [tok.pad_id] * (tok.max_token_seq - 1)
        out[name] = [bos] + rows + [eos]
    return out


def augment_v2():
    """tests/golden/augment_v2.npz: the reference's MIDITokenizerV2.augment on `_augment_files`, with its six
    `random.randint` draws forced, for every (pitch shift, channel shift) pair of train.py's ranges on every file; the
    velocity / cc value / bpm shifts cycle through -10, 0, 10 and other values.  Track shift 0, as train.py draws it."""
    import random
    _, rt = ref_loader.load()
    tok = rt.MIDITokenizerV2()
    files = _augment_files(tok)
    others = [-10, 0, 10, -7, 3, 1, -1, 6]
    tokens, offsets, cases, outs, out_off = [], [0], [], [], [0]
    for f, (name, rows) in enumerate(files.items()):
        tokens.append(np.asarray(rows, np.int16))
        offsets.append(offsets[-1] + len(rows))
        i = 0
        for ps in range(-4, 5):
            for ch in range(17):
                vs, cs, bs = others[i % 8], others[(i + 3) % 8], others[(i + 5) % 8]
                i += 1
                forced = iter([ps, vs, cs, bs, 0, ch])
                saved = random.randint

                def randint(a, b):
                    v = next(forced)
                    assert a <= v <= b, (a, b, v)
                    return v
                random.randint = randint
                try:
                    res = tok.augment([list(r) for r in rows])
                finally:
                    random.randint = saved
                cases.append([f, ps, vs, cs, bs, 0, ch])
                outs.append(np.asarray(res, np.int16))
                out_off.append(out_off[-1] + len(res))
    out = {"names": np.array(list(files)), "tokens": np.concatenate(tokens), "offsets": np.asarray(offsets, np.int64),
           "cases": np.asarray(cases, np.int32), "out": np.concatenate(outs), "out_offsets": np.asarray(out_off, np.int64)}
    np.savez_compressed(os.path.join(OUT, "augment_v2.npz"), **out)
    print("augment_v2.npz:", len(cases), "cases,", int(out["tokens"].shape[0]), "rows")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    augment_v2()
