"""TEST INFRASTRUCTURE: train.py's augmentation (`MIDITokenizerV2.augment`, midi_tokenizer.py:1023-1102) restated with
numpy, vectorised over the rows of one sequence.  It is the checker of the device kernel `b200_augment_i16` and of the
corpus loader's abort / drum metadata, and is itself pinned to the reference's own `augment` by
tests/golden/augment_v2.npz (written by tests/make_golden_augment.py).  The product never imports it."""
import numpy as np

def _v2_ids():
    """Event ids and first parameter ids of the v2 layout (midi_tokenizer.py:517-534): pad, bos, eos, six event ids, then
    one block per parameter in declaration order."""
    events = ("note", "patch_change", "control_change", "set_tempo", "time_signature", "key_signature")
    params = (("time1", 128), ("time2", 16), ("duration", 2048), ("track", 128), ("channel", 16), ("pitch", 128),
              ("velocity", 128), ("patch", 128), ("controller", 128), ("value", 128), ("bpm", 384), ("nn", 16), ("dd", 4),
              ("sf", 15), ("mi", 2))
    ids = {e: 3 + i for i, e in enumerate(events)}
    nxt = 3 + len(events)
    for p, n in params:
        ids[p] = nxt
        nxt += n
    return ids


V2_IDS = _v2_ids()


def augment_v2(tokens, shifts, aborted: bool, drum_mask):
    """The reference's `augment` of one whole v2 sequence, restated with numpy.  tokens: int [L, T]; shifts: (pitch,
    velocity, cc value, bpm, channel) with track shift 0; aborted: the reference's early return (a shifted non-drum note
    outside 0..127 anywhere in the file) -- the input comes back unchanged; drum_mask: bool [128], the tracks whose notes
    all have original channel 9 (at least one note), whose key signatures get sf = 0.  Returns a new int64 array."""
    d = V2_IDS
    t = np.array(tokens, dtype=np.int64)
    if aborted:
        return t
    ps, vs, cs, bs, chs = (int(s) for s in shifts)
    drum = np.asarray(drum_mask, dtype=bool)
    ev = t[:, 0]
    out = t.copy()
    has_ch = (ev == d["note"]) | (ev == d["patch_change"]) | (ev == d["control_change"])
    c0 = t[:, 4] - d["channel"]
    c = (c0 + chs) % 16                              # numpy's % is floored, like Python's
    c = np.where(c0 == 9, 9, np.where(c == 9, (9 + chs) % 16, c))
    out[:, 4] = np.where(has_ch, d["channel"] + c, out[:, 4])
    note = ev == d["note"]
    p = t[:, 5] - d["pitch"] + np.where(c0 != 9, ps, 0)
    out[:, 5] = np.where(note, d["pitch"] + p, out[:, 5])
    out[:, 6] = np.where(note, d["velocity"] + np.clip(t[:, 6] - d["velocity"] + vs, 1, 127), out[:, 6])
    cc = (ev == d["control_change"]) & np.isin(t[:, 5] - d["controller"], [1, 2, 7, 11])
    out[:, 6] = np.where(cc, d["value"] + np.clip(t[:, 6] - d["value"] + cs, 1, 127), out[:, 6])
    tempo = ev == d["set_tempo"]
    out[:, 4] = np.where(tempo, d["bpm"] + np.clip(t[:, 4] - d["bpm"] + bs, 1, 383), out[:, 4])
    ks = ev == d["key_signature"]
    mi = t[:, 5] - d["mi"]
    k = ((((t[:, 4] - d["sf"] - 7) * 7) % 12) + ps) % 12
    sf = (k * 7) % 12
    sf = np.where((sf > 6) | ((mi == 1) & (sf >= 5)), sf - 12, sf)
    tr = np.clip(t[:, 3] - d["track"], 0, 127)
    sf = np.where(drum[tr], 0, sf)
    out[:, 4] = np.where(ks, d["sf"] + sf + 7, out[:, 4])
    return out
