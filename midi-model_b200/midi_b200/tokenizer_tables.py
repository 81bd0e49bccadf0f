"""Token-id tables of the MIDI event vocabulary (data layout only).

The hot path never tokenises MIDI files; it only needs the id layout of the
`(batch, events, 8)` tensors: vocabulary size, pad/bos/eos, the event-type ids
and the contiguous id range of every event parameter.  These are the tables
the reference defines in `midi_tokenizer.py:8-35` (V1) and `:506-535` (V2).

When the reference's own `midi_tokenizer` module is importable (the drop-in
deployment: this repo's `midi_model.py` placed ahead of the reference on
`sys.path`) the drop-in uses that class unchanged, so `tokenize/detokenize`
keep working.  When it is not (the GPU box, unit tests, the benchmark) this
table-only stand-in provides the same attributes.  Score <-> token conversion,
augmentation and quality filters are out of scope.
"""
from __future__ import annotations

from typing import Any, Dict, List

# (event name -> ordered parameter names) and (parameter name -> cardinality), per tokenizer version.
_SPECS = {
    "v1": dict(
        events=(
            ("note", ("time1", "time2", "track", "duration", "channel", "pitch", "velocity")),
            ("patch_change", ("time1", "time2", "track", "channel", "patch")),
            ("control_change", ("time1", "time2", "track", "channel", "controller", "value")),
            ("set_tempo", ("time1", "time2", "track", "bpm")),
        ),
        params=(("time1", 128), ("time2", 16), ("duration", 2048), ("track", 128), ("channel", 16), ("pitch", 128),
                ("velocity", 128), ("patch", 128), ("controller", 128), ("value", 128), ("bpm", 256)),
    ),
    "v2": dict(
        events=(
            ("note", ("time1", "time2", "track", "channel", "pitch", "velocity", "duration")),
            ("patch_change", ("time1", "time2", "track", "channel", "patch")),
            ("control_change", ("time1", "time2", "track", "channel", "controller", "value")),
            ("set_tempo", ("time1", "time2", "track", "bpm")),
            ("time_signature", ("time1", "time2", "track", "nn", "dd")),
            ("key_signature", ("time1", "time2", "track", "sf", "mi")),
        ),
        params=(("time1", 128), ("time2", 16), ("duration", 2048), ("track", 128), ("channel", 16), ("pitch", 128),
                ("velocity", 128), ("patch", 128), ("controller", 128), ("value", 128), ("bpm", 384), ("nn", 16),
                ("dd", 4), ("sf", 15), ("mi", 2)),
    ),
}


class TokenizerTables:
    """Id layout: [pad, bos, eos] + one id per event type + one contiguous block per parameter."""

    def __init__(self, version: str = "v2"):
        if version not in _SPECS:
            raise ValueError(f"Unsupported version: {version}")
        spec = _SPECS[version]
        self.version = version
        self.optimise_midi = False
        self.pad_id, self.bos_id, self.eos_id = 0, 1, 2
        nxt = 3
        self.events: Dict[str, List[str]] = {name: list(ps) for name, ps in spec["events"]}
        self.event_parameters: Dict[str, int] = dict(spec["params"])
        self.event_ids: Dict[str, int] = {}
        for name in self.events:
            self.event_ids[name] = nxt
            nxt += 1
        self.id_events = {i: e for e, i in self.event_ids.items()}
        self.parameter_ids: Dict[str, List[int]] = {}
        for pname, card in spec["params"]:
            self.parameter_ids[pname] = list(range(nxt, nxt + card))
            nxt += card
        self.vocab_size = nxt
        self.max_token_seq = 1 + max(len(ps) for ps in self.events.values())

    # -- the small API the model and its callers use --------------------
    def set_optimise_midi(self, optimise_midi: bool = True):
        self.optimise_midi = optimise_midi

    def to_dict(self) -> Dict[str, Any]:
        return {"version": self.version, "optimise_midi": self.optimise_midi, "vocab_size": self.vocab_size,
                "events": self.events, "event_parameters": self.event_parameters,
                "max_token_seq": self.max_token_seq, "pad_id": self.pad_id, "bos_id": self.bos_id,
                "eos_id": self.eos_id}

    def event2tokens(self, event) -> List[int]:
        """['note', t1, t2, ...] -> 8 ids (pad-filled); [] if a parameter is out of range."""
        name, vals = event[0], event[1:]
        out = [self.event_ids[name]]
        for pname, v in zip(self.events[name], vals):
            if not 0 <= v < self.event_parameters[pname]:
                return []
            out.append(self.parameter_ids[pname][v])
        return out + [self.pad_id] * (self.max_token_seq - len(out))

    def tokens2event(self, tokens) -> list:
        name = self.id_events.get(int(tokens[0]))
        if name is None or len(tokens) <= len(self.events[name]):
            return []
        out = [name]
        for pname, t in zip(self.events[name], tokens[1:]):
            v = int(t) - self.parameter_ids[pname][0]
            if not 0 <= v < self.event_parameters[pname]:
                return []
            out.append(v)
        return out

    # -- grammar as id ranges (what the device-side generate loop consumes) --
    def grammar_ranges(self):
        """Returns {event_id: [(lo, hi), ...]} with one half-open id range per parameter position."""
        return {self.event_ids[n]: [(self.parameter_ids[p][0], self.parameter_ids[p][-1] + 1) for p in ps]
                for n, ps in self.events.items()}


def make_tokenizer(version: str = "v2"):
    """Prefer the reference's tokenizer class when it is importable (drop-in
    deployment), else the table-only stand-in."""
    try:
        from midi_tokenizer import MIDITokenizer  # the reference's module, if on sys.path
        return MIDITokenizer(version)
    except Exception:
        return TokenizerTables(version)
