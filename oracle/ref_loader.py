"""Import the UNMODIFIED reference (a checkout of SkyTNT/midi-model named by MIDI_REFERENCE_DIR) read-only -- used by
oracle/make_golden.py to produce the fixtures under tests/golden/.

The reference fails to import without peft only because `midi_model.py:9`
imports four `peft` names that are used solely inside `load_merge_lora`
(`midi_model.py:109-114`).  We register a 4-name stub module and import the
reference's own `midi_model` / `midi_tokenizer` under private module names so
they never shadow the drop-in `midi_model` of this repo.

Without MIDI_REFERENCE_DIR `available()` is False; the tests never need the reference (they read the fixtures).
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REF_DIR = os.environ.get("MIDI_REFERENCE_DIR", "")


def available() -> bool:
    return bool(REF_DIR) and os.path.isfile(os.path.join(REF_DIR, "midi_model.py"))


def _load(name: str, alias: str):
    spec = importlib.util.spec_from_file_location(alias, os.path.join(REF_DIR, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[alias] = mod
    spec.loader.exec_module(mod)
    return mod


_cache = {}


def load():
    """Returns (ref_midi_model_module, ref_midi_tokenizer_module)."""
    if "m" in _cache:
        return _cache["m"], _cache["t"]
    if not available():
        raise RuntimeError(f"reference not present (MIDI_REFERENCE_DIR={REF_DIR!r})")
    if "peft" not in sys.modules:
        try:
            import peft  # noqa: F401
        except Exception:
            stub = types.ModuleType("peft")
            for n in ("PeftConfig", "LoraModel", "load_peft_weights", "set_peft_model_state_dict"):
                setattr(stub, n, None)
            sys.modules["peft"] = stub
    saved = {k: sys.modules.get(k) for k in ("midi_tokenizer", "midi_model", "MIDI")}
    try:
        for k in saved:
            sys.modules.pop(k, None)
        tok = _load("midi_tokenizer", "midi_tokenizer")      # reference imports it by this name
        mm = _load("midi_model", "_ref_midi_model")
        sys.modules["_ref_midi_tokenizer"] = tok
    finally:
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v
            else:
                sys.modules.pop(k, None)
    _cache["m"], _cache["t"] = mm, tok
    return mm, tok
