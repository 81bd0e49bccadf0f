"""Ragged prompts (`generate_ragged` / `generate_stream_ragged`): the host logic of the device-resident loop (ragged state,
rectangular prefill, per-row offsets handed to the `_ragged` kernel entries, per-row stop check and output layout) over
the CPU stand-in for the kernel layer (tests/mock_kernels.py), B200_GENERATE=nograph.  The kernels themselves are checked on
the GPU (tests/test_gpu_ragged_generate.py)."""
import numpy as np
import pytest
import torch

import host_model
import mock_kernels


def test_ragged_signatures():
    """generate_ragged / generate_stream_ragged: generate's and generate_stream's parameters (whose signatures stay the
    reference's) with the prompt and its lengths first."""
    import inspect
    import midi_model as mm
    gen = inspect.signature(mm.MIDIModel.generate_ragged).parameters
    assert list(gen)[1:] == ["prompt", "lengths", "batch_size", "max_len", "temp", "top_p", "top_k", "generator"]
    assert [gen[k].default for k in list(gen)[3:]] == [1, 512, 1.0, 0.98, 20, None]
    st = inspect.signature(mm.MIDIModel.generate_stream_ragged).parameters
    assert list(st)[1:] == ["prompt", "lengths", "batch_size", "max_len", "temp", "top_p", "top_k", "disable_patch_change",
                            "disable_control_change", "disable_channels", "generator"]
    assert inspect.isgeneratorfunction(inspect.unwrap(mm.MIDIModel.generate_stream_ragged))


@pytest.fixture
def model(monkeypatch):
    return host_model.generate_model(monkeypatch, "nograph")


def _prompt(model, B, P, seed):
    from midi_b200.synth import synth_batch
    return synth_batch(model.tokenizer, B, P, seed=seed).numpy()


def _check_rows_match_solo(model, prompt, lengths, n_new, ids):
    """Row b of a greedy ragged run against generating prompt b[:L_b] alone (same loop, batch 1)."""
    pad = model.tokenizer.pad_id
    eos = model.tokenizer.eos_id
    B, P = len(lengths), max(lengths)
    n_done = ids.shape[1] - P
    assert 1 <= n_done <= n_new
    for b, L in enumerate(lengths):
        solo = model.generate(prompt=prompt[b:b + 1, :L], batch_size=1, max_len=L + n_new, top_k=1)[0]
        k = solo.shape[0] - L                              # solo stops early when its row emits EOS (all rows = one row)
        assert (ids[b, :L] == prompt[b, :L]).all()
        assert (ids[b, L:L + k] == solo[L:]).all(), b
        assert k == n_done or (k < n_done and solo[-1, 0] == eos), (b, k, n_done)
        assert (ids[b, L + n_done:] == pad).all()           # data.collate layout: pad events after the row's end


@pytest.mark.parametrize("fused", [True, False])
def test_greedy_rows_equal_their_solo_generation(model, monkeypatch, fused):
    """L = [P, 1, P-3, 2] with P = 67: rows whose positions cross the 64-position page boundary and rows that start at
    position 0 or 1.  `fused`: the B <= 16 single-launch attention path, or the unfused rope / append / attention path
    the loop takes for B > 16."""
    from midi_b200 import decode
    monkeypatch.setattr(decode, "FUSED_DECODE", fused)
    P, n_new = 67, 4
    lengths = [P, 1, P - 3, 2]
    prompt = _prompt(model, 4, P, seed=3)
    ids = model.generate_ragged(prompt=prompt, batch_size=4, max_len=P + n_new, top_k=1, lengths=lengths)
    assert ids.dtype == np.int64 and ids.shape[0] == 4 and ids.shape[2] == 8
    _check_rows_match_solo(model, prompt, lengths, n_new, ids)


def test_few_new_events_still_use_the_device_loop(model, monkeypatch):
    """With lengths the device-resident loop runs even for fewer than 4 new events (without them generate takes the eager
    loop there); a prompt already at max_len comes back in the collate layout."""
    P = 5
    lengths = torch.tensor([3, 5, 1])
    prompt = _prompt(model, 3, P, seed=4)
    with monkeypatch.context() as mp:
        names = mock_kernels.trace(mp, lambda: model.generate_ragged(prompt=prompt, batch_size=3, max_len=P + 2, top_k=1,
                                                                     lengths=lengths))
    assert "b200_event_commit_ragged" in names
    ids = model.generate_ragged(prompt=prompt, batch_size=3, max_len=P + 2, top_k=1, lengths=lengths)
    _check_rows_match_solo(model, prompt, lengths.tolist(), 2, ids)
    same = model.generate_ragged(prompt=prompt, batch_size=3, max_len=P, top_k=1, lengths=lengths)
    pad = model.tokenizer.pad_id
    assert same.shape == (3, P, 8)
    for b, L in enumerate(lengths.tolist()):
        assert (same[b, :L] == prompt[b, :L]).all() and (same[b, L:] == pad).all()


def test_full_lengths_match_rectangular_call_for_call(model, monkeypatch):
    """generate_ragged with lengths = [P] * B gives generate's output bit for bit, and issues the rectangular loop's calls
    one for one with the `_ragged` entries in place of their counterparts; generate never reaches a `_ragged` entry."""
    P, n_new, B = 6, 5, 2
    prompt = _prompt(model, B, P, seed=5)
    kw = dict(prompt=prompt, batch_size=B, max_len=P + n_new, top_k=1)
    out = {}
    model.generate(**kw)                                       # one-time set-up (RoPE tables, grammar) outside the traces
    with monkeypatch.context() as mp:
        rect = mock_kernels.trace(mp, lambda: out.setdefault("rect", model.generate(**kw)))
    with monkeypatch.context() as mp:
        ragged = mock_kernels.trace(mp, lambda: out.setdefault("ragged", model.generate_ragged(**kw, lengths=[P] * B)))
    assert (out["rect"] == out["ragged"]).all() and out["rect"].shape == out["ragged"].shape
    assert not [n for n in rect if "ragged" in n]
    assert [n.replace("_ragged", "") for n in ragged] == rect
    assert "b200_attn_decode_fused_ragged" in ragged and "b200_event_commit_ragged" in ragged


def test_padding_past_the_lengths_is_never_read(model):
    P, n_new = 9, 4
    lengths = [9, 4, 6]
    prompt = _prompt(model, 3, P, seed=6)
    ref = model.generate_ragged(prompt=prompt, batch_size=3, max_len=P + n_new, top_k=1, lengths=lengths)
    junk = prompt.copy()
    rng = np.random.default_rng(0)
    for b, L in enumerate(lengths):
        junk[b, L:] = rng.integers(-7, 10 ** 6, size=junk[b, L:].shape)           # out-of-range ids included
    got = model.generate_ragged(prompt=junk, batch_size=3, max_len=P + n_new, top_k=1, lengths=lengths)
    assert got.shape == ref.shape and (got == ref).all()


def test_stream_yields_the_generated_events(model):
    P, n_new = 7, 5
    lengths = [2, 7, 5]
    prompt = _prompt(model, 3, P, seed=7)
    ids = model.generate_ragged(prompt=prompt, batch_size=3, max_len=P + n_new, top_k=1, lengths=lengths)
    evs = [e.copy() for e in model.generate_stream_ragged(prompt=prompt, batch_size=3, max_len=P + n_new, top_k=1,
                                                          lengths=lengths)]
    n_done = ids.shape[1] - P
    assert len(evs) == n_done and all(e.shape == (3, 8) for e in evs)
    for b, L in enumerate(lengths):
        assert (np.stack([e[b] for e in evs]) == ids[b, L:L + n_done]).all()


def test_stream_context_window_is_per_row(model, monkeypatch):
    """app.py:55's 4096-event window applies per row: row b keeps its last min(L_b, 4096) events."""
    from midi_b200 import decode
    seen = {}

    def spy(self, prompt, use_graph=True, lengths=None):      # records what the loop would get, without running it
        seen["prompt"], seen["lengths"] = prompt.clone(), list(lengths)
        return iter(())

    monkeypatch.setattr(decode.GraphGenerator, "events", spy)
    P = 4100
    prompt = np.full((2, P, 8), model.tokenizer.pad_id, dtype=np.int64)
    prompt[:, :, 0] = np.arange(P) % 50 + 3                  # a recognisable position code in column 0
    lengths = [4099, 10]
    assert list(model.generate_stream_ragged(prompt=prompt, batch_size=2, max_len=4097, top_k=1, lengths=lengths)) == []
    assert seen["lengths"] == [4096, 10]
    got = seen["prompt"].numpy()
    assert got.shape[1] == 4096
    assert (got[0] == prompt[0, 4099 - 4096:4099]).all()
    assert (got[1, :10] == prompt[1, :10]).all()


def test_input_errors_raise(model, monkeypatch):
    from midi_b200.lib import B200Error
    P = 5
    prompt = _prompt(model, 2, P, seed=8)
    kw = dict(prompt=prompt, batch_size=2, max_len=P + 3, top_k=1)
    bad = [[1], [1, 2, 3], [0, 3], [3, 6], [2.0, 3], torch.tensor([2.0, 3.0]), torch.tensor([[2, 3]]), "23", 3]
    for lengths in bad:
        with pytest.raises(B200Error):
            model.generate_ragged(**kw, lengths=lengths)
        with pytest.raises(B200Error):
            list(model.generate_stream_ragged(**kw, lengths=lengths))
    with pytest.raises(B200Error):
        model.generate_ragged(prompt=None, batch_size=2, max_len=6, top_k=1, lengths=[1, 1])
    with pytest.raises(B200Error):
        list(model.generate_stream_ragged(prompt=None, batch_size=2, max_len=6, top_k=1, lengths=[1, 1]))
    monkeypatch.setenv("B200_GENERATE", "eager")
    with pytest.raises(B200Error):
        model.generate_ragged(**kw, lengths=[2, 3])
    with pytest.raises(B200Error):
        list(model.generate_stream_ragged(**kw, lengths=[2, 3]))


def test_device_lengths_tensor_raises(model):
    from midi_b200.lib import B200Error
    meta = torch.tensor([2, 3], device="meta")                # any non-CPU tensor is refused before its values are read
    with pytest.raises(B200Error):
        model.generate_ragged(prompt=_prompt(model, 2, 5, seed=9), batch_size=2, max_len=8, top_k=1, lengths=meta)
