"""Host side of the persistent kernel's limits: which loop a call takes for (mode, slots, top_k), and the C entries' batch
checks (tests/abi/abi_wide.c), without a GPU."""
import os
import shutil
import subprocess
import sys
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "midi-model_b200"))


def _loop(B, rows, top_ks):
    cfg1 = SimpleNamespace(hidden=1024, head_dim=64, inner=4096)
    cfg2 = SimpleNamespace(hidden=1024, head_dim=256, inner=4096)
    return SimpleNamespace(B=B, rows=rows, req_top_k=list(top_ks) if rows else [], top_k=top_ks[0],
                           outer=SimpleNamespace(eng=SimpleNamespace(cfg=cfg1)), inner=SimpleNamespace(eng=SimpleNamespace(cfg=cfg2)),
                           T=8, kv1=SimpleNamespace(page=64))


# (per-request mode, slots, top_k of every request) -> the persistent kernel runs the call
TABLE = [
    (False, 1, (1,), True), (False, 16, (64,), True), (False, 16, (65,), True), (False, 16, (128,), True),
    (False, 16, (129,), False), (False, 17, (20,), False), (False, 32, (20,), False), (False, 1, (0,), False),
    (True, 1, (128,), True), (True, 16, (20, 100), True), (True, 17, (20,), True), (True, 24, (1, 65, 128), True),
    (True, 32, (20, 128), True), (True, 32, (20, 129), False), (True, 33, (20,), False), (True, 8, (100, 4096), False),
    (True, 4, (0, 20), False),
]


@pytest.mark.parametrize("rows,B,top_ks,want", TABLE)
def test_persistent_loop_choice(rows, B, top_ks, want):
    from midi_b200 import decode as dec
    assert dec.GraphGenerator.persistent_ok(_loop(B, rows, top_ks)) is want
    # "persist" falls back to the graph loop exactly where the kernel does not apply
    assert dec.GraphGenerator._mode(SimpleNamespace(persistent_ok=lambda: want), "persist") == ("persist" if want else True)


def test_persistent_loop_needs_its_model_shape():
    from midi_b200 import decode as dec
    gg = _loop(32, True, (20,))
    gg.inner.eng.cfg.head_dim = 128
    assert not dec.GraphGenerator.persistent_ok(gg)


def test_batch_limits_of_the_c_entries_without_a_gpu():
    """tests/abi/abi_wide.c: the per-request entry refuses batch 33 and passes 17 and 32 on to its next check; the plain
    entry refuses batch 17 and passes 16 on."""
    from midi_b200 import lib
    if not os.path.exists(lib.LIB_PATH):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "midi-model_b200", "build_ext.py")])
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"abi_wide_{os.getpid()}")
    libdir = os.path.dirname(lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "abi", "abi_wide.c"), "-L", libdir, "-lmidi_b200",
                           f"-Wl,-rpath,{libdir}", "-o", exe])
    try:
        r = subprocess.run([exe], capture_output=True, text=True)
    finally:
        os.remove(exe)
    assert r.returncode == 0 and "abi wide ok" in r.stdout, r.stdout + r.stderr
