"""Build libmidi_b200.so (all CUDA kernels + the C ABI) in-tree with nvcc for sm_90a (H100).

    python midi-model_b200/build_ext.py [--force]

nvcc cross-compiles without a GPU; the .so and the objects are build products (git-ignored).
Objects are rebuilt only when their source (or a header) is newer.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "midi_b200", "libmidi_b200.so")
SOURCES = ["runtime.cu", "elementwise.cu", "gemm_wgmma.cu", "attn_flash.cu", "attn_wgmma.cu", "attn_tiny.cu", "train_misc.cu", "decode.cu", "decode_persist.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--threads", "2"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(a: str, b: str) -> bool:
    return not os.path.exists(b) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdr_time = max(os.path.getmtime(h) for h in headers)
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(s, o) or os.path.getmtime(o) < hdr_time:
            jobs.append([nvcc, *NVCC_FLAGS, "-I", CSRC, "-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print("[build]", os.path.basename(cmd[-3]), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {cmd[-3]}:\n{r.stdout}\n{r.stderr}")
        return r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(4, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or force or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", *ARCH, "-o", LIB, *objs]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print("[build] linked", LIB, flush=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
