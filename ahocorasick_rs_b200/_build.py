"""Builds libacb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Called by __graft_entry__.build(); the .so is git-ignored.  A library built with
other flags (another architecture) counts as stale and is rebuilt: the nvcc
command line is kept next to it."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libacb200.so")
STAMP = LIB + ".cmd"
SOURCES = ["capi.cu", "automaton.cpp", "sieve.cpp", "completions.cpp", "vocab.cpp"]
HEADERS = ["automaton.h", "scan_core.cuh", "scan_staged.cuh", "scan_global.cuh", "scan_sieve.cuh", "sieve.h", "repair.cuh", "tokens.cuh", "completions.h", "completions.cuh", "vocab.h", "vocab.cuh", os.path.join("..", "..", "include", "acb200.h")]
FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-diag-suppress", "186",
         "-shared", "-Xcompiler", "-fPIC,-pthread"]


def _stale() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != " ".join(FLAGS):
            return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    cmd = [nvcc] + FLAGS + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    with open(STAMP, "w") as f:
        f.write(" ".join(FLAGS))
    return LIB
