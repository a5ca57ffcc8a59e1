"""Builds fast_lio_b200/libfastlio_b200.so in-tree with nvcc for sm_90a (H100).

The .so is a build product and stays out of git; there is no JIT and no fallback: if the
library is missing, importing the bindings raises.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfastlio_b200.so")
SOURCES = ["map.cu", "filter.cu", "reloc.cu", "scan.cu", "preprocess.cu", "capi.cu"]
HEADERS = ["common.cuh", "map.cuh", "map.h", "map_rules.h", "lie.cuh", "filter.h", "scan.h", "gj.cuh", "measure.cuh", "update.cuh", "wave_row.cuh", "wave_search.cuh", "wave_solver.cuh", "upd_plan.h", "preprocess.h", "reloc.cuh", os.path.join("..", "..", "include", "fastlio_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    # parity: the reference's float32 arithmetic runs on x86-64 without FMA contraction
    "--fmad=false", "-prec-div=true", "-prec-sqrt=true",
    "-Xcompiler", "-fPIC", "-shared",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    tmp = LIB + ".tmp"          # link into a temporary, then rename: a snapshot of the tree never sees a half-written library
    cmd = [_nvcc()] + NVCC_FLAGS + ["-ccbin", "/usr/bin/g++"] + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", tmp, "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed")
    os.replace(tmp, LIB)
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
