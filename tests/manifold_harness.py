"""ctypes front of tests/kernels/manifold_harness.cu (lie.cuh, measure.cuh and gj.cuh over batches of inputs), compiled with the library's nvcc flags into a temporary directory."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fast_lio_b200 import build

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernels", "manifold_harness.cu")

FNS = ["cos_sinc_sqrt", "so3_exp", "so3_log", "A_matrix", "S2_Bx", "S2_boxplus", "S2_boxminus", "S2_Nx_yy", "S2_Mx",
       "S2_congruence", "state_boxplus", "state_boxminus", "esti_plane", "measure"]
GJ = ["gj_eliminate", "gj_warp", "gj_warp_reg6", "gj_warp_reg12", "gj_cols6", "gj_cols12"]

_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def compile_harness(out_dir: str) -> str:
    """nvcc with build.NVCC_FLAGS (sm_90a, --fmad=false, -prec-div, -prec-sqrt) -> out_dir/libmanifold_harness.so."""
    out = os.path.join(str(out_dir), "libmanifold_harness.so")
    res = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-ccbin", "/usr/bin/g++", SRC, "-o", out], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return out


class Harness:
    def __init__(self, path: str):
        L = C.CDLL(path)
        L.mh_width.argtypes = [C.c_int, C.c_int]
        L.mh_eval.argtypes = [C.c_int, C.c_int, _f64p, _f64p, C.c_int]
        L.mh_gj.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f64p, _f64p, _i32p, _i32p]
        self.L = L

    def width(self, fn: str):
        i = FNS.index(fn)
        return self.L.mh_width(i, 0), self.L.mh_width(i, 1)

    def eval(self, fn: str, inputs, device: bool) -> np.ndarray:
        nin, nout = self.width(fn)
        x = np.ascontiguousarray(np.asarray(inputs, dtype=np.float64).reshape(-1, nin))
        out = np.zeros((len(x), nout))
        rc = self.L.mh_eval(FNS.index(fn), len(x), x, out, int(device))
        assert rc == 0, f"mh_eval({fn}) -> {rc}"
        return out

    def gj(self, variant: str, systems, n: int, nc: int, threads: int = 32):
        """Solves each n x nc system [A | B] (row stride nc); returns (X (count, n, nc - n), row map (count, n), ok (count))."""
        a = np.ascontiguousarray(np.asarray(systems, dtype=np.float64).reshape(-1, n * nc))
        x = np.zeros((len(a), n, nc - n))
        rmap = np.zeros((len(a), n), dtype=np.int32)
        ok = np.zeros(len(a), dtype=np.int32)
        rc = self.L.mh_gj(GJ.index(variant), len(a), n, nc, nc, threads, a, x, rmap, ok)
        assert rc == 0, f"mh_gj({variant}) -> {rc}"
        return x, rmap, ok.astype(bool)
