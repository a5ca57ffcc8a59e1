"""Build recipe and ctypes binding of the reference's KD_TREE::Nearest_Search with max_dist -- TEST INFRASTRUCTURE ONLY.

oracle/ref_knn_capi.cpp is compiled against the reference's include/ikd-Tree/ikd_Tree.h (REF, default /root/reference, as
in oracle/Makefile) and linked to oracle/_ref/libikdtree_ref.so, whose tree handles (oracle.bind.KdTree(..., "reference").h)
it takes.  The output, oracle/_ref/libikdtree_knn.so, stays out of git like the rest of oracle/_ref.  Where neither the
reference's sources nor a prebuilt library exist, available() is False and the tests replay stored answers.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import bind

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ref_knn_capi.cpp")
LIB_PATH = os.path.join(HERE, "_ref", "libikdtree_knn.so")
REF = os.environ.get("REF", "/root/reference")

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def build(force: bool = False) -> None:
    """Compile oracle/_ref/libikdtree_knn.so when the reference's header and oracle/_ref/libikdtree_ref.so are present."""
    bind.build()
    hdr = os.path.join(REF, "include", "ikd-Tree", "ikd_Tree.h")
    if not (os.path.exists(hdr) and os.path.exists(bind.REF_PATH)):
        return
    deps = (SRC, hdr, bind.REF_PATH, os.path.join(HERE, "shim", "pcl", "point_types.h"))
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(d) <= os.path.getmtime(LIB_PATH) for d in deps):
        return
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")     # as oracle/Makefile
    subprocess.check_call([cxx, "-O3", "-std=c++14", "-fPIC", "-fopenmp", "-w", "-shared",
                           "-I", os.path.join(HERE, "shim"), "-I", os.path.dirname(hdr), SRC, "-o", LIB_PATH,
                           "-L", os.path.dirname(bind.REF_PATH), "-l:libikdtree_ref.so", "-Wl,-rpath,$ORIGIN", "-lpthread"])


def available() -> bool:
    build()
    return bind.have_ref() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        bind.ref()                     # the tree library first: this one resolves its KD_TREE symbols there
        L = C.CDLL(LIB_PATH)
        L.ref_kdtree_nearest_search.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_float, _f32p, _f32p, _i32p, C.c_int]
        L.ref_kdtree_nearest_search.restype = None
        _lib = L
    return _lib


def nearest_search(tree: bind.KdTree, q4, k: int, max_dist: float = np.inf, nthreads: int = 0):
    """KD_TREE::Nearest_Search(q, k, .., max_dist) per row: (pts[nq, k, 4], d2[nq, k], cnt[nq]) in the layout of
    fl_map_nearest_search."""
    assert tree.backend == "reference"
    q4 = np.ascontiguousarray(q4, dtype=np.float32).reshape(-1, 4)
    pts = np.zeros((len(q4), k, 4), dtype=np.float32)
    d2 = np.zeros((len(q4), k), dtype=np.float32)
    cnt = np.zeros(len(q4), dtype=np.int32)
    lib().ref_kdtree_nearest_search(tree.h, q4, len(q4), k, max_dist, pts, d2, cnt, nthreads)
    return pts, d2, cnt
