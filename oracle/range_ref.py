"""Build recipe and ctypes binding of the reference's KD_TREE::Box_Search / Radius_Search -- TEST INFRASTRUCTURE ONLY.

oracle/ref_range_capi.cpp is compiled against the reference's include/ikd-Tree/ikd_Tree.h (REF, default /root/reference, as
in oracle/Makefile) and linked to oracle/_ref/libikdtree_ref.so, whose tree handles (oracle.bind.KdTree(..., "reference").h)
it takes.  The output, oracle/_ref/libikdtree_range.so, stays out of git like the rest of oracle/_ref.  Where neither the
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
SRC = os.path.join(HERE, "ref_range_capi.cpp")
LIB_PATH = os.path.join(HERE, "_ref", "libikdtree_range.so")
REF = os.environ.get("REF", "/root/reference")

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def build(force: bool = False) -> None:
    """Compile oracle/_ref/libikdtree_range.so when the reference's header and oracle/_ref/libikdtree_ref.so are present."""
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
        for fn in (L.ref_kdtree_box_search, L.ref_kdtree_radius_search):
            fn.argtypes = [C.c_void_p, _f32p, C.c_int, _i32p, _f32p, C.c_int, C.c_int]
            fn.restype = C.c_int
        _lib = L
    return _lib


def _range(fn, tree: bind.KdTree, q, nthreads):
    assert tree.backend == "reference"
    offsets = np.zeros(len(q) + 1, dtype=np.int32)
    cap = max(1024, tree.size())
    out = np.empty((cap, 4), dtype=np.float32)
    total = fn(tree.h, q, len(q), offsets, out, cap, nthreads)
    if total > cap:
        out = np.empty((total, 4), dtype=np.float32)
        total = fn(tree.h, q, len(q), offsets, out, total, nthreads)
    return offsets, out[:total]


def box_search(tree: bind.KdTree, boxes6, nthreads: int = 0):
    """KD_TREE::Box_Search per (min xyz, max xyz) row: (offsets, points) in the CSR layout of fl_map_box_search."""
    return _range(lib().ref_kdtree_box_search, tree, np.ascontiguousarray(boxes6, dtype=np.float32).reshape(-1, 6), nthreads)


def radius_search(tree: bind.KdTree, centers_xyzr, nthreads: int = 0):
    """KD_TREE::Radius_Search per (x, y, z, radius) row: (offsets, points) like box_search."""
    return _range(lib().ref_kdtree_radius_search, tree, np.ascontiguousarray(centers_xyzr, dtype=np.float32).reshape(-1, 4), nthreads)
