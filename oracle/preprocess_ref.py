"""Build recipe and ctypes binding of the reference's own Preprocess::process -- TEST INFRASTRUCTURE ONLY.

The reference's src/preprocess.cpp is compiled unmodified where it lies (REF, default /root/reference, as in
oracle/Makefile), together with oracle/ref_preprocess_capi.cpp, against the ROS / PCL / Eigen / Livox stand-ins under
oracle/shim, with the reference's own flags (-O3 -std=c++14, OpenMP; no -march, so no FMA contraction).  The output,
oracle/_ref/libpreprocess_ref.so, stays out of git like the rest of oracle/_ref.  Where neither the reference's sources nor
a prebuilt library exist, available() is False and the tests replay stored answers.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ref_preprocess_capi.cpp")
LIB_PATH = os.path.join(HERE, "_ref", "libpreprocess_ref.so")
REF = os.environ.get("REF", "/root/reference")
SHIMS = [os.path.join(HERE, "shim", p) for p in ("ros/ros.h", "pcl_conversions/pcl_conversions.h", "sensor_msgs/PointCloud2.h",
                                                  "livox_ros_driver/CustomMsg.h", "pcl/point_types.h")]

# field order of the off8 argument (and of fl_preprocess_params_t's offsets)
FIELDS = ("x", "y", "z", "intensity", "time", "ring", "tag", "line")

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def build(force: bool = False) -> None:
    """Compile oracle/_ref/libpreprocess_ref.so when the reference's src/preprocess.cpp is present."""
    src = os.path.join(REF, "src", "preprocess.cpp")
    if not os.path.exists(src):
        return
    deps = [SRC, src, os.path.join(REF, "src", "preprocess.h")] + SHIMS
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(d) <= os.path.getmtime(LIB_PATH) for d in deps):
        return
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")     # as oracle/Makefile
    tmp = LIB_PATH + ".tmp"
    subprocess.check_call([cxx, "-O3", "-std=c++14", "-fPIC", "-fopenmp", "-w", "-shared",
                           "-I", os.path.join(HERE, "shim"), "-I", os.path.dirname(src), SRC, src, "-o", tmp, "-lpthread"])
    os.replace(tmp, LIB_PATH)


def available() -> bool:
    build()
    return os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        L.ref_preprocess.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _u8p, C.c_int, C.c_int, _i32p,
                                     _f32p, _f32p, C.c_int, C.POINTER(C.c_double)]
        L.ref_preprocess.restype = C.c_int
        _lib = L
    return _lib


def process(raw: np.ndarray, offsets, lidar_type: int, n_scans: int, scan_rate: int, time_unit: int, point_filter_num: int,
            blind: float, timed: bool = False):
    """Preprocess::process of one raw frame (a structured or (n, point_step) uint8 array) -> (xyzi (m, 4) f32, curvature (m,) f32),
    plus the seconds process() took when `timed`."""
    raw = np.ascontiguousarray(raw)
    n = len(raw)
    step = raw.dtype.itemsize if raw.dtype.fields else raw.shape[1]
    buf = np.ascontiguousarray(raw.view(np.uint8).reshape(-1)) if n else np.zeros(1, np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.int32).reshape(8)
    cap = max(n, 1)
    xyzi = np.empty((cap, 4), dtype=np.float32)
    ms = np.empty(cap, dtype=np.float32)
    sec = C.c_double(0.0)
    m = lib().ref_preprocess(lidar_type, n_scans, scan_rate, time_unit, point_filter_num, blind, buf, n, step, off, xyzi, ms, cap,
                             C.byref(sec))
    out = (xyzi[:m].copy(), ms[:m].copy())
    return out + (sec.value,) if timed else out
