"""A numpy restatement of Preprocess::process (src/preprocess.cpp of the reference) with feature extraction off: the paths
avia_handler :161-186, oust64_handler :253-279, velodyne_handler :284-322 + :399-455 and sim_handler :458-481.

Every arithmetic type is the reference's: float32 where it computes in float, float64 where C++ promotes to double.  The
reference's atan2(float, float) is the float overload (glibc's atan2f), which this module calls through ctypes from the
process's libm.  Also here: the Velodyne per-ring time recurrence as an associative scan of (t, a, b) maps, the form the
device runs.
"""
from __future__ import annotations

import ctypes
import ctypes.util

import numpy as np

AVIA, VELO16, OUST64, MARSIM = 1, 2, 3, 4
SEC, MS, US, NS = 0, 1, 2, 3

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.atan2f.restype = ctypes.c_float
_libm.atan2f.argtypes = [ctypes.c_float, ctypes.c_float]


def atan2f(y, x) -> np.float32:
    return np.float32(_libm.atan2f(float(y), float(x)))


def time_unit_scale(unit: int) -> np.float32:
    """preprocess.cpp:52-69: any other unit gives 1."""
    return np.float32({SEC: 1.e3, MS: 1.0, US: 1.e-3, NS: 1.e-6}.get(unit, 1.0))


def _range2(x, y, z):
    """x*x + y*y + z*z in float, then double"""
    return ((x * x + y * y) + z * z).astype(np.float64)


def avia(f, n_scans, pfn, blind):
    """f: dict of arrays x, y, z (f32), reflectivity, tag, line (u8), offset_time (u32).  Returns (rows kept, curvature)."""
    x, y, z = f["x"], f["y"], f["z"]
    n = len(x)
    i = np.arange(n)
    tag = f["tag"] & 0x30
    valid = (i >= 1) & (f["line"].astype(np.int64) < n_scans) & ((tag == 0x10) | (tag == 0x00))
    vnum = np.cumsum(valid)                                   # valid_num, uint, from row 1
    sel = valid & (vnum % pfn == 0)
    # pl_full is cleared and resized each call: row i-1 holds a point only when it was selected, else PCL's zero point
    psel = np.concatenate([[False], sel[:-1]])
    def prev(a):
        return np.where(psel, np.concatenate([[np.float32(0)], a[:-1]]), np.float32(0)).astype(np.float32)
    new = ((np.abs(x - prev(x)).astype(np.float64) > 1e-7) | (np.abs(y - prev(y)).astype(np.float64) > 1e-7)
           | (np.abs(z - prev(z)).astype(np.float64) > 1e-7))
    keep = sel & new & (_range2(x, y, z) > blind * blind)
    curv = f["offset_time"].astype(np.float32) / np.float32(1000000)
    return np.nonzero(keep)[0], curv


def oust64(f, pfn, blind, unit):
    x, y, z = f["x"], f["y"], f["z"]
    i = np.arange(len(x))
    keep = (i % pfn == 0) & ~(_range2(x, y, z) < blind * blind)
    curv = f["t"].astype(np.float32) * time_unit_scale(unit)
    return np.nonzero(keep)[0], curv.astype(np.float32)


def sim(f, blind):
    x, y, z = f["x"], f["y"], f["z"]
    keep = ~(_range2(x, y, z) < blind * blind)
    return np.nonzero(keep)[0], np.zeros(len(x), np.float32)


def velodyne_yaw(x, y):
    """yaw_angle: atan2f(y, x) as float, times 57.2957 in double"""
    return np.array([np.float64(atan2f(a, b)) for a, b in zip(y, x)], dtype=np.float64) * 57.2957


def velodyne(f, n_scans, scan_rate, pfn, blind, unit, yaw=None):
    """Returns (rows kept, curvature, given_offset_time).  yaw: the per-row yaw_angle (default velodyne_yaw)."""
    x, y, z = f["x"], f["y"], f["z"]
    n = len(x)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.float32), False
    i = np.arange(n)
    given = bool(f["time"][n - 1] > 0)
    curv = (f["time"] * time_unit_scale(unit)).astype(np.float32)
    keep = (i % pfn == 0) & (_range2(x, y, z) > blind * blind)
    if given:
        return np.nonzero(keep)[0], curv, True
    yaw = velodyne_yaw(x, y) if yaw is None else yaw
    omega_l = 0.361 * scan_rate
    is_first = [True] * n_scans
    yaw_fp = [0.0] * n_scans
    time_last = [np.float32(0)] * n_scans
    for k in range(n):
        layer = int(f["ring"][k])
        if is_first[layer]:
            yaw_fp[layer] = yaw[k]
            is_first[layer] = False
            curv[k] = 0.0
            time_last[layer] = np.float32(0)
            keep[k] = False                                   # the `continue` comes before the decimation
            continue
        c = lo_of(yaw[k], yaw_fp[layer], omega_l)
        if c < time_last[layer]:
            c = np.float32(np.float64(c) + 360.0 / omega_l)
        curv[k] = c
        time_last[layer] = c
    return np.nonzero(keep)[0], curv, False


def lo_of(yaw, yaw_fp, omega_l) -> np.float32:
    return np.float32((yaw_fp - yaw) / omega_l if yaw <= yaw_fp else (yaw_fp - yaw + 360.0) / omega_l)


# ---------------------------------------------------------------------------------------------------- the scan form
def compose(first, second):
    """(t2, a2, b2) o (t1, a1, b1) = (t1, F2(a1), F2(b1)) with F(c) = (t < c) ? b : a; arrays of float32 triples."""
    t1, a1, b1 = first
    t2, a2, b2 = second
    return (t1, np.where(t2 < a1, b2, a2).astype(np.float32), np.where(t2 < b1, b2, a2).astype(np.float32))


def scan_by_key(keys, t, a, b):
    """Segmented inclusive scan (Hillis-Steele) of the maps over runs of equal keys, each applied to c = 0.0f."""
    t, a, b = (np.asarray(v, np.float32).copy() for v in (t, a, b))
    keys = np.asarray(keys)
    n = len(keys)
    d = 1
    while d < n:
        same = np.zeros(n, bool)
        same[d:] = keys[d:] == keys[:-d]
        # every row j with keys[j - d] == keys[j] takes map(j - d .. j) = map(j) o map(j - d ..); runs are contiguous
        nt, na, nb = compose((t[:-d], a[:-d], b[:-d]), (t[d:], a[d:], b[d:]))
        m = same[d:]
        t[d:][m], a[d:][m], b[d:][m] = nt[m], na[m], nb[m]
        d *= 2
    zero = np.float32(0)
    return np.where(t < zero, b, a).astype(np.float32)


def sequential(keys, lo, hi):
    """The reference's loop for rows already grouped by ring: c = 0 at a run's start, then c = lo < c ? hi : lo."""
    out = np.empty(len(lo), np.float32)
    c, prev = np.float32(0), None
    for j, k in enumerate(keys):
        if k != prev:
            c, prev = np.float32(0), k
        c = hi[j] if lo[j] < c else lo[j]
        out[j] = c
    return out


# ---------------------------------------------------------------------------------------------------- whole frames
_TYPES = {AVIA: (("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("reflectivity", "u1"), ("offset_time", "<u4"), None, ("tag", "u1"), ("line", "u1")),
          VELO16: (("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), ("time", "<f4"), ("ring", "<u2"), None, None),
          OUST64: (("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), ("t", "<u4"), None, None, None),
          MARSIM: (("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), None, None, None, None)}


def decode(raw, offsets, lidar_type):
    """The fields of each row at the 8 byte offsets (x, y, z, intensity, time, ring, tag, line), in the reference's types for
    `lidar_type`; an absent field (-1) reads as 0."""
    raw = np.ascontiguousarray(raw)
    step = raw.dtype.itemsize if raw.dtype.fields else raw.shape[1]
    b = raw.view(np.uint8).reshape(-1, step) if len(raw) else np.zeros((0, step), np.uint8)
    out = {}
    for spec, off in zip(_TYPES[lidar_type], offsets):
        if spec is None:
            continue
        name, dt = spec
        dt = np.dtype(dt)
        if off < 0:
            out[name] = np.zeros(len(b), dt)
        else:
            out[name] = np.ascontiguousarray(b[:, off:off + dt.itemsize]).view(dt).reshape(-1)
    return out


def process(raw, offsets, lidar_type, n_scans, scan_rate, time_unit, pfn, blind):
    """Preprocess::process -> (xyzi (m, 4) float32, curvature (m,) float32), pl_surf in raw order."""
    f = decode(raw, offsets, lidar_type)
    if lidar_type == AVIA:
        rows, curv = avia(f, n_scans, pfn, blind)
        inten = f["reflectivity"].astype(np.float32)
    elif lidar_type == OUST64:
        rows, curv = oust64(f, pfn, blind, time_unit)
        inten = f["intensity"]
    elif lidar_type == VELO16:
        rows, curv, _ = velodyne(f, n_scans, scan_rate, pfn, blind, time_unit)
        inten = f["intensity"]
    else:
        rows, curv = sim(f, blind)
        inten = f["intensity"]
    xyzi = np.stack([f["x"], f["y"], f["z"], inten], axis=1).astype(np.float32)[rows] if len(rows) else np.zeros((0, 4), np.float32)
    return np.ascontiguousarray(xyzi), np.ascontiguousarray(curv[rows], dtype=np.float32)
