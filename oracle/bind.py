"""ctypes binding of the CPU oracle -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module (see oracle/fastlio_oracle.cpp header).  The product
package `fast_lio_b200` never imports it.

Two kNN back-ends feed the same restatement:
  * "reference": oracle/_ref/libikdtree_ref.so = the reference's unmodified
    include/ikd-Tree/ikd_Tree.cpp compiled from /root/reference (oracle/Makefile);
  * "port": oracle/knn_port.cpp.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "liboracle.so")
REF_PATH = os.path.join(HERE, "_ref", "libikdtree_ref.so")

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")

KNN_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float))


class PassLog(C.Structure):
    _fields_ = [("searched", C.c_int), ("valid", C.c_int), ("effct", C.c_int), ("converged", C.c_int),
                ("res_sum", C.c_double), ("HtH", C.c_double * 144), ("Hth", C.c_double * 12),
                ("x_after", C.c_double * 26)]


class LocalMapState(C.Structure):
    _fields_ = [("vmin", C.c_float * 3), ("vmax", C.c_float * 3), ("initialized", C.c_int)]


def build(force: bool = False) -> None:
    """Compile oracle/liboracle.so and, when /root/reference is present, oracle/_ref."""
    srcs = [os.path.join(HERE, f) for f in ("fastlio_oracle.cpp", "knn_port.cpp", "frontend_oracle.cpp")]
    stale = os.path.exists(LIB_PATH) and any(os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in srcs)
    if force or stale or not os.path.exists(LIB_PATH) or (os.path.isdir("/root/reference") and not os.path.exists(REF_PATH)):
        subprocess.check_call(["make", "-C", HERE], stdout=subprocess.DEVNULL)


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        assert L.oracle_pass_log_size() == C.sizeof(PassLog)
        L.oracle_esti_plane.argtypes = [_f32p, C.c_float, _f32p]
        L.oracle_esti_plane.restype = C.c_int
        L.oracle_esti_plane_trace.argtypes = [_f32p, C.c_float, _f32p, _i32p]
        L.oracle_esti_plane_trace.restype = C.c_int
        L.oracle_measure_point.argtypes = [_f64p, _f32p, _f32p, C.c_int, C.c_float, C.c_int, _f64p]
        L.oracle_measure_point.restype = None
        L.oracle_state_boxplus.argtypes = [_f64p, _f64p]
        L.oracle_state_boxminus.argtypes = [_f64p, _f64p, _f64p]
        L.oracle_inverse.argtypes = [_f64p, _f64p, C.c_int]
        L.oracle_A_matrix.argtypes = [_f64p, _f64p]
        L.oracle_transform_point.argtypes = [_f64p, _f32p, _f32p]
        L.oracle_update_iterated.argtypes = [_f32p, C.c_int, _f64p, _f64p, C.c_int, C.c_double, _f64p, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_int,
                                             _f32p, _i32p, _u8p, C.POINTER(PassLog), C.POINTER(C.c_int)]
        L.oracle_update_iterated.restype = C.c_int
        L.port_kdtree_build.argtypes = [_f32p, C.c_int]
        L.port_kdtree_build.restype = C.c_void_p
        L.port_kdtree_destroy.argtypes = [C.c_void_p]
        L.port_kdtree_knn.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, _f32p, _f32p, _i32p, C.c_int]
        L.oracle_fov_segment.argtypes = [C.POINTER(LocalMapState), _f64p, C.c_double, C.c_float, _f32p]
        L.oracle_fov_segment.restype = C.c_int
        L.oracle_undistort.argtypes = [_f32p, _f32p, C.c_int, _f64p, C.c_int, _f64p]
        L.oracle_undistort.restype = None
        L.oracle_voxelgrid.argtypes = [_f32p, C.c_int, C.c_float, _f32p]
        L.oracle_voxelgrid.restype = C.c_int
        _lib = L
    return _lib


def have_ref() -> bool:
    build()
    return os.path.exists(REF_PATH)


def ref():
    global _ref
    if _ref is None:
        build()
        R = C.CDLL(REF_PATH)
        R.ref_kdtree_create.argtypes = [C.c_float, C.c_float, C.c_float]
        R.ref_kdtree_create.restype = C.c_void_p
        R.ref_kdtree_destroy.argtypes = [C.c_void_p]
        R.ref_kdtree_set_downsample.argtypes = [C.c_void_p, C.c_float]
        R.ref_kdtree_build.argtypes = [C.c_void_p, _f32p, C.c_int]
        R.ref_kdtree_size.argtypes = [C.c_void_p]
        R.ref_kdtree_validnum.argtypes = [C.c_void_p]
        R.ref_kdtree_knn.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, _f32p, _f32p, _i32p, C.c_int]
        R.ref_kdtree_add.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int]
        R.ref_kdtree_add.restype = C.c_int
        R.ref_kdtree_delete_boxes.argtypes = [C.c_void_p, _f32p, C.c_int]
        R.ref_kdtree_delete_boxes.restype = C.c_int
        R.ref_kdtree_flatten.argtypes = [C.c_void_p, _f32p, C.c_int]
        R.ref_kdtree_flatten.restype = C.c_int
        _ref = R
    return _ref


class KdTree:
    """Exact kNN map with the ikd-Tree semantics.  backend = "reference" | "port" | "auto"."""

    def __init__(self, pts4: np.ndarray, backend: str = "auto", downsample: float = 0.5):
        pts4 = np.ascontiguousarray(pts4, dtype=np.float32)
        if backend == "auto":
            backend = "reference" if have_ref() else "port"
        self.backend = backend
        if backend == "reference":
            R = ref()
            self.h = C.c_void_p(R.ref_kdtree_create(0.5, 0.6, 0.2))
            R.ref_kdtree_set_downsample(self.h, downsample)
            R.ref_kdtree_build(self.h, pts4, len(pts4))
            self.knn1_addr = C.cast(R.ref_kdtree_knn1, C.c_void_p)
        elif backend == "port":
            L = lib()
            self.h = C.c_void_p(L.port_kdtree_build(pts4, len(pts4)))
            self.knn1_addr = C.cast(L.port_kdtree_knn1, C.c_void_p)
        else:
            raise ValueError(backend)

    def close(self):
        if self.h:
            if self.backend == "reference":
                ref().ref_kdtree_destroy(self.h)
            else:
                lib().port_kdtree_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def knn(self, q4: np.ndarray, k: int = 5, nthreads: int = 0):
        q4 = np.ascontiguousarray(q4, dtype=np.float32)
        nq = len(q4)
        pts = np.zeros((nq, k, 4), dtype=np.float32)
        d2 = np.full((nq, k), np.inf, dtype=np.float32)
        cnt = np.zeros(nq, dtype=np.int32)
        fn = ref().ref_kdtree_knn if self.backend == "reference" else lib().port_kdtree_knn
        fn(self.h, q4, nq, k, pts, d2, cnt, nthreads)
        return pts, d2, cnt

    # --- mutation (reference back-end only)
    def add(self, pts4, downsample_on: bool) -> int:
        assert self.backend == "reference"
        pts4 = np.ascontiguousarray(pts4, dtype=np.float32)
        return ref().ref_kdtree_add(self.h, pts4, len(pts4), int(downsample_on))

    def delete_boxes(self, boxes6) -> int:
        assert self.backend == "reference"
        boxes6 = np.ascontiguousarray(boxes6, dtype=np.float32).reshape(-1, 6)
        return ref().ref_kdtree_delete_boxes(self.h, boxes6, len(boxes6))

    def size(self) -> int:
        assert self.backend == "reference"
        return ref().ref_kdtree_size(self.h)

    def validnum(self) -> int:
        assert self.backend == "reference"
        return ref().ref_kdtree_validnum(self.h)

    def flatten(self) -> np.ndarray:
        assert self.backend == "reference"
        cap = max(1, self.size() + 16)
        out = np.zeros((cap, 4), dtype=np.float32)
        n = ref().ref_kdtree_flatten(self.h, out, cap)
        return out[:n].copy()


class UpdateResult:
    pass


def update_iterated(tree: KdTree, scan4, x26, P, max_iter, R=0.001, limit=0.001, extrinsic_est_en=0, nthreads=0):
    """Run the restated update_iterated_dyn_share_modified on the CPU.  Returns an object with
    x (26), P (23x23), nearest (Q,5,4), nearest_cnt (Q), selected (Q), passes (list of dict)."""
    L = lib()
    scan4 = np.ascontiguousarray(scan4, dtype=np.float32)
    Q = len(scan4)
    x = np.array(x26, dtype=np.float64).copy()
    Pm = np.ascontiguousarray(np.array(P, dtype=np.float64).copy())
    lim = np.full(23, limit, dtype=np.float64)
    nearest = np.zeros((Q, 5, 4), dtype=np.float32)
    ncnt = np.zeros(Q, dtype=np.int32)
    sel = np.zeros(Q, dtype=np.uint8)
    logs = (PassLog * (max_iter + 2))()
    npass = C.c_int(0)
    rc = L.oracle_update_iterated(scan4, Q, x, Pm, max_iter, R, lim, extrinsic_est_en,
                                  tree.knn1_addr, tree.h, nthreads, nearest, ncnt, sel, logs, C.byref(npass))
    assert rc == 0
    r = UpdateResult()
    r.x, r.P, r.nearest, r.nearest_cnt, r.selected = x, Pm, nearest, ncnt, sel
    r.passes = []
    for i in range(npass.value):
        l = logs[i]
        r.passes.append(dict(searched=l.searched, valid=l.valid, effct=l.effct, converged=l.converged,
                             res_sum=l.res_sum, HtH=np.array(l.HtH).reshape(12, 12).copy(),
                             Hth=np.array(l.Hth).copy(), x_after=np.array(l.x_after).copy()))
    return r


def esti_plane(pts5x3, threshold=0.1):
    out = np.zeros(4, dtype=np.float32)
    ok = lib().oracle_esti_plane(np.ascontiguousarray(pts5x3, dtype=np.float32).reshape(-1), threshold, out)
    return bool(ok), out


def esti_plane_trace(pts5x3, threshold=0.1):
    """esti_plane plus the branches it took: (ok, pabcd, trace) with trace = dict(nonzero_pivots, transp (3),
    tiny_tail (3), norm (3x3): 0 not visited, 1 downdated, 2 recomputed, 3 skipped as a zero column)."""
    out = np.zeros(4, dtype=np.float32)
    tr = np.zeros(16, dtype=np.int32)
    ok = lib().oracle_esti_plane_trace(np.ascontiguousarray(pts5x3, dtype=np.float32).reshape(-1), threshold, out, tr)
    return bool(ok), out, dict(nonzero_pivots=int(tr[0]), transp=tr[1:4].copy(), tiny_tail=tr[4:7].copy(), norm=tr[7:16].reshape(3, 3).copy())


def measure_point(x26, pb3, near5x3, cnt, d2_last, extrinsic_est_en):
    """One point of h_share_model with every stage evaluated: 25 doubles = world point (3), kNN gate, plane ok,
    score gate, pabcd (4), pd2, score, row (12), h."""
    out = np.zeros(25)
    lib().oracle_measure_point(np.ascontiguousarray(x26, dtype=np.float64), np.ascontiguousarray(pb3, dtype=np.float32).reshape(-1),
                               np.ascontiguousarray(near5x3, dtype=np.float32).reshape(-1), int(cnt), float(d2_last),
                               int(extrinsic_est_en), out)
    return out


class LocalMap:
    """lasermap_fov_segment (laserMapping.cpp:229-277) restated; one segment() per scan."""

    def __init__(self, cube_len: float, det_range: float):
        self.st = LocalMapState()
        self.cube_len, self.det_range = float(cube_len), float(det_range)

    def segment(self, pos_lid) -> np.ndarray:
        boxes = np.zeros((3, 6), dtype=np.float32)
        nb = lib().oracle_fov_segment(C.byref(self.st), np.ascontiguousarray(pos_lid, dtype=np.float64), self.cube_len, self.det_range, boxes)
        return boxes[:nb].copy()

    def box(self) -> np.ndarray:
        return np.array(list(self.st.vmin) + list(self.st.vmax), dtype=np.float32)


def undistort(xyzi, offset_ms, imu_pose22, x26_end):
    """UndistortPcl: stable sort by offset time (IMU_Processing.hpp:234) + backward pass (:312-346).  Returns (pts, t)."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    t = np.ascontiguousarray(offset_ms, dtype=np.float32).reshape(-1)
    order = np.argsort(t, kind="stable")
    pts, ts = np.ascontiguousarray(xyzi[order]), np.ascontiguousarray(t[order])
    poses = np.ascontiguousarray(imu_pose22, dtype=np.float64).reshape(-1, 22)
    lib().oracle_undistort(pts, ts, len(pts), poses, len(poses), np.ascontiguousarray(x26_end, dtype=np.float64))
    return pts, ts


def voxelgrid(xyzi, leaf: float) -> np.ndarray:
    """pcl::VoxelGrid::filter as called at laserMapping.cpp:904-905 (restated; see frontend_oracle.cpp)."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    out = np.zeros((max(len(xyzi), 1), 4), dtype=np.float32)
    n = lib().oracle_voxelgrid(xyzi, len(xyzi), leaf, out)
    return out[:n].copy()
