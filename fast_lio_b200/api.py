"""ctypes binding of libfastlio_b200.so (the C ABI in include/fastlio_b200.h).

The reference is C++ (no Python anywhere), so this module is only the harness the tests,
bench.py and __graft_entry__ use to reach the product; names mirror the reference's two
classes: `KdTree` ~ KD_TREE<PointType> (include/ikd-Tree/ikd_Tree.h:48-341) and `Esekf` ~
esekfom::esekf<state_ikfom,12,input_ikfom> (include/IKFoM_toolkit/esekfom/esekfom.hpp:105).

There is no CPU fallback: a missing library or a missing GPU raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


class PassLog(C.Structure):
    _fields_ = [("searched", C.c_int), ("valid", C.c_int), ("effct", C.c_int), ("converged", C.c_int),
                ("res_sum", C.c_double), ("HtH", C.c_double * 144), ("Hth", C.c_double * 12),
                ("x_after", C.c_double * 26)]


def _log_dict(l: PassLog) -> dict:
    return dict(searched=l.searched, valid=l.valid, effct=l.effct, converged=l.converged,
                res_sum=l.res_sum, HtH=np.array(l.HtH).reshape(12, 12).copy(),
                Hth=np.array(l.Hth).copy(), x_after=np.array(l.x_after).copy())


def decode_pass_logs(raw, passes: int) -> list:
    """The first `passes` entries of one hypothesis's log bytes from Esekf.update_batch_device (a (max_iter + 1,
    sizeof(fl_pass_log_t)) uint8 array or tensor) as the dicts Esekf.pass_logs() returns."""
    if hasattr(raw, "cpu"):
        raw = raw.cpu().numpy()
    buf = np.ascontiguousarray(raw, dtype=np.uint8).reshape(-1, C.sizeof(PassLog))
    if not 0 <= passes <= len(buf):
        raise ValueError(f"passes must be in [0, {len(buf)}], got {passes}")
    return [_log_dict(PassLog.from_buffer_copy(buf[i].tobytes())) for i in range(passes)]


class RelocGrid(C.Structure):
    """fl_reloc_grid_t: grid counts and steps on x, y, z (m) and yaw (rad)"""
    _fields_ = [("n", C.c_int * 4), ("step", C.c_double * 4)]


class RelocParams(C.Structure):
    """fl_reloc_params_t"""
    _fields_ = [("keep", C.c_int), ("stride", C.c_int), ("r_inlier", C.c_float), ("min_effct", C.c_int)]


class RelocRow(C.Structure):
    """fl_reloc_row_t: one survivor of a relocalisation's screen"""
    _fields_ = [("hyp", C.c_int), ("inliers", C.c_int), ("status", C.c_int), ("passes", C.c_int), ("effct", C.c_int),
                ("pad", C.c_int), ("res_sum", C.c_double)]


RELOC_ROW = np.dtype({"names": ["hyp", "inliers", "status", "passes", "effct", "res_sum"],
                      "formats": ["<i4"] * 5 + ["<f8"], "offsets": [0, 4, 8, 12, 16, 24], "itemsize": 32})


def decode_reloc_rows(raw) -> np.ndarray:
    """The rows of Esekf.relocalize_device (a (keep, sizeof(fl_reloc_row_t)) uint8 array or tensor) as a structured array with the
    fields hyp, inliers, status, passes, effct and res_sum."""
    if hasattr(raw, "cpu"):
        raw = raw.cpu().numpy()
    return np.ascontiguousarray(raw, dtype=np.uint8).reshape(-1).view(RELOC_ROW).copy()


class ScanRef(C.Structure):
    """fl_scan_ref_t: a scan's rows and its row count, both in device memory"""
    _fields_ = [("body_xyzi", C.c_void_p), ("n", C.c_void_p)]


def scan_refs(pairs, device=None):
    """The device table of fl_filter_update_scans_device: an (S, 2) int64 CUDA tensor of fl_scan_ref_t rows.  Each entry is a
    `Scan` (Scan.ref(): its device forms' feats_down_body and feats_down_size) or a (rows, n) pair: rows an (m, 4) float32 CUDA
    tensor and n a one-element int32 CUDA tensor, or either one a raw device address (an int, 0 for null).  The table is copied
    from the host, so build it outside stream capture; what it points at must outlive the calls that read it."""
    import torch

    def addr(v, name):
        if isinstance(v, torch.Tensor):
            if not v.is_cuda or not v.is_contiguous():
                raise ValueError(f"scan_refs: {name} must be a contiguous CUDA tensor")
            return v.data_ptr()
        return int(v or 0)

    rows = []
    for p in pairs:
        if isinstance(p, Scan):
            b, n, _ = p.ref()
        else:
            body, n = p
            if isinstance(body, torch.Tensor) and (body.dtype != torch.float32 or body.dim() != 2 or body.shape[1] != 4):
                raise ValueError("scan_refs: rows must be an (m, 4) float32 tensor")
            if isinstance(n, torch.Tensor) and n.dtype != torch.int32:
                raise ValueError("scan_refs: n must be an int32 tensor")
            b, n = addr(body, "rows"), addr(n, "n")
        rows.append((b, n))
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 2).to(device)


class ScanRaw(C.Structure):
    """fl_scan_raw_t: one slot's raw scan for fl_scan_batch_run_device, every pointer in device memory"""
    _fields_ = [("xyzi", C.c_void_p), ("offset_ms", C.c_void_p), ("n", C.c_void_p), ("imu_pose22", C.c_void_p), ("n_pose", C.c_void_p),
                ("x26_end", C.c_void_p)]


def scan_raws(entries, device=None):
    """The device table of fl_scan_batch_run_device: an (S, 6) int64 CUDA tensor of fl_scan_raw_t rows.  Each entry is a tuple
    (xyzi, offset_ms, n, imu_pose22, n_pose, x26_end), or a dict with those keys (imu_pose22, n_pose and x26_end may be left out
    when not de-skewing): xyzi an (m, 4) float32, offset_ms an (m,) float32, n and n_pose one-element int32, imu_pose22 an
    (n_pose_max, 22) float64 and x26_end a (26,) float64 CUDA tensor, or any of them a raw device address (an int, 0 or None for
    null).  The table is copied from the host, so build it outside stream capture; what it points at must stay alive until the
    stream has passed the calls that read it."""
    import torch
    names = ("xyzi", "offset_ms", "n", "imu_pose22", "n_pose", "x26_end")
    dtypes = (torch.float32, torch.float32, torch.int32, torch.float64, torch.int32, torch.float64)
    rows = []
    for e in entries:
        vals = [e.get(k) for k in names] if isinstance(e, dict) else list(e) + [None] * (6 - len(e))
        row = []
        for v, name, dt in zip(vals, names, dtypes):
            if isinstance(v, torch.Tensor):
                if not v.is_cuda or not v.is_contiguous() or v.dtype != dt:
                    raise ValueError(f"scan_raws: {name} must be a contiguous {dt} CUDA tensor")
                row.append(v.data_ptr())
            else:
                row.append(int(v or 0))
        rows.append(row)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 6).to(device)


class PreprocessRaw(C.Structure):
    """fl_preprocess_raw_t: one slot's raw frame for fl_preprocess_batch_run_device, both pointers in device memory"""
    _fields_ = [("raw", C.c_void_p), ("n_raw", C.c_void_p)]


def preprocess_raws(entries, device=None):
    """The device table of fl_preprocess_batch_run_device: an (S, 2) int64 CUDA tensor of fl_preprocess_raw_t rows.  Each entry
    is a (raw, n_raw) pair: raw a contiguous uint8 CUDA tensor of the frame's points (point_step bytes each), n_raw a one-element
    int32 CUDA tensor, or either one a raw device address (an int, 0 or None for null).  The table is copied from the host, so
    build it outside stream capture; what it points at must stay alive until the stream has passed the calls that read it."""
    import torch
    rows = []
    for raw, n in entries:
        row = []
        for v, name, dt in ((raw, "raw", torch.uint8), (n, "n_raw", torch.int32)):
            if isinstance(v, torch.Tensor):
                if not v.is_cuda or not v.is_contiguous() or v.dtype != dt:
                    raise ValueError(f"preprocess_raws: {name} must be a contiguous {dt} CUDA tensor")
                row.append(v.data_ptr())
            else:
                row.append(int(v or 0))
        rows.append(row)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 2).to(device)


class FastLioError(RuntimeError):
    pass

# the frames of Scan.frame / frame_device: as stored, RGBpointBodyLidarToIMU, RGBpointBodyToWorld (laserMapping.cpp:200-220)
FRAME_LIDAR, FRAME_IMU, FRAME_WORLD = 0, 1, 2

# ---- sensor preprocessing: the reference's raw point structs as numpy dtypes (the default layouts of Preprocess)
LIDAR_AVIA, LIDAR_VELO16, LIDAR_OUST64, LIDAR_MARSIM = 1, 2, 3, 4          # enum LID_TYPE, preprocess.h:16
TIME_SEC, TIME_MS, TIME_US, TIME_NS = 0, 1, 2, 3                           # enum TIME_UNIT, preprocess.h:17
# livox_ros_driver::CustomPoint: 20 bytes
CUSTOM_POINT = np.dtype({"names": ["offset_time", "x", "y", "z", "reflectivity", "tag", "line"],
                         "formats": ["<u4", "<f4", "<f4", "<f4", "u1", "u1", "u1"],
                         "offsets": [0, 4, 8, 12, 16, 17, 18], "itemsize": 20})
# velodyne_ros::Point (preprocess.h:41-49): PCL_ADD_POINT4D, 16-byte aligned, 32 bytes
VELODYNE_POINT = np.dtype({"names": ["x", "y", "z", "intensity", "time", "ring"],
                           "formats": ["<f4", "<f4", "<f4", "<f4", "<f4", "<u2"],
                           "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
# ouster_ros::Point (preprocess.h:59-84): 48 bytes
OUSTER_POINT = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                         "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "u1", "<u2", "<u4"],
                         "offsets": [0, 4, 8, 16, 20, 24, 26, 28, 32], "itemsize": 48})
# pcl::PointXYZI (MARSIM): 32 bytes
POINT_XYZI = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 16], "itemsize": 32})
DEFAULT_LAYOUT = {LIDAR_AVIA: CUSTOM_POINT, LIDAR_VELO16: VELODYNE_POINT, LIDAR_OUST64: OUSTER_POINT, LIDAR_MARSIM: POINT_XYZI}
# fl_preprocess_params_t's offsets, in order, and the struct member each one is in the reference's point type
OFFSET_FIELDS = ("x", "y", "z", "intensity", "time", "ring", "tag", "line")
_FIELD_NAMES = {LIDAR_AVIA: {"intensity": "reflectivity", "time": "offset_time"}, LIDAR_OUST64: {"time": "t"}}


def layout_offsets(dtype: np.dtype, lidar_type: int) -> list[int]:
    """The 8 byte offsets (x, y, z, intensity, time, ring, tag, line) of a structured dtype for `lidar_type`, -1 where the dtype
    has no such field; Avia's intensity is `reflectivity` and its time `offset_time`, Ouster's time is `t`."""
    names = _FIELD_NAMES.get(lidar_type, {})
    fields = dtype.fields or {}
    return [int(fields[names.get(f, f)][1]) if names.get(f, f) in fields else -1 for f in OFFSET_FIELDS]


class PreprocessParams(C.Structure):
    """fl_preprocess_params_t"""
    _fields_ = [("lidar_type", C.c_int), ("n_scans", C.c_int), ("scan_rate", C.c_int), ("time_unit", C.c_int),
                ("point_filter_num", C.c_int), ("blind", C.c_double), ("point_step", C.c_int)] + \
               [("off_" + f, C.c_int) for f in OFFSET_FIELDS]


_lib = None

# every symbol include/fastlio_b200.h declares (tests check that the library exports all of them)
SYMBOLS = [
    "fl_last_error", "fl_device_count", "fl_version", "fl_host_register", "fl_host_unregister", "fl_filter_debug_prof",
    "fl_map_create", "fl_map_destroy", "fl_map_set_downsample", "fl_map_build", "fl_map_size", "fl_map_validnum",
    "fl_map_knn", "fl_map_nearest_search", "fl_map_add_points", "fl_map_delete_boxes", "fl_map_flatten", "fl_map_tree_range",
    "fl_map_rebuild", "fl_map_stats", "fl_map_add_boxes", "fl_map_box_search", "fl_map_radius_search", "fl_map_acquire_removed", "fl_map_set_cell_directory", "fl_map_dir_stats",
    "fl_map_set_deterministic", "fl_map_get_deterministic",
    "fl_map_nearest_search_device", "fl_map_range_workspace_bytes", "fl_map_box_search_device", "fl_map_radius_search_device",
    "fl_map_build_device", "fl_map_add_points_device",
    "fl_filter_create", "fl_filter_destroy", "fl_filter_set_params", "fl_filter_set_solver", "fl_filter_set_search", "fl_filter_set_fused", "fl_filter_update",
    "fl_filter_map_incremental", "fl_filter_get_nearest", "fl_filter_get_selected", "fl_filter_get_pass_logs", "fl_filter_upload_scan",
    "fl_filter_upload_state", "fl_filter_run", "fl_filter_download_state", "fl_filter_sync",
    "fl_filter_time_resident", "fl_filter_time_search_pass", "fl_filter_time_e2e", "fl_filter_gpu_launches",
    "fl_scan_create", "fl_scan_destroy", "fl_scan_upload", "fl_scan_undistort", "fl_scan_voxel_downsample", "fl_scan_download",
    "fl_filter_update_scan", "fl_localmap_create", "fl_localmap_destroy", "fl_localmap_segment", "fl_localmap_get",
    "fl_comm_unique_id", "fl_filter_comm_init", "fl_filter_set_shard", "fl_filter_p2p_handle", "fl_filter_p2p_connect",
    "fl_filter_update_device", "fl_filter_get_nearest_device", "fl_filter_get_selected_device",
    "fl_map_add_points_async", "fl_map_maintain", "fl_filter_map_incremental_device",
    "fl_scan_reserve", "fl_scan_upload_device", "fl_scan_undistort_device", "fl_scan_voxel_downsample_device",
    "fl_filter_update_scan_device", "fl_map_delete_boxes_async", "fl_localmap_segment_device",
    "fl_filter_reserve_batch", "fl_filter_batch_plan", "fl_filter_update_batch_device",
    "fl_reloc_expand_grid_device", "fl_filter_reserve_reloc", "fl_filter_relocalize_device",
    "fl_preprocess_create", "fl_preprocess_destroy", "fl_preprocess_device", "fl_preprocess",
    "fl_scan_frame", "fl_scan_frame_device",
    "fl_scan_get_ref", "fl_filter_update_scans_device",
    "fl_scan_batch_create", "fl_scan_batch_destroy", "fl_scan_batch_reserve", "fl_scan_batch_run_device", "fl_scan_batch_get_refs",
    "fl_scan_batch_download",
    "fl_preprocess_batch_create", "fl_preprocess_batch_destroy", "fl_preprocess_batch_run_device", "fl_preprocess_batch_get_outputs",
    "fl_preprocess_batch_download",
]


def lib_path() -> str:
    return _build.LIB


def load():
    """Load libfastlio_b200.so (never builds implicitly on a GPU box: the .so ships with the tree)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_build.LIB):
        raise FastLioError(f"{_build.LIB} is missing -- run `python -m fast_lio_b200.build` (nvcc, sm_90a); "
                           "there is no CPU fallback")
    L = C.CDLL(_build.LIB)
    L.fl_last_error.restype = C.c_char_p
    L.fl_host_register.argtypes = [C.c_void_p, C.c_ulonglong]
    L.fl_host_unregister.argtypes = [C.c_void_p]
    L.fl_map_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_float]
    L.fl_map_destroy.argtypes = [C.c_void_p]
    L.fl_map_set_downsample.argtypes = [C.c_void_p, C.c_float]
    L.fl_map_build.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_map_size.argtypes = [C.c_void_p]
    L.fl_map_validnum.argtypes = [C.c_void_p]
    L.fl_map_knn.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, _f32p, _f32p, _i32p]
    L.fl_map_nearest_search.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_float, _f32p, _f32p, _i32p]
    L.fl_map_add_points.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int]
    L.fl_map_delete_boxes.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_map_flatten.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_map_box_search.argtypes = [C.c_void_p, _f32p, C.c_int, _i32p, _f32p, C.c_int]
    L.fl_map_radius_search.argtypes = [C.c_void_p, _f32p, C.c_int, _i32p, _f32p, C.c_int]
    L.fl_map_add_boxes.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_map_acquire_removed.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_map_tree_range.argtypes = [C.c_void_p, _f32p]
    L.fl_map_rebuild.argtypes = [C.c_void_p]
    L.fl_map_stats.argtypes = [C.c_void_p, _i32p]
    L.fl_map_set_cell_directory.argtypes = [C.c_void_p, C.c_int, C.c_float]
    L.fl_map_dir_stats.argtypes = [C.c_void_p, _i32p]
    L.fl_map_set_deterministic.argtypes = [C.c_void_p, C.c_int]
    L.fl_map_get_deterministic.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    # device-buffer forms: raw device addresses and a cudaStream_t
    _vp = C.c_void_p
    L.fl_map_nearest_search_device.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_float, _vp, _vp, _vp, _vp]
    L.fl_map_range_workspace_bytes.argtypes = [_vp, C.c_int, C.c_longlong, C.POINTER(C.c_ulonglong)]
    for fn in (L.fl_map_box_search_device, L.fl_map_radius_search_device):
        fn.argtypes = [_vp, _vp, C.c_int, _vp, _vp, C.c_longlong, _vp, C.c_ulonglong, _vp, _vp]
    L.fl_map_build_device.argtypes = [_vp, _vp, C.c_int, _vp]
    L.fl_map_add_points_device.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp]
    L.fl_map_add_points_async.argtypes = [_vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp]
    L.fl_map_maintain.argtypes = [_vp, C.POINTER(C.c_int)]
    L.fl_map_delete_boxes_async.argtypes = [_vp, _vp, _vp, C.c_int, _vp, _vp]
    L.fl_filter_map_incremental_device.argtypes = [_vp, C.c_double, C.c_int, _vp, _vp]
    L.fl_filter_update_device.argtypes = [_vp, _vp, C.c_int, _vp, _vp, C.c_double, _vp, _vp]
    L.fl_filter_get_nearest_device.argtypes = [_vp, _vp, _vp, C.c_int, _vp]
    L.fl_filter_get_selected_device.argtypes = [_vp, _vp, C.c_int, _vp]
    L.fl_filter_reserve_batch.argtypes = [_vp, C.c_int]
    L.fl_filter_batch_plan.argtypes = [_vp, C.c_int, C.c_int, _i32p]
    L.fl_filter_update_batch_device.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp, _vp, C.c_double, _vp, _vp, _vp]
    L.fl_filter_update_scans_device.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp, _vp, C.c_double, _vp, _vp, _vp]
    L.fl_scan_get_ref.argtypes = [_vp, C.POINTER(ScanRef), C.POINTER(C.c_int)]
    L.fl_scan_batch_create.argtypes = [C.POINTER(C.c_void_p), _vp]
    L.fl_scan_batch_destroy.argtypes = [_vp]
    L.fl_scan_batch_reserve.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.fl_scan_batch_run_device.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _vp, _vp]
    L.fl_scan_batch_get_refs.argtypes = [_vp, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
    L.fl_scan_batch_download.argtypes = [_vp, C.c_int, C.c_int, _f32p, C.c_int]
    L.fl_reloc_expand_grid_device.argtypes = [_vp, C.POINTER(RelocGrid), _vp, _vp]
    L.fl_filter_reserve_reloc.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.fl_filter_relocalize_device.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp, _vp, C.c_double, C.POINTER(RelocParams), _vp, _vp,
                                              _vp, _vp, _vp, _vp]
    L.fl_filter_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int]
    L.fl_filter_destroy.argtypes = [C.c_void_p]
    L.fl_filter_set_params.argtypes = [C.c_void_p, C.c_int, _f64p, C.c_int]
    L.fl_filter_set_solver.argtypes = [C.c_void_p, C.c_int]
    L.fl_filter_set_search.argtypes = [C.c_void_p, C.c_int]
    L.fl_filter_set_fused.argtypes = [C.c_void_p, C.c_int]
    L.fl_filter_update.argtypes = [C.c_void_p, _f32p, C.c_int, _f64p, _f64p, C.c_double, C.POINTER(C.c_double)]
    L.fl_filter_map_incremental.argtypes = [C.c_void_p, C.c_double, C.c_int, _i32p]
    L.fl_filter_get_nearest.argtypes = [C.c_void_p, _f32p, _i32p, C.c_int]
    L.fl_filter_get_selected.argtypes = [C.c_void_p, _u8p, C.c_int]
    L.fl_filter_get_pass_logs.argtypes = [C.c_void_p, C.POINTER(PassLog), C.c_int]
    L.fl_filter_upload_scan.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.fl_filter_upload_state.argtypes = [C.c_void_p, _f64p, _f64p, C.c_double]
    L.fl_filter_run.argtypes = [C.c_void_p]
    L.fl_filter_download_state.argtypes = [C.c_void_p, _f64p, _f64p, C.POINTER(C.c_int)]
    L.fl_filter_sync.argtypes = [C.c_void_p]
    L.fl_filter_time_resident.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]
    L.fl_filter_time_search_pass.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]
    L.fl_filter_gpu_launches.argtypes = [C.c_void_p]
    L.fl_filter_time_e2e.argtypes = [C.c_void_p, _f32p, C.c_int, _f64p, _f64p, C.c_double, C.c_int, C.POINTER(C.c_double), _f64p, _f64p]
    L.fl_scan_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p]
    L.fl_scan_destroy.argtypes = [C.c_void_p]
    L.fl_scan_upload.argtypes = [C.c_void_p, _f32p, _f32p, C.c_int]
    L.fl_scan_undistort.argtypes = [C.c_void_p, _f64p, C.c_int, _f64p]
    L.fl_scan_voxel_downsample.argtypes = [C.c_void_p, C.c_float]
    L.fl_scan_download.argtypes = [C.c_void_p, C.c_int, _f32p, C.c_int]
    L.fl_filter_update_scan.argtypes = [C.c_void_p, C.c_void_p, _f64p, _f64p, C.c_double, C.POINTER(C.c_double)]
    L.fl_scan_reserve.argtypes = [_vp, C.c_int, C.c_int]
    L.fl_scan_upload_device.argtypes = [_vp, _vp, _vp, _vp, C.c_int, _vp]
    L.fl_scan_undistort_device.argtypes = [_vp, _vp, _vp, C.c_int, _vp, _vp]
    L.fl_scan_voxel_downsample_device.argtypes = [_vp, C.c_float, _vp, _vp]
    L.fl_filter_update_scan_device.argtypes = [_vp, _vp, _vp, _vp, C.c_double, _vp, _vp]
    L.fl_scan_frame.argtypes = [_vp, C.c_int, C.c_int, _vp, _f32p, C.c_int]
    L.fl_scan_frame_device.argtypes = [_vp, C.c_int, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp]
    L.fl_localmap_create.argtypes = [C.POINTER(C.c_void_p), C.c_double, C.c_float]
    L.fl_localmap_destroy.argtypes = [C.c_void_p]
    L.fl_localmap_segment.argtypes = [C.c_void_p, C.c_void_p, _f64p, _f32p, C.POINTER(C.c_int)]
    L.fl_localmap_get.argtypes = [C.c_void_p, _f32p]
    L.fl_localmap_segment_device.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp]
    L.fl_preprocess_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(PreprocessParams), C.c_int]
    L.fl_preprocess_destroy.argtypes = [_vp]
    L.fl_preprocess_device.argtypes = [_vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp]
    L.fl_preprocess.argtypes = [_vp, _vp, C.c_int, _f32p, _f32p, C.c_int, C.POINTER(C.c_float)]
    L.fl_preprocess_batch_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(PreprocessParams), C.c_int, C.c_int]
    L.fl_preprocess_batch_destroy.argtypes = [_vp]
    L.fl_preprocess_batch_run_device.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp, _vp]
    _pp = C.POINTER(C.c_void_p)
    L.fl_preprocess_batch_get_outputs.argtypes = [_vp, _pp, _pp, _pp, _pp, C.POINTER(C.c_int)]
    L.fl_preprocess_batch_download.argtypes = [_vp, C.c_int, _f32p, _f32p, C.c_int, C.POINTER(C.c_float)]
    L.fl_comm_unique_id.argtypes = [C.c_char_p]
    L.fl_filter_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    L.fl_filter_set_shard.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.fl_filter_p2p_handle.argtypes = [C.c_void_p, C.c_char_p]
    L.fl_filter_p2p_connect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    _lib = L
    return L


def _check(rc: int) -> int:
    if rc < 0:
        raise FastLioError(f"fastlio_b200 error {rc}: {load().fl_last_error().decode(errors='replace')}")
    return rc


def device_count() -> int:
    return load().fl_device_count()


class KdTree:
    """Device point map with the KD_TREE<PointType> call surface used by laserMapping.cpp."""

    def __init__(self, device: int = 0, downsample: float = 0.5, cell_directory: bool = True, cell_size: float = 0.0):
        self._L = load()
        h = C.c_void_p()
        _check(self._L.fl_map_create(C.byref(h), device, downsample))
        self.h = h
        self.device = device
        if not cell_directory or cell_size > 0.0:
            _check(self._L.fl_map_set_cell_directory(self.h, int(cell_directory), cell_size))

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # extension: the deterministic mode (fl_map_set_deterministic): k-NN answers, the down-sampling survivor, the update and
    # flatten's row order depend only on the map's point set
    def set_deterministic(self, on: bool):
        _check(self._L.fl_map_set_deterministic(self.h, int(bool(on))))

    @property
    def deterministic(self) -> bool:
        on = C.c_int(0)
        _check(self._L.fl_map_get_deterministic(self.h, C.byref(on)))
        return bool(on.value)

    # KD_TREE::set_downsample_param
    def set_downsample_param(self, v: float):
        _check(self._L.fl_map_set_downsample(self.h, v))

    # KD_TREE::Build
    def Build(self, pts4):
        pts4 = np.ascontiguousarray(pts4, dtype=np.float32).reshape(-1, 4)
        _check(self._L.fl_map_build(self.h, pts4, len(pts4)))

    def size(self) -> int:
        return _check(self._L.fl_map_size(self.h))

    def validnum(self) -> int:
        return _check(self._L.fl_map_validnum(self.h))

    # KD_TREE::Nearest_Search, batched
    def Nearest_Search(self, q4, k: int = 5):
        q4 = np.ascontiguousarray(q4, dtype=np.float32).reshape(-1, 4)
        nq = len(q4)
        pts = np.zeros((nq, k, 4), dtype=np.float32)
        d2 = np.zeros((nq, k), dtype=np.float32)
        cnt = np.zeros(nq, dtype=np.int32)
        _check(self._L.fl_map_knn(self.h, q4, nq, k, pts, d2, cnt))
        return pts, d2, cnt

    # KD_TREE::Nearest_Search(point, k_nearest, .., max_dist), batched, 1 <= k <= 32
    def Nearest_Search_K(self, q4, k: int, max_dist: float = np.inf):
        """The min(k, #candidates) nearest points with float32 d2 <= fl(max_dist * max_dist), nearest first.  Returns
        (pts[nq, k, 4], d2[nq, k], cnt[nq]); entries past cnt[i] are zero with d2 = +inf."""
        q4 = np.ascontiguousarray(q4, dtype=np.float32).reshape(-1, 4)
        nq = len(q4)
        pts = np.zeros((nq, max(k, 0), 4), dtype=np.float32)
        d2 = np.zeros((nq, max(k, 0)), dtype=np.float32)
        cnt = np.zeros(nq, dtype=np.int32)
        _check(self._L.fl_map_nearest_search(self.h, q4, nq, k, max_dist, pts, d2, cnt))
        return pts, d2, cnt

    # KD_TREE::Add_Points
    def Add_Points(self, pts4, downsample_on: bool) -> int:
        pts4 = np.ascontiguousarray(pts4, dtype=np.float32).reshape(-1, 4)
        return _check(self._L.fl_map_add_points(self.h, pts4, len(pts4), int(downsample_on)))

    # KD_TREE::Delete_Point_Boxes
    def Delete_Point_Boxes(self, boxes6) -> int:
        boxes6 = np.ascontiguousarray(boxes6, dtype=np.float32).reshape(-1, 6)
        return _check(self._L.fl_map_delete_boxes(self.h, boxes6, len(boxes6)))

    # KD_TREE::Add_Point_Boxes
    def Add_Point_Boxes(self, boxes6) -> int:
        boxes6 = np.ascontiguousarray(boxes6, dtype=np.float32).reshape(-1, 6)
        return _check(self._L.fl_map_add_boxes(self.h, boxes6, len(boxes6)))

    # KD_TREE::acquire_removed_points
    def acquire_removed_points(self, cap: int = 1 << 20) -> np.ndarray:
        out = np.zeros((max(cap, 1), 4), dtype=np.float32)
        n = _check(self._L.fl_map_acquire_removed(self.h, out, cap))
        return out[:min(n, cap)].copy()

    # KD_TREE::flatten(Root_Node, ..., NOT_RECORD)
    def flatten(self) -> np.ndarray:
        n = self.validnum()
        out = np.zeros((max(n, 1), 4), dtype=np.float32)
        got = _check(self._L.fl_map_flatten(self.h, out, len(out)))
        return out[:got].copy()

    # KD_TREE::Box_Search, batched
    def Box_Search(self, boxes6, cap: int | None = None):
        """boxes6: (nb, 6) = (min xyz, max xyz); a point is found when min <= p < max on every axis.  Returns (offsets, points):
        the points of box i are points[offsets[i]:offsets[i + 1]], rows (x, y, z, intensity)."""
        boxes6 = np.ascontiguousarray(boxes6, dtype=np.float32).reshape(-1, 6)
        return self._range(self._L.fl_map_box_search, boxes6, cap)

    # KD_TREE::Radius_Search, batched
    def Radius_Search(self, centers_xyz, radius, cap: int | None = None):
        """centers_xyz: (nq, 3) (or (nq, 4): the fourth column is ignored); radius: a scalar or one per centre.  A point is found
        when its float32 squared distance is <= radius * radius rounded to float32.  Returns (offsets, points) like Box_Search."""
        c = np.asarray(centers_xyz, dtype=np.float32)
        c = c.reshape(-1, c.shape[-1])[:, :3]
        q = np.empty((len(c), 4), dtype=np.float32)
        q[:, :3] = c
        q[:, 3] = np.broadcast_to(np.asarray(radius, dtype=np.float32), (len(c),))
        return self._range(self._L.fl_map_radius_search, q, cap)

    def _range(self, fn, q, cap):
        """One call with room for `cap` points (default: the map size or the last total, whichever is larger); a second one
        when the total turns out to be larger."""
        offsets = np.zeros(len(q) + 1, dtype=np.int32)
        if cap is None:
            cap = max(self.validnum(), getattr(self, "_range_hint", 0), 1024)
        out = np.empty((max(cap, 1), 4), dtype=np.float32)
        total = _check(fn(self.h, q, len(q), offsets, out, cap))
        if total > cap:
            out = np.empty((total, 4), dtype=np.float32)
            total = _check(fn(self.h, q, len(q), offsets, out, total))
        self._range_hint = total
        return offsets, out[:total]

    # ---- device-buffer forms: CUDA tensors on the map's device, enqueued on torch.cuda.current_stream()
    def _tensor(self, t, name: str, cols: int | None, dtype=None, shape: tuple | None = None):
        """t checked to be a contiguous CUDA tensor on the map's device of `dtype` (default float32), shaped (n, cols) or
        exactly `shape`."""
        import torch
        dtype = torch.float32 if dtype is None else dtype
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name}: expected a torch.Tensor, got {type(t).__name__}")
        if t.device.type != "cuda" or t.device.index != self.device:
            raise ValueError(f"{name}: expected a tensor on cuda:{self.device}, got one on {t.device}")
        if t.dtype != dtype:
            raise TypeError(f"{name}: expected {str(dtype).replace('torch.', '')}, got {t.dtype}")
        if not t.is_contiguous():
            raise ValueError(f"{name}: expected a contiguous tensor")
        if cols is not None and (t.dim() != 2 or t.shape[1] != cols):
            raise ValueError(f"{name}: expected shape (n, {cols}), got {tuple(t.shape)}")
        if shape is not None and tuple(t.shape) != shape:
            raise ValueError(f"{name}: expected shape {shape}, got {tuple(t.shape)}")
        return t

    def _stream(self):
        import torch
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def nearest_search_device(self, q, k: int, max_dist: float = float("inf")):
        """fl_map_nearest_search on device tensors: q (nq, 4) float32.  Returns (pts [nq, k, 4], d2 [nq, k], cnt [nq] int32),
        the bytes Nearest_Search_K returns, written on the current stream without a host synchronisation."""
        import torch
        q = self._tensor(q, "q", 4)
        nq = q.shape[0]
        if not 1 <= k <= 32:
            raise ValueError(f"k must be in [1, 32], got {k}")
        pts = torch.empty((nq, k, 4), dtype=torch.float32, device=q.device)
        d2 = torch.empty((nq, k), dtype=torch.float32, device=q.device)
        cnt = torch.empty((nq,), dtype=torch.int32, device=q.device)
        _check(self._L.fl_map_nearest_search_device(self.h, q.data_ptr(), nq, k, max_dist, pts.data_ptr(), d2.data_ptr(),
                                                    cnt.data_ptr(), self._stream()))
        return pts, d2, cnt

    def range_workspace_bytes(self, nq: int, max_pairs: int) -> int:
        out = C.c_ulonglong(0)
        _check(self._L.fl_map_range_workspace_bytes(self.h, nq, max_pairs, C.byref(out)))
        return out.value

    def range_workspace(self, nq: int, max_pairs: int):
        """A uint8 CUDA tensor large enough for a range query of nq queries and up to max_pairs (query, leaf) pairs."""
        import torch
        return torch.empty(self.range_workspace_bytes(nq, max_pairs), dtype=torch.uint8, device=f"cuda:{self.device}")

    def box_search_device(self, boxes, cap: int | None = None, workspace=None):
        """fl_map_box_search_device: boxes (nb, 6) float32.  Returns (offsets [nb + 1] int32, pts, status [2] int64) as tensors.
        With both `cap` and `workspace` given, one call is enqueued and nothing synchronises: pts has `cap` rows, of which the
        first min(status[0], cap) are written when status[0] >= 0 (see the header).  Otherwise the status is read (a
        synchronisation) and the call is repeated once with enough room; pts then holds exactly the points found."""
        return self._range_device(self._L.fl_map_box_search_device, self._tensor(boxes, "boxes", 6), cap, workspace)

    def radius_search_device(self, centers_xyzr, cap: int | None = None, workspace=None):
        """fl_map_radius_search_device: centers_xyzr (nq, 4) float32 = (x, y, z, radius).  Returns like box_search_device."""
        return self._range_device(self._L.fl_map_radius_search_device, self._tensor(centers_xyzr, "centers_xyzr", 4), cap, workspace)

    def _range_device(self, fn, q, cap, workspace):
        import torch
        nq = q.shape[0]
        dev = q.device
        offsets = torch.empty(nq + 1, dtype=torch.int32, device=dev)
        status = torch.empty(2, dtype=torch.int64, device=dev)

        def call(cap_, ws):
            if ws is not None and (not isinstance(ws, torch.Tensor) or ws.device != dev or not ws.is_contiguous()):
                raise ValueError(f"workspace: expected a contiguous tensor on {dev}")
            pts = torch.empty((max(cap_, 0), 4), dtype=torch.float32, device=dev)
            _check(fn(self.h, q.data_ptr(), nq, offsets.data_ptr(), pts.data_ptr() if cap_ > 0 else None, cap_,
                      ws.data_ptr() if ws is not None and nq > 0 else None, ws.numel() * ws.element_size() if ws is not None else 0,
                      status.data_ptr(), self._stream()))
            return pts

        if cap is not None and workspace is not None:
            return offsets, call(cap, workspace), status
        if cap is None:
            cap = max(self.validnum(), getattr(self, "_range_hint", 0), 1024)
        if workspace is None:
            workspace = self.range_workspace(nq, max(getattr(self, "_pairs_hint", 0), 4 * nq, 1024)) if nq > 0 else None
        pts = call(cap, workspace)
        total, npairs = (int(x) for x in status.cpu())
        if total < 0:                                         # the pairs did not fit: a workspace sized from status[1]
            workspace = self.range_workspace(nq, npairs)
            pts = call(cap, workspace)
            total, npairs = (int(x) for x in status.cpu())
        if total > 2**31 - 1:
            raise FastLioError(f"{total} points found exceed INT_MAX; split the batch")
        if total > cap:
            pts = call(total, workspace)
        self._range_hint, self._pairs_hint = total, npairs
        return offsets, pts[:total], status

    def build_device(self, pts):
        """KD_TREE::Build from a (n, 4) float32 tensor on the map's device (synchronous)."""
        pts = self._tensor(pts, "pts", 4)
        _check(self._L.fl_map_build_device(self.h, pts.data_ptr() if len(pts) else None, len(pts), self._stream()))

    def add_points_device(self, pts, downsample_on: bool) -> int:
        """KD_TREE::Add_Points from a (n, 4) float32 tensor on the map's device (synchronous); the reference's return value."""
        pts = self._tensor(pts, "pts", 4)
        return _check(self._L.fl_map_add_points_device(self.h, pts.data_ptr() if len(pts) else None, len(pts), int(downsample_on),
                                                       self._stream()))

    def add_points_async(self, pts, n, n_max: int, downsample_on: bool, status=None):
        """fl_map_add_points_async: Add_Points of the first *n rows of pts ((>= n_max, 4) float32), n an int32 CUDA tensor of one
        element read when the current stream reaches the call.  Returns status, an int32 tensor (2,) = (FL_OK, 1 = maintenance
        due, or FL_ERR_CAPACITY = nothing changed; the reference's return value), written on the current stream."""
        import torch
        pts = self._tensor(pts, "pts", 4)
        if pts.shape[0] < n_max:
            raise ValueError(f"pts: {pts.shape[0]} rows, fewer than n_max = {n_max}")
        n = self._tensor(n, "n", None, torch.int32, (1,))
        if status is None:
            status = torch.empty(2, dtype=torch.int32, device=pts.device)
        status = self._tensor(status, "status", None, torch.int32, (2,))
        _check(self._L.fl_map_add_points_async(self.h, pts.data_ptr() if n_max > 0 else None, n.data_ptr(), n_max,
                                               int(downsample_on), status.data_ptr(), self._stream()))
        return status

    def delete_boxes_async(self, boxes, nb, nb_max: int, status=None):
        """fl_map_delete_boxes_async: Delete_Point_Boxes of the first *nb rows of boxes ((>= nb_max, 6) float32), nb an int32 CUDA
        tensor of one element read when the current stream reaches the call.  Returns status, an int32 tensor (2,) = (FL_OK, 1 =
        maintenance due, or FL_ERR_CAPACITY = nothing changed; the number of points deleted), written on the current stream."""
        import torch
        boxes = self._tensor(boxes, "boxes", 6)
        if boxes.shape[0] < nb_max:
            raise ValueError(f"boxes: {boxes.shape[0]} rows, fewer than nb_max = {nb_max}")
        nb = self._tensor(nb, "nb", None, torch.int32, (1,))
        if status is None:
            status = torch.empty(2, dtype=torch.int32, device=boxes.device)
        status = self._tensor(status, "status", None, torch.int32, (2,))
        _check(self._L.fl_map_delete_boxes_async(self.h, boxes.data_ptr() if nb_max > 0 else None, nb.data_ptr(), nb_max,
                                                 status.data_ptr(), self._stream()))
        return status

    def maintain(self) -> bool:
        """fl_map_maintain: settle the map and run the deferred re-pack / re-list; True when graphs must be captured again."""
        changed = C.c_int(0)
        _check(self._L.fl_map_maintain(self.h, C.byref(changed)))
        return bool(changed.value)

    def tree_range(self) -> np.ndarray:
        box = np.zeros(6, dtype=np.float32)
        _check(self._L.fl_map_tree_range(self.h, box))
        return box

    def rebuild(self):
        _check(self._L.fl_map_rebuild(self.h))

    def stats(self) -> dict:
        s = np.zeros(4, dtype=np.int32)
        _check(self._L.fl_map_stats(self.h, s))
        return dict(main_leaves=int(s[0]), overflow_leaves=int(s[1]), levels=int(s[2]), rebuilds=int(s[3]))

    def dir_stats(self) -> dict:
        s = np.zeros(6, dtype=np.int32)
        _check(self._L.fl_map_dir_stats(self.h, s))
        return dict(cells=int(s[0]), ext_buckets=int(s[1]), crowded_cells=int(s[2]), capacity=int(s[3]), relists=int(s[4]), walked=int(s[5]), enabled=bool(s[5] >= 0))


class Esekf:
    """esekf::update_iterated_dyn_share_modified with the fused device measurement model."""

    def __init__(self, tree: KdTree, max_points: int = 100000, max_iter: int = 4, limit: float = 0.001,
                 extrinsic_est_en: bool = False, solver: int = 1, search: int = -1, fused: int = -1):
        self._L = load()
        self.tree = tree
        h = C.c_void_p()
        _check(self._L.fl_filter_create(C.byref(h), tree.h, max_points))
        self.h = h
        self.max_iter = max_iter
        lim = np.full(23, limit, dtype=np.float64)
        _check(self._L.fl_filter_set_params(self.h, max_iter, lim, int(extrinsic_est_en)))
        _check(self._L.fl_filter_set_solver(self.h, solver))
        if search >= 0:
            _check(self._L.fl_filter_set_search(self.h, search))
        if fused >= 0:
            _check(self._L.fl_filter_set_fused(self.h, fused))
        self._fused = (fused != 0) and solver == 1 and os.environ.get('FASTLIO_B200_LEGACY', '0') != '1'

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_filter_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def update_iterated_dyn_share_modified(self, scan4, x26, P, R: float = 0.001):
        """Returns (x, P, solve_time_s).  Host buffers in, host buffers out."""
        scan4 = np.ascontiguousarray(scan4, dtype=np.float32).reshape(-1, 4)
        x = np.array(x26, dtype=np.float64).copy()
        Pm = np.ascontiguousarray(np.array(P, dtype=np.float64).copy())
        st = C.c_double(0.0)
        _check(self._L.fl_filter_update(self.h, scan4, len(scan4), x, Pm, R, C.byref(st)))
        return x, Pm, st.value

    def map_incremental(self, filter_size_map_min: float = 0.5, flg_EKF_inited: bool = True):
        """laserMapping.cpp:427-474 on the device; returns (|PointToAdd|, |PointNoNeedDownsample|, Add_Points return)."""
        out = np.zeros(3, dtype=np.int32)
        _check(self._L.fl_filter_map_incremental(self.h, filter_size_map_min, int(flg_EKF_inited), out))
        return int(out[0]), int(out[1]), int(out[2])

    def nearest(self, nq: int):
        pts = np.zeros((nq, 5, 4), dtype=np.float32)
        cnt = np.zeros(nq, dtype=np.int32)
        _check(self._L.fl_filter_get_nearest(self.h, pts, cnt, nq))
        return pts, cnt

    def selected(self, nq: int):
        out = np.zeros(nq, dtype=np.uint8)
        _check(self._L.fl_filter_get_selected(self.h, out, nq))
        return out

    def pass_logs(self):
        logs = (PassLog * 16)()
        n = _check(self._L.fl_filter_get_pass_logs(self.h, logs, 16))
        return [_log_dict(logs[i]) for i in range(n)]

    # ---- device-buffer form: CUDA tensors on the map's device, enqueued on torch.cuda.current_stream()
    def update_device(self, scan, x, P, R: float = 0.001, status=None):
        """fl_filter_update_device: scan (nq, 4) float32, x (26,) float64, P (23, 23) float64.  x and P are updated in place
        (only when the update succeeds); returns status, an int32 tensor of shape (2,) = (FL_OK or FL_ERR_STATE, passes run),
        written on the current stream.  Nothing synchronises, so the call can be captured into a CUDA graph."""
        import torch
        t = self.tree
        scan = t._tensor(scan, "scan", 4)
        x = t._tensor(x, "x", None, torch.float64, (26,))
        P = t._tensor(P, "P", None, torch.float64, (23, 23))
        if status is None:
            status = torch.empty(2, dtype=torch.int32, device=x.device)
        status = t._tensor(status, "status", None, torch.int32, (2,))
        nq = scan.shape[0]
        _check(self._L.fl_filter_update_device(self.h, scan.data_ptr() if nq else None, nq, x.data_ptr(), P.data_ptr(), R,
                                               status.data_ptr(), t._stream()))
        return status

    # ---- batched form: one scan from many priors (fl_filter_update_batch_device)
    def reserve_batch(self, nq_max: int):
        """fl_filter_reserve_batch: size the batch's own buffers for scans of up to nq_max points (synchronous, grow-only)."""
        _check(self._L.fl_filter_reserve_batch(self.h, int(nq_max)))

    def batch_plan(self, nq: int, n_hyp: int):
        """(workers per hypothesis, hypotheses per wave, waves) of a batch of n_hyp priors on an nq-point scan."""
        out = np.zeros(3, dtype=np.int32)
        _check(self._L.fl_filter_batch_plan(self.h, int(nq), int(n_hyp), out))
        return int(out[0]), int(out[1]), int(out[2])

    def update_batch_device(self, scan, x, P, R: float = 0.001, status=None, logs: bool = False):
        """fl_filter_update_batch_device on the current stream: scan (nq, 4) float32, x (H, 26) and P (H, 23, 23) float64, updated
        in place per hypothesis (only where it succeeds).  Returns status, an (H, 2) int32 tensor of (FL_OK or FL_ERR_STATE,
        passes run); with logs=True also the pass logs as an (H, max_iter + 1, sizeof(fl_pass_log_t)) uint8 tensor (entries from
        `passes` on stay zero; decode_pass_logs reads them).  Nothing synchronises, so the call can be captured into a CUDA graph."""
        import torch
        t = self.tree
        scan = t._tensor(scan, "scan", 4)
        x = t._tensor(x, "x", 26, torch.float64)
        H = x.shape[0]
        P = t._tensor(P, "P", None, torch.float64, (H, 23, 23))
        if status is None:
            status = torch.empty((H, 2), dtype=torch.int32, device=x.device)
        status = t._tensor(status, "status", None, torch.int32, (H, 2))
        lg = torch.zeros((H, self.max_iter + 1, C.sizeof(PassLog)), dtype=torch.uint8, device=x.device) if logs else None
        nq = scan.shape[0]
        _check(self._L.fl_filter_update_batch_device(self.h, scan.data_ptr() if nq else None, nq, H, x.data_ptr() if H else None,
                                                     P.data_ptr() if H else None, R, status.data_ptr() if H else None,
                                                     lg.data_ptr() if (logs and H) else None, t._stream()))
        return (status, lg) if logs else status

    # ---- batched form over many scans: a scan and a prior per slot, one shared map (fl_filter_update_scans_device)
    def update_scans_device(self, refs, x, P, nq_max: int, R: float = 0.001, status=None, logs: bool = False):
        """fl_filter_update_scans_device on the current stream: refs the (S, 2) int64 table of scan_refs, x (S, 26) and P (S, 23,
        23) float64, updated in place per slot (only where it succeeds).  Slot s runs rows [0, *n) of its scan, read on the device;
        counts above nq_max are refused.  Returns status, an (S, 2) int32 tensor of (FL_OK, FL_ERR_STATE, or FL_ERR_ARG /
        FL_ERR_CAPACITY for a refused slot, passes run); with logs=True also the pass logs as an (S, max_iter + 1,
        sizeof(fl_pass_log_t)) uint8 tensor (decode_pass_logs reads them).  Nothing synchronises, so the call can be captured into
        a CUDA graph."""
        import torch
        t = self.tree
        x = t._tensor(x, "x", 26, torch.float64)
        S = x.shape[0]
        refs = t._tensor(refs, "refs", None, torch.int64, (S, 2))
        P = t._tensor(P, "P", None, torch.float64, (S, 23, 23))
        if status is None:
            status = torch.empty((S, 2), dtype=torch.int32, device=x.device)
        status = t._tensor(status, "status", None, torch.int32, (S, 2))
        lg = torch.zeros((S, self.max_iter + 1, C.sizeof(PassLog)), dtype=torch.uint8, device=x.device) if logs else None
        _check(self._L.fl_filter_update_scans_device(self.h, refs.data_ptr() if S else None, S, int(nq_max),
                                                     x.data_ptr() if S else None, P.data_ptr() if S else None, R,
                                                     status.data_ptr() if S else None, lg.data_ptr() if (logs and S) else None,
                                                     t._stream()))
        return (status, lg) if logs else status

    # ---- relocalisation: screen many hypotheses by inliers, update from the best, choose one (fl_filter_relocalize_device)
    def reserve_reloc(self, nq_max: int, n_hyp_max: int, keep_max: int):
        """fl_filter_reserve_reloc: size the relocalisation's buffers (and the batch's, for nq_max points); synchronous, grow-only."""
        _check(self._L.fl_filter_reserve_reloc(self.h, int(nq_max), int(n_hyp_max), int(keep_max)))

    def relocalize_device(self, scan, x_hyp, P, keep: int, r_inlier: float, min_effct: int, stride: int = 1, R: float = 0.001,
                          x_out=None, P_out=None):
        """fl_filter_relocalize_device on the current stream: scan (nq, 4) float32, x_hyp (H, 26) and P (23, 23) float64.  Returns
        (x, P, status4, rows, inliers): the winner's updated state and covariance (x_out / P_out when given, left as they were when
        no survivor qualifies), status4 int32 (4,) = (FL_OK or FL_ERR_STATE, h or -1, effct, inliers), rows a (min(keep, H),
        sizeof(fl_reloc_row_t)) uint8 tensor (decode_reloc_rows reads it) and inliers int32 (H,).  Nothing synchronises, so the call
        can be captured into a CUDA graph."""
        import torch
        t = self.tree
        scan = t._tensor(scan, "scan", 4)
        x_hyp = t._tensor(x_hyp, "x_hyp", 26, torch.float64)
        P = t._tensor(P, "P", None, torch.float64, (23, 23))
        H, dev_ = x_hyp.shape[0], x_hyp.device
        if x_out is None:
            x_out = torch.zeros(26, dtype=torch.float64, device=dev_)
        if P_out is None:
            P_out = torch.zeros((23, 23), dtype=torch.float64, device=dev_)
        x_out = t._tensor(x_out, "x_out", None, torch.float64, (26,))
        P_out = t._tensor(P_out, "P_out", None, torch.float64, (23, 23))
        status4 = torch.empty(4, dtype=torch.int32, device=dev_)
        inliers = torch.empty(max(H, 1), dtype=torch.int32, device=dev_)[:H]
        rows = torch.empty((max(min(int(keep), H), 1), C.sizeof(RelocRow)), dtype=torch.uint8, device=dev_)[:max(min(int(keep), H), 0)]
        prm = RelocParams(int(keep), int(stride), float(r_inlier), int(min_effct))
        nq = scan.shape[0]
        _check(self._L.fl_filter_relocalize_device(self.h, scan.data_ptr() if nq else None, nq, H, x_hyp.data_ptr() if H else None,
                                                   P.data_ptr(), R, C.byref(prm), x_out.data_ptr(), P_out.data_ptr(),
                                                   inliers.data_ptr() if H else None, rows.data_ptr() if rows.numel() else None,
                                                   status4.data_ptr(), t._stream()))
        return x_out, P_out, status4, rows, inliers

    def map_incremental_device(self, filter_size_map_min: float = 0.5, flg_EKF_inited: bool = True, out4=None):
        """fl_filter_map_incremental_device on the current stream.  Returns out4, an int32 tensor (4,) = (|PointToAdd|,
        |PointNoNeedDownsample|, Add_Points return, status), written without a host synchronisation (capturable)."""
        import torch
        t = self.tree
        if out4 is None:
            out4 = torch.empty(4, dtype=torch.int32, device=f"cuda:{t.device}")
        out4 = t._tensor(out4, "out4", None, torch.int32, (4,))
        _check(self._L.fl_filter_map_incremental_device(self.h, filter_size_map_min, int(flg_EKF_inited), out4.data_ptr(), t._stream()))
        return out4

    def nearest_device(self, nq: int):
        """Nearest_Points of the last update as tensors (pts [nq, 5, 4] float32, cnt [nq] int32), copied on the current stream."""
        import torch
        dev = f"cuda:{self.tree.device}"
        pts = torch.empty((nq, 5, 4), dtype=torch.float32, device=dev)
        cnt = torch.empty((nq,), dtype=torch.int32, device=dev)
        _check(self._L.fl_filter_get_nearest_device(self.h, pts.data_ptr() if nq else None, cnt.data_ptr() if nq else None, nq,
                                                    self.tree._stream()))
        return pts, cnt

    def selected_device(self, nq: int):
        """point_selected_surf of the last update as a uint8 tensor [nq], copied on the current stream."""
        import torch
        out = torch.empty((nq,), dtype=torch.uint8, device=f"cuda:{self.tree.device}")
        _check(self._L.fl_filter_get_selected_device(self.h, out.data_ptr() if nq else None, nq, self.tree._stream()))
        return out

    # device-resident pieces
    def upload_scan(self, scan4):
        scan4 = np.ascontiguousarray(scan4, dtype=np.float32).reshape(-1, 4)
        _check(self._L.fl_filter_upload_scan(self.h, scan4, len(scan4)))

    def upload_state(self, x26, P, R: float = 0.001):
        _check(self._L.fl_filter_upload_state(self.h, np.ascontiguousarray(x26, dtype=np.float64),
                                              np.ascontiguousarray(P, dtype=np.float64), R))

    def run(self):
        _check(self._L.fl_filter_run(self.h))

    def download_state(self):
        x = np.zeros(26, dtype=np.float64)
        P = np.zeros((23, 23), dtype=np.float64)
        n = C.c_int(0)
        _check(self._L.fl_filter_download_state(self.h, x, P, C.byref(n)))
        return x, P, n.value

    def time_resident(self, reps: int, flush_l2: bool = True) -> float:
        ms = C.c_float(0.0)
        _check(self._L.fl_filter_time_resident(self.h, reps, int(flush_l2), C.byref(ms)))
        return ms.value

    def time_search_pass(self, reps: int, flush_l2: bool = True) -> float:
        ms = C.c_float(0.0)
        _check(self._L.fl_filter_time_search_pass(self.h, reps, int(flush_l2), C.byref(ms)))
        return ms.value

    def time_e2e(self, scan4, x26, P, R: float, reps: int):
        """Seconds for `reps` native back-to-back fl_filter_update calls with host buffers; returns (seconds, x, P)."""
        scan4 = np.ascontiguousarray(scan4, dtype=np.float32).reshape(-1, 4)
        x_out = np.zeros(26, dtype=np.float64)
        P_out = np.zeros((23, 23), dtype=np.float64)
        sec = C.c_double(0.0)
        _check(self._L.fl_filter_time_e2e(self.h, scan4, len(scan4), np.ascontiguousarray(x26, dtype=np.float64),
                                          np.ascontiguousarray(P, dtype=np.float64), R, reps, C.byref(sec), x_out, P_out))
        return sec.value, x_out, P_out

    def gpu_launches(self) -> int:
        return _check(self._L.fl_filter_gpu_launches(self.h))

    def fused(self) -> bool:
        return self._fused

    def comm_init(self, nranks: int, rank: int, unique_id: bytes):
        _check(self._L.fl_filter_comm_init(self.h, nranks, rank, unique_id))

    def p2p_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        _check(self._L.fl_filter_p2p_handle(self.h, buf))
        return buf.raw

    def p2p_connect(self, nranks: int, rank: int, handles: bytes):
        _check(self._L.fl_filter_p2p_connect(self.h, nranks, rank, handles))

    def set_shard(self, q_begin: int, q_end: int):
        _check(self._L.fl_filter_set_shard(self.h, q_begin, q_end))


class Scan:
    """feats_undistort / feats_down_body kept in HBM: UndistortPcl's backward pass (IMU_Processing.hpp:232-346) and the
    pcl::VoxelGrid down-sampling (laserMapping.cpp:904-905) in front of the update."""

    def __init__(self, tree: KdTree):
        self._L = load()
        self.tree = tree
        h = C.c_void_p()
        _check(self._L.fl_scan_create(C.byref(h), tree.h))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_scan_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, xyzi, offset_ms):
        xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
        offset_ms = np.ascontiguousarray(offset_ms, dtype=np.float32).reshape(-1)
        if len(offset_ms) != len(xyzi):
            raise ValueError("one offset time per point")
        _check(self._L.fl_scan_upload(self.h, xyzi, offset_ms, len(xyzi)))
        self.n = len(xyzi)

    def undistort(self, imu_pose22, x26_end):
        poses = np.ascontiguousarray(imu_pose22, dtype=np.float64).reshape(-1, 22)
        _check(self._L.fl_scan_undistort(self.h, poses, len(poses), np.ascontiguousarray(x26_end, dtype=np.float64)))

    def voxel_downsample(self, leaf: float) -> int:
        return _check(self._L.fl_scan_voxel_downsample(self.h, leaf))

    def download(self, which: int = 1) -> np.ndarray:
        n = _check(self._L.fl_scan_download(self.h, which, np.zeros((1, 4), dtype=np.float32), 0))
        out = np.zeros((max(n, 1), 4), dtype=np.float32)
        _check(self._L.fl_scan_download(self.h, which, out, n))
        return out[:n].copy()

    def update(self, filt: "Esekf", x26, P, R: float = 0.001):
        """fl_filter_update on the down-sampled cloud without a host hop; returns (x, P, solve_time_s)."""
        x = np.array(x26, dtype=np.float64).copy()
        Pm = np.ascontiguousarray(np.array(P, dtype=np.float64).copy())
        st = C.c_double(0.0)
        _check(self._L.fl_filter_update_scan(filt.h, self.h, x, Pm, R, C.byref(st)))
        return x, Pm, st.value

    # ---- device-buffer forms: CUDA tensors on the map's device, enqueued on torch.cuda.current_stream(), counts in device memory
    def reserve(self, n_max: int, n_pose_max: int):
        """fl_scan_reserve: size the device forms' buffers for up to n_max points and n_pose_max IMU poses (synchronous)."""
        _check(self._L.fl_scan_reserve(self.h, n_max, n_pose_max))

    def _count(self, n, default: int, name: str):
        import torch
        t = self.tree
        if n is None:
            # building the count is a host-to-device copy, which a capturing stream cannot take
            if torch.cuda.is_current_stream_capturing():
                raise ValueError(f"{name}: pass an int32 CUDA tensor while capturing a CUDA graph")
            return torch.tensor([default], dtype=torch.int32, device=f"cuda:{t.device}")
        return t._tensor(n, name, None, torch.int32, (1,))

    def upload_device(self, xyzi, offset_ms, n=None, n_max: int | None = None):
        """fl_scan_upload_device: the first *n rows of xyzi ((>= n_max, 4) float32) and offset_ms ((>= n_max,) float32).  n is an
        int32 CUDA tensor of one element (None: the tensor's length, which is copied from the host, so pass a tensor when capturing
        a CUDA graph); n_max defaults to the number of rows."""
        import torch
        t = self.tree
        xyzi = t._tensor(xyzi, "xyzi", 4)
        offset_ms = t._tensor(offset_ms, "offset_ms", None, torch.float32, (xyzi.shape[0],))
        n_max = xyzi.shape[0] if n_max is None else n_max
        if xyzi.shape[0] < n_max:
            raise ValueError(f"xyzi: {xyzi.shape[0]} rows, fewer than n_max = {n_max}")
        self._n = self._count(n, xyzi.shape[0], "n")           # kept alive until the stream has read it
        _check(self._L.fl_scan_upload_device(self.h, xyzi.data_ptr() if n_max else None, offset_ms.data_ptr() if n_max else None,
                                             self._n.data_ptr(), n_max, t._stream()))

    def undistort_device(self, poses, n_pose, x_end):
        """fl_scan_undistort_device: poses (n_pose_max, 22) float64, n_pose an int32 CUDA tensor (1,) (None: all rows, copied
        from the host, so pass a tensor when capturing), x_end (26,) float64; all read when the current stream reaches the call."""
        import torch
        t = self.tree
        poses = t._tensor(poses, "poses", 22, torch.float64)
        x_end = t._tensor(x_end, "x_end", None, torch.float64, (26,))
        self._n_pose = self._count(n_pose, poses.shape[0], "n_pose")
        _check(self._L.fl_scan_undistort_device(self.h, poses.data_ptr() if poses.shape[0] else None, self._n_pose.data_ptr(),
                                                poses.shape[0], x_end.data_ptr(), t._stream()))

    def voxel_downsample_device(self, leaf: float, out=None):
        """fl_scan_voxel_downsample_device; returns out, an int32 tensor (1,) that receives feats_down_size on the current stream."""
        import torch
        t = self.tree
        if out is None:
            out = torch.empty(1, dtype=torch.int32, device=f"cuda:{t.device}")
        out = t._tensor(out, "out", None, torch.int32, (1,))
        _check(self._L.fl_scan_voxel_downsample_device(self.h, leaf, out.data_ptr(), t._stream()))
        return out

    def ref(self):
        """fl_scan_get_ref: (body_ptr, n_ptr, n_max), the device forms' feats_down_body, the device address of feats_down_size and
        the rows fl_scan_reserve sized; valid until a reserve that grows the scan."""
        r = ScanRef()
        m = C.c_int(0)
        _check(self._L.fl_scan_get_ref(self.h, C.byref(r), C.byref(m)))
        return int(r.body_xyzi or 0), int(r.n or 0), int(m.value)

    def update_device(self, filt: "Esekf", x, P, R: float = 0.001, status=None):
        """fl_filter_update_scan_device: x (26,) and P (23, 23) float64 tensors updated in place on success; returns status, an
        int32 tensor (2,) = (FL_OK or FL_ERR_STATE, passes run), written on the current stream."""
        import torch
        t = self.tree
        x = t._tensor(x, "x", None, torch.float64, (26,))
        P = t._tensor(P, "P", None, torch.float64, (23, 23))
        if status is None:
            status = torch.empty(2, dtype=torch.int32, device=x.device)
        status = t._tensor(status, "status", None, torch.int32, (2,))
        _check(self._L.fl_filter_update_scan_device(filt.h, self.h, x.data_ptr(), P.data_ptr(), R, status.data_ptr(), t._stream()))
        return status

    def frame(self, which: int, frame: int, x26=None) -> np.ndarray:
        """fl_scan_frame: the cloud `which` (0 feats_undistort, 1 feats_down_body) in FRAME_LIDAR / FRAME_IMU / FRAME_WORLD with
        the state x26 (26 float64; unused, may be None, for FRAME_LIDAR), as an (n, 4) float32 array."""
        x = None if x26 is None else np.ascontiguousarray(x26, dtype=np.float64).reshape(26)
        xp = None if x is None else x.ctypes.data
        n = _check(self._L.fl_scan_frame(self.h, which, frame, xp, np.zeros((1, 4), dtype=np.float32), 0))
        out = np.zeros((max(n, 1), 4), dtype=np.float32)
        _check(self._L.fl_scan_frame(self.h, which, frame, xp, out, n))
        return out[:n].copy()

    def frame_device(self, which: int, frame: int, x, out, n_io=None, status=None):
        """fl_scan_frame_device: the device forms' cloud `which` in `frame` with the state x ((26,) float64 tensor; None for
        FRAME_LIDAR) appended to out ((cap, 4) float32) at *n_io (int32 (1,); None: a zeroed position, copied from the host, so
        pass a tensor when capturing), which advances by n when the cloud fits.  Returns status, an int32 tensor (2,) = (FL_OK,
        FL_ERR_CAPACITY or FL_ERR_ARG, n), written on the current stream."""
        import torch
        t = self.tree
        out = t._tensor(out, "out", 4)
        if x is not None:
            x = t._tensor(x, "x", None, torch.float64, (26,))
        self._n_io = self._count(n_io, 0, "n_io")               # kept alive until the stream has read it
        if status is None:
            status = torch.empty(2, dtype=torch.int32, device=out.device)
        status = t._tensor(status, "status", None, torch.int32, (2,))
        _check(self._L.fl_scan_frame_device(self.h, which, frame, None if x is None else x.data_ptr(), out.data_ptr(),
                                            self._n_io.data_ptr(), out.shape[0], status.data_ptr(), t._stream()))
        return status


class _DeviceTable:
    """A view of device memory the batch owns, for torch.as_tensor (the __cuda_array_interface__ protocol); holds the batch.
    Default: `rows` fl_scan_ref_t entries as (rows, 2) int64."""

    def __init__(self, owner, ptr: int, rows: int, shape: tuple | None = None, typestr: str = "<i8"):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": (rows, 2) if shape is None else shape, "typestr": typestr, "data": (ptr, False),
                                         "version": 2}


class ScanBatch:
    """The scan front end of many scans in one call (fl_scan_batch_run_device): per slot UndistortPcl's sort and backward pass
    (IMU_Processing.hpp:232-346) and the pcl::VoxelGrid down-sampling (laserMapping.cpp:904-905), each slot equal to a `Scan`'s
    device forms on the same inputs, into the table Esekf.update_scans_device reads."""

    def __init__(self, tree: KdTree):
        self._L = load()
        self.tree = tree
        h = C.c_void_p()
        _check(self._L.fl_scan_batch_create(C.byref(h), tree.h))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_scan_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reserve(self, n_scans_max: int, n_max: int, n_pose_max: int):
        """fl_scan_batch_reserve: buffers for up to n_scans_max slots of n_max rows and n_pose_max IMU poses (synchronous, grow-only;
        a grow moves the buffers and the ref tables, so capture graphs again after one)."""
        _check(self._L.fl_scan_batch_reserve(self.h, n_scans_max, n_max, n_pose_max))
        self._slots_max = max(getattr(self, "_slots_max", 1), n_scans_max)

    def run_device(self, raws, n_max: int, n_pose_max: int, leaf: float, undistort: bool = True, status=None):
        """fl_scan_batch_run_device on the current stream: raws the (S, 6) int64 table of scan_raws.  Returns status, an (S, 2)
        int32 tensor = (FL_OK, feats_down_size) or (refusal, 0) per slot, written on the current stream."""
        import torch
        t = self.tree
        if not isinstance(raws, torch.Tensor) or raws.dtype != torch.int64 or raws.dim() != 2 or raws.shape[1] != 6:
            raise TypeError("raws must be the (S, 6) int64 tensor of scan_raws")
        S = raws.shape[0]
        if S:
            raws = t._tensor(raws, "raws", 6, torch.int64)
        if status is None:
            status = torch.empty((S, 2), dtype=torch.int32, device=f"cuda:{t.device}")
        if S:
            status = t._tensor(status, "status", None, torch.int32, (S, 2))
        _check(self._L.fl_scan_batch_run_device(self.h, raws.data_ptr() if S else None, S, n_max, n_pose_max, 1 if undistort else 0,
                                                leaf, status.data_ptr() if S else None, t._stream()))
        return status

    def refs(self, which: int = 1):
        """fl_scan_batch_get_refs: the device table of n_scans_max fl_scan_ref_t entries (feats_undistort for which 0,
        feats_down_body for 1) as an (n_scans_max, 2) int64 CUDA tensor over the batch's own memory, for Esekf.update_scans_device
        (slice the first S rows), and the reserved n_max, its nq_max."""
        import torch
        p, m = C.c_void_p(), C.c_int(0)
        _check(self._L.fl_scan_batch_get_refs(self.h, which, C.byref(p), C.byref(m)))
        return torch.as_tensor(_DeviceTable(self, int(p.value), self._slots_max), device=f"cuda:{self.tree.device}"), int(m.value)

    def download(self, which: int, slot: int) -> np.ndarray:
        """fl_scan_batch_download: slot `slot`'s rows of the last call (which 0 feats_undistort, 1 feats_down_body) as an (n, 4)
        float32 array; a refused slot has none."""
        n = _check(self._L.fl_scan_batch_download(self.h, which, slot, np.zeros((1, 4), dtype=np.float32), 0))
        out = np.zeros((max(n, 1), 4), dtype=np.float32)
        _check(self._L.fl_scan_batch_download(self.h, which, slot, out, n))
        return out[:n].copy()


class LocalMap:
    """lasermap_fov_segment() (laserMapping.cpp:229-277): the sliding cube that issues the delete boxes."""

    def __init__(self, cube_len: float, det_range: float):
        self._L = load()
        h = C.c_void_p()
        _check(self._L.fl_localmap_create(C.byref(h), cube_len, det_range))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_localmap_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def segment(self, pos_lid, tree: "KdTree | None" = None):
        """Returns (cub_needrm as an (nb, 6) array, kdtree_delete_counter)."""
        boxes = np.zeros((3, 6), dtype=np.float32)
        nd = C.c_int(0)
        nb = _check(self._L.fl_localmap_segment(self.h, tree.h if tree is not None else None,
                                                np.ascontiguousarray(pos_lid, dtype=np.float64), boxes, C.byref(nd)))
        return boxes[:nb].copy(), nd.value

    def segment_device(self, tree: "KdTree", x, out3=None, boxes=None, n_scan=None):
        """fl_localmap_segment_device on the current stream: pos_lid from x ((26,) float64 CUDA tensor), the cube slid on the map's
        device and Delete_Point_Boxes of cub_needrm on `tree`, all-or-nothing.  Returns out3, an int32 tensor (3,) = (|cub_needrm|,
        kdtree_delete_counter, status); boxes ((3, 6) float32, optional) receives cub_needrm; n_scan (int32 (1,), optional): a 0
        there skips the call's work, as the reference skips an empty scan."""
        import torch
        x = tree._tensor(x, "x", None, torch.float64, (26,))
        if out3 is None:
            out3 = torch.empty(3, dtype=torch.int32, device=x.device)
        out3 = tree._tensor(out3, "out3", None, torch.int32, (3,))
        if boxes is not None:
            boxes = tree._tensor(boxes, "boxes", None, torch.float32, (3, 6))
        if n_scan is not None:
            n_scan = tree._tensor(n_scan, "n_scan", None, torch.int32, (1,))
        _check(self._L.fl_localmap_segment_device(self.h, tree.h, x.data_ptr(), n_scan.data_ptr() if n_scan is not None else None,
                                                  boxes.data_ptr() if boxes is not None else None, out3.data_ptr(), tree._stream()))
        return out3

    def box(self) -> np.ndarray:
        b = np.zeros(6, dtype=np.float32)
        _check(self._L.fl_localmap_get(self.h, b))
        return b


class Preprocess:
    """Preprocess::process (src/preprocess.cpp) with feature extraction off, on the device: one raw LiDAR frame -> pl_surf, the
    (xyzi, offset time in ms) rows fl_scan_upload[_device] take.  layout: the raw points' structured numpy dtype (default: the
    reference's struct for lidar_type, DEFAULT_LAYOUT); its itemsize is point_step and its fields give the offsets."""

    def __init__(self, device: int, lidar_type: int, n_scans: int, scan_rate: int = 10, time_unit: int = TIME_US,
                 point_filter_num: int = 1, blind: float = 0.01, layout: np.dtype | None = None, n_raw_max: int = 65536):
        self._L = load()
        self.device = device
        self.layout = np.dtype(DEFAULT_LAYOUT[lidar_type] if layout is None else layout)
        self.n_raw_max = n_raw_max
        off = layout_offsets(self.layout, lidar_type)
        p = PreprocessParams(lidar_type, n_scans, scan_rate, time_unit, point_filter_num, blind, self.layout.itemsize, *off)
        h = C.c_void_p()
        _check(self._L.fl_preprocess_create(C.byref(h), device, C.byref(p), n_raw_max))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_preprocess_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _raw_bytes(self, raw) -> np.ndarray:
        raw = np.ascontiguousarray(raw)
        if raw.dtype.fields is not None:
            if raw.dtype.itemsize != self.layout.itemsize:
                raise ValueError(f"raw: {raw.dtype.itemsize}-byte points, the layout has {self.layout.itemsize}")
            return raw.reshape(-1).view(np.uint8)
        return np.ascontiguousarray(raw, dtype=np.uint8).reshape(-1)

    def process(self, raw):
        """The host form (fl_preprocess): raw, a structured array of the layout (or its bytes).  Returns (xyzi (m, 4) float32,
        offset_ms (m,) float32, last_ms), last_ms = pl_surf.points.back().curvature (0.0 when nothing is kept)."""
        buf = self._raw_bytes(raw)
        n = len(buf) // self.layout.itemsize
        xyzi = np.empty((max(n, 1), 4), dtype=np.float32)
        ms = np.empty(max(n, 1), dtype=np.float32)
        last = C.c_float(0.0)
        m = _check(self._L.fl_preprocess(self.h, buf.ctypes.data if n else None, n, xyzi, ms, n, C.byref(last)))
        return xyzi[:m].copy(), ms[:m].copy(), last.value

    def process_device(self, raw, n=None, n_max: int | None = None, xyzi=None, offset_ms=None, out2=None, last_ms=None):
        """fl_preprocess_device on torch.cuda.current_stream(): raw a uint8 CUDA tensor (>= n_max * point_step bytes; (rows,
        point_step) or flat), n an int32 CUDA tensor (1,) (None: all rows, copied from the host, so pass a tensor when capturing a
        CUDA graph), n_max defaults to the number of rows.  The outputs (allocated when not given, n_max rows): xyzi (n_max, 4)
        float32, offset_ms (n_max,) float32, out2 int32 (2,) = (kept, dropped rings), last_ms float32 (1,).  Returns them."""
        import torch
        dev = f"cuda:{self.device}"
        step = self.layout.itemsize
        if not isinstance(raw, torch.Tensor) or raw.dtype != torch.uint8 or not raw.is_contiguous() or raw.device != torch.device(dev):
            raise TypeError(f"raw: expected a contiguous uint8 tensor on {dev}")
        rows = raw.numel() // step
        n_max = rows if n_max is None else n_max
        if rows < n_max:
            raise ValueError(f"raw: {rows} rows, fewer than n_max = {n_max}")
        if n is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("n: pass an int32 CUDA tensor while capturing a CUDA graph")
            n = torch.tensor([rows], dtype=torch.int32, device=dev)
        xyzi = torch.empty((n_max, 4), dtype=torch.float32, device=dev) if xyzi is None else xyzi
        offset_ms = torch.empty(n_max, dtype=torch.float32, device=dev) if offset_ms is None else offset_ms
        out2 = torch.empty(2, dtype=torch.int32, device=dev) if out2 is None else out2
        last_ms = torch.empty(1, dtype=torch.float32, device=dev) if last_ms is None else last_ms
        for name, t, dt in (("n", n, torch.int32), ("xyzi", xyzi, torch.float32), ("offset_ms", offset_ms, torch.float32),
                            ("out2", out2, torch.int32), ("last_ms", last_ms, torch.float32)):
            if not isinstance(t, torch.Tensor) or t.dtype != dt or not t.is_contiguous() or t.device != torch.device(dev):
                raise TypeError(f"{name}: expected a contiguous {dt} tensor on {dev}")
        if xyzi.numel() < 4 * n_max or offset_ms.numel() < n_max or out2.numel() < 2 or n.numel() < 1 or last_ms.numel() < 1:
            raise ValueError("an output tensor is smaller than n_max rows")
        self._n = n                                    # kept alive until the stream has read it
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        _check(self._L.fl_preprocess_device(self.h, raw.data_ptr() if n_max else None, n.data_ptr(), n_max,
                                            xyzi.data_ptr() if n_max else None, offset_ms.data_ptr() if n_max else None,
                                            out2.data_ptr(), last_ms.data_ptr(), stream))
        return xyzi, offset_ms, out2, last_ms


class PreprocessBatch:
    """Preprocess::process of many raw frames in one call (fl_preprocess_batch_run_device): every slot a frame of one LiDAR type and
    layout (the arguments of `Preprocess`), each slot's pl_surf equal to Preprocess.process_device's on the same frame.  The
    outputs live in the handle, n_slots_max slots of n_raw_max rows at addresses fixed at creation (outputs())."""

    def __init__(self, device: int, lidar_type: int, n_scans: int, scan_rate: int = 10, time_unit: int = TIME_US,
                 point_filter_num: int = 1, blind: float = 0.01, layout: np.dtype | None = None, n_slots_max: int = 1,
                 n_raw_max: int = 65536):
        self._L = load()
        self.device = device
        self.layout = np.dtype(DEFAULT_LAYOUT[lidar_type] if layout is None else layout)
        self.n_slots_max, self.n_raw_max = n_slots_max, n_raw_max
        off = layout_offsets(self.layout, lidar_type)
        p = PreprocessParams(lidar_type, n_scans, scan_rate, time_unit, point_filter_num, blind, self.layout.itemsize, *off)
        h = C.c_void_p()
        _check(self._L.fl_preprocess_batch_create(C.byref(h), device, C.byref(p), n_slots_max, n_raw_max))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._L.fl_preprocess_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run_device(self, raws, n_slots: int, n_max: int, status=None):
        """fl_preprocess_batch_run_device on torch.cuda.current_stream(): raws the (>= n_slots, 2) int64 table of
        preprocess_raws.  Returns status, an (n_slots, 2) int32 tensor = (FL_OK, |pl_surf|) or (refusal, 0) per slot."""
        import torch
        dev = torch.device("cuda", self.device)
        if not isinstance(raws, torch.Tensor) or raws.dtype != torch.int64 or raws.dim() != 2 or raws.shape[1] != 2 \
                or not raws.is_contiguous() or raws.device != dev or raws.shape[0] < n_slots:
            raise TypeError(f"raws must be the contiguous (S, 2) int64 tensor of preprocess_raws on {dev}, S >= n_slots")
        if status is None:
            status = torch.empty((max(n_slots, 0), 2), dtype=torch.int32, device=dev)
        if not isinstance(status, torch.Tensor) or status.dtype != torch.int32 or not status.is_contiguous() or status.device != dev \
                or status.numel() < 2 * max(n_slots, 0):
            raise TypeError(f"status must be a contiguous int32 tensor of (n_slots, 2) on {dev}")
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        _check(self._L.fl_preprocess_batch_run_device(self.h, raws.data_ptr() if n_slots > 0 else None, n_slots, n_max,
                                                      status.data_ptr() if n_slots > 0 else None, stream))
        return status

    def outputs(self):
        """fl_preprocess_batch_get_outputs as CUDA tensors over the handle's memory: xyzi (n_slots_max, n_raw_max, 4) float32,
        offset_ms (n_slots_max, n_raw_max) float32, out2 (n_slots_max, 2) int32 and last_ms (n_slots_max,) float32."""
        import torch
        ptrs = [C.c_void_p() for _ in range(4)]
        m = C.c_int(0)
        _check(self._L.fl_preprocess_batch_get_outputs(self.h, *[C.byref(p) for p in ptrs], C.byref(m)))
        S, m = self.n_slots_max, int(m.value)
        views = [((S, m, 4), "<f4"), ((S, m), "<f4"), ((S, 2), "<i4"), ((S,), "<f4")]
        return tuple(torch.as_tensor(_DeviceTable(self, int(p.value or 0), S, shape, ts), device=f"cuda:{self.device}")
                     for p, (shape, ts) in zip(ptrs, views))

    def download(self, slot: int):
        """fl_preprocess_batch_download: slot `slot`'s pl_surf of the last call as (xyzi (m, 4) float32, offset_ms (m,) float32,
        last_ms); a refused or uncovered slot has no rows."""
        last = C.c_float(0.0)
        one4, one = np.zeros((1, 4), np.float32), np.zeros(1, np.float32)
        n = _check(self._L.fl_preprocess_batch_download(self.h, slot, one4, one, 0, C.byref(last)))
        xyzi, ms = np.zeros((max(n, 1), 4), np.float32), np.zeros(max(n, 1), np.float32)
        _check(self._L.fl_preprocess_batch_download(self.h, slot, xyzi, ms, n, C.byref(last)))
        return xyzi[:n].copy(), ms[:n].copy(), last.value

    def scan_raws(self, poses=None, n_pose=None, x_end=None, n_slots: int | None = None):
        """The fl_scan_raw_t table of ScanBatch.run_device over this handle's outputs, slot s reading xyzi[s], offset_ms[s] and
        the count out2[s, 0] in place: poses an (S, n_pose_max, 22) float64, n_pose an (S,) int32 and x_end an (S, 26) float64
        CUDA tensor (each may be None when not de-skewing).  S is their first dimension, else n_slots, else n_slots_max."""
        xyzi, ms, out2, _ = self.outputs()
        S = next((t.shape[0] for t in (poses, n_pose, x_end) if t is not None), self.n_slots_max if n_slots is None else n_slots)
        if S > self.n_slots_max:
            raise ValueError(f"{S} slots, the handle has {self.n_slots_max}")
        entries = []
        for s in range(S):
            entries.append((xyzi[s], ms[s], out2[s, :1], None if poses is None else poses[s], None if n_pose is None else n_pose[s:s + 1],
                            None if x_end is None else x_end[s]))
        return scan_raws(entries, device=xyzi.device)


def reloc_grid_device(x_prior, n, step):
    """fl_reloc_expand_grid_device on the current stream: the (n0 n1 n2 n3, 26) float64 hypotheses of the grid n (4 counts) x step
    (x, y, z in m, yaw in rad) around x_prior, a (26,) float64 CUDA tensor.  Hypothesis h = ((i_yaw n2 + i_z) n1 + i_y) n0 + i_x."""
    import torch
    if not isinstance(x_prior, torch.Tensor) or x_prior.device.type != "cuda" or x_prior.dtype != torch.float64 \
            or tuple(x_prior.shape) != (26,) or not x_prior.is_contiguous():
        raise TypeError("x_prior: expected a contiguous (26,) float64 CUDA tensor")
    g = RelocGrid((C.c_int * 4)(*[int(v) for v in n]), (C.c_double * 4)(*[float(v) for v in step]))
    H = int(np.prod([max(int(v), 0) for v in n]))
    out = torch.empty((max(H, 1), 26), dtype=torch.float64, device=x_prior.device)[:H]
    _check(load().fl_reloc_expand_grid_device(x_prior.data_ptr(), C.byref(g), out.data_ptr(),
                                              C.c_void_p(torch.cuda.current_stream(x_prior.device).cuda_stream)))
    return out


def host_register(arr: np.ndarray):
    """Page-lock a numpy array that will be passed repeatedly (the reference's scan buffer)."""
    _check(load().fl_host_register(arr.ctypes.data, arr.nbytes))


def host_unregister(arr: np.ndarray):
    _check(load().fl_host_unregister(arr.ctypes.data))


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _check(load().fl_comm_unique_id(buf))
    return buf.raw


def shard_range(n: int, nranks: int, rank: int):
    """Contiguous shard of n scan points for `rank` (SURVEY.md section 8e)."""
    base, rem = divmod(n, nranks)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
