"""Deterministic synthetic scenes / scans / priors for the measurement-update path.

The reference ships no data and no tests (SURVEY.md section 4); BASELINE.json's
configs are "synthetic".  This module is the single generator used by the
tests, by bench.py and by tests/golden/make_golden.py, so that the CPU oracle
and the CUDA path always see byte-identical inputs.

Scene (SURVEY.md section 8d, adapted): a ground plane plus a lattice of vertical
walls, sampled on the map voxel grid (`voxel`, default 0.5 m = filter_size_map
in launch/mapping_*.launch:12) with AT MOST ONE point per voxel -- the
invariant that ikd-Tree's Add_Points(downsample_on=true) maintains
(include/ikd-Tree/ikd_Tree.cpp:489-521).  The world origin is the first sensor
pose (as in FAST-LIO), so the ground sits at z = -1.77 m and no plane passes
through the origin (esti_plane solves A n = -1, common_lib.h:225-257, which is
singular for planes through the origin).

State layout (26 doubles, the C-ABI / oracle flat layout):
  pos(3) rot(x,y,z,w) offset_R_L_I(x,y,z,w) offset_T_L_I(3) vel(3) bg(3) ba(3) grav(3)
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

VOXEL = 0.5
GROUND_Z = -1.77
WALL_SPACING = 40.0
WALL_OFFSET = 0.23          # keeps wall points 0.23 m inside a voxel along the normal
WALL_CELLS_H = 16           # 8 m high walls
G_LEN = 9.809               # use-ikfom.hpp:8  (98090/10000)

EXTRINSIC_T = {             # config/*.yaml mapping/extrinsic_T
    "avia": (0.04165, 0.02326, -0.0284),
    "velodyne": (0.0, 0.0, 0.28),
    "ouster64": (0.0, 0.0, 0.0),
}


@dataclasses.dataclass
class Config:
    name: str
    lidar: str
    n_map: int
    n_scan: int
    max_iter: int
    seed: int = 1


CONFIGS = {
    # BASELINE.json configs[0..4]
    "avia_2k_50k": Config("avia_2k_50k", "avia", 50_000, 2_000, 3),
    "velodyne_30k_1m": Config("velodyne_30k_1m", "velodyne", 1_000_000, 30_000, 4),
    "ouster64_131k_5m": Config("ouster64_131k_5m", "ouster64", 5_000_000, 131_072, 4),
    "avia_stream_24k": Config("avia_stream_24k", "avia", 1_000_000, 24_000, 3),
    "dense_200k_20m": Config("dense_200k_20m", "ouster64", 20_000_000, 200_000, 4),
    # small cases for CPU-only tests / smoke
    "tiny": Config("tiny", "avia", 6_000, 400, 3),
    "small": Config("small", "velodyne", 20_000, 1_000, 4),
}


# --------------------------------------------------------------------------- quaternion helpers (x,y,z,w)
def quat_from_rpy(roll, pitch, yaw):
    cr, sr = math.cos(roll / 2), math.sin(roll / 2)
    cp, sp = math.cos(pitch / 2), math.sin(pitch / 2)
    cy, sy = math.cos(yaw / 2), math.sin(yaw / 2)
    return np.array([sr * cp * cy - cr * sp * sy,
                     cr * sp * cy + sr * cp * sy,
                     cr * cp * sy - sr * sp * cy,
                     cr * cp * cy + sr * sp * sy], dtype=np.float64)


def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz], dtype=np.float64)


def quat_to_mat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=np.float64)


def quat_exp(v):
    """Unit quaternion of the rotation vector v."""
    th = float(np.linalg.norm(v))
    if th < 1e-12:
        return np.array([0.5 * v[0], 0.5 * v[1], 0.5 * v[2], 1.0])
    s = math.sin(th / 2) / th
    return np.array([s * v[0], s * v[1], s * v[2], math.cos(th / 2)])


# --------------------------------------------------------------------------- state packing
def pack_state(pos, rot, off_r, off_t, vel, bg, ba, grav):
    return np.concatenate([pos, rot, off_r, off_t, vel, bg, ba, grav]).astype(np.float64)


def state_pos(x):
    return x[0:3]


def state_rot(x):
    return x[3:7]


def true_state(lidar: str, step: int = 0) -> np.ndarray:
    """Ground-truth state; `step` translates the sensor 0.1 m per scan (config 4)."""
    pos = np.array([1.3 + 0.1 * step, -0.7, 0.2])
    rot = quat_from_rpy(math.radians(2.0), math.radians(-3.0), math.radians(25.0))
    off_r = np.array([0.0, 0.0, 0.0, 1.0])
    off_t = np.array(EXTRINSIC_T[lidar], dtype=np.float64)
    vel = np.array([0.5, 0.1, 0.0])
    bg = np.array([0.001, -0.002, 0.0005])
    ba = np.array([0.01, 0.02, -0.01])
    grav = np.array([0.0, 0.0, -G_LEN])
    return pack_state(pos, rot, off_r, off_t, vel, bg, ba, grav)


def make_prior(x_true: np.ndarray, seed: int = 3, pos_sigma=0.05, rot_sigma_deg=0.5, coupling: float = 0.3,
               rot_err_deg=(0.0, 0.0, 0.0), grav_var: float = 0.0, grav_rot_corr: float = 0.0, grav_deg: float = 0.0,
               offr_deg: float = 0.0):
    """Prior = truth [+] perturbation (SURVEY.md 8d) and the init_P pattern of
    src/IMU_Processing.hpp:204-211.

    Large corrections (all off by default; they draw no random numbers, so the default prior is unchanged):
      rot_err_deg    adds a (roll, pitch, yaw) error and gives the rotation block a standard deviation of its angle;
      grav_var       gives the gravity block that variance, grav_rot_corr of it coupled to the rotation block
                     (gravity tangent = own part + k * rotation error), and grav_deg tilts the prior's gravity;
      offr_deg       rotates offset_R_L_I by that angle about (1, 1, 1) / sqrt(3), with a matching standard deviation.
    Each is a congruence P := T P T^T of the covariance above, so P stays symmetric positive definite."""
    rng = np.random.default_rng(seed)
    x = x_true.copy()
    x[0:3] += rng.normal(0.0, pos_sigma, 3)
    drot = rng.normal(0.0, math.radians(rot_sigma_deg), 3)
    x[3:7] = quat_mul(x[3:7], quat_exp(drot))
    P = np.eye(23, dtype=np.float64)
    for i in (6, 7, 8, 9, 10, 11):
        P[i, i] = 0.00001
    for i in (15, 16, 17):
        P[i, i] = 0.0001
    for i in (18, 19, 20):
        P[i, i] = 0.001
    P[21, 21] = P[22, 22] = 0.00001
    if coupling > 0.0:
        # a propagated covariance is not diagonal (pos-vel, rot-bg, ... couplings): blend in a
        # random correlation matrix so that every block of the 23x23 algebra is exercised.
        G = rng.normal(size=(23, 23))
        Cm = G @ G.T
        d = np.sqrt(np.diag(Cm))
        Cm = Cm / d[:, None] / d[None, :]
        S = np.sqrt(np.diag(P))
        P = ((1.0 - coupling) * np.eye(23) + coupling * Cm) * S[:, None] * S[None, :]
        P = 0.5 * (P + P.T)
    T = np.eye(23)
    sr = math.radians(float(np.linalg.norm(rot_err_deg)))
    if sr:
        x[3:7] = quat_mul(x[3:7], quat_exp(np.radians(np.asarray(rot_err_deg, dtype=np.float64))))
        T[3:6, 3:6] *= sr / np.sqrt(np.diag(P)[3:6])
    if offr_deg:
        x[7:11] = quat_mul(x[7:11], quat_exp(np.full(3, math.radians(offr_deg) / math.sqrt(3.0))))
        T[6:9, 6:9] *= math.radians(offr_deg) / np.sqrt(np.diag(P)[6:9])
    if grav_var:
        k = grav_rot_corr * math.sqrt(grav_var) / (sr or math.radians(rot_sigma_deg))
        T[21:23, 21:23] *= math.sqrt(grav_var * (1.0 - grav_rot_corr ** 2)) / np.sqrt(np.diag(P)[21:23])
        T[21, 3:6] = k * T[4, 3:6]               # tangent 0 follows pitch, tangent 1 follows roll
        T[22, 3:6] = k * T[3, 3:6]
    if grav_deg:
        g = x[23:26] / np.linalg.norm(x[23:26])
        axis = np.cross(g, [1.0, 0.0, 0.0])
        axis /= np.linalg.norm(axis)
        x[23:26] = quat_to_mat(quat_exp(axis * math.radians(grav_deg))) @ x[23:26]
    if not np.array_equal(T, np.eye(23)):
        P = T @ P @ T.T
        P = 0.5 * (P + P.T)
    return x, np.ascontiguousarray(P)


# --------------------------------------------------------------------------- scene
@dataclasses.dataclass
class Scene:
    extent: float               # half side length of the square scene, metres
    wall_coords: np.ndarray     # wall plane coordinates (used for both x- and y-walls)
    n_cells: int


def _wall_coords(half):
    k = int(math.floor(half / WALL_SPACING))
    base = np.arange(-k, k + 1, dtype=np.float64) * WALL_SPACING
    # snap to the voxel grid then offset inside the cell
    return np.floor(base / VOXEL) * VOXEL + WALL_OFFSET


def _scene_for(n_map: int, fill: float = 0.85) -> Scene:
    half = 10.0
    while True:
        side = int(round(2 * half / VOXEL))
        walls = _wall_coords(half - 1.0)
        cells = side * side + 2 * len(walls) * side * WALL_CELLS_H
        if cells * fill >= n_map:
            return Scene(half, walls, cells)
        half += 5.0


def _ground_cells(ix0, ix1, iy0, iy1):
    ix, iy = np.meshgrid(np.arange(ix0, ix1, dtype=np.int64), np.arange(iy0, iy1, dtype=np.int64), indexing="ij")
    return ix.ravel(), iy.ravel()


def _points_from_cells(rng, kind, a, b, wall_c):
    """kind 0: ground cell (ix=a, iy=b); kind 1: wall x=wall_c, cell (iy=a, iz=b);
    kind 2: wall y=wall_c, cell (ix=a, iz=b).  Returns float64 xyz."""
    n = len(kind)
    u = rng.uniform(0.02, 0.48, size=(n, 2))
    jit = rng.normal(0.0, 0.01, size=n)
    xyz = np.empty((n, 3), dtype=np.float64)
    g = kind == 0
    xyz[g, 0] = a[g] * VOXEL + u[g, 0]
    xyz[g, 1] = b[g] * VOXEL + u[g, 1]
    xyz[g, 2] = GROUND_Z + np.clip(jit[g], -0.04, 0.04)
    wx = kind == 1
    xyz[wx, 0] = wall_c[wx] + np.clip(jit[wx], -0.04, 0.04)
    xyz[wx, 1] = a[wx] * VOXEL + u[wx, 0]
    xyz[wx, 2] = b[wx] * VOXEL + u[wx, 1]
    wy = kind == 2
    xyz[wy, 0] = a[wy] * VOXEL + u[wy, 0]
    xyz[wy, 1] = wall_c[wy] + np.clip(jit[wy], -0.04, 0.04)
    xyz[wy, 2] = b[wy] * VOXEL + u[wy, 1]
    return xyz


def _enumerate_cells(scene: Scene, cx=0.0, cy=0.0, radius=None):
    """All surface cells of the scene (optionally only those whose cell origin is within
    `radius` of (cx, cy) horizontally).  Returns (kind, a, b, wall_c)."""
    half = scene.extent
    lo = int(round(-half / VOXEL))
    hi = int(round(half / VOXEL))
    if radius is None:
        ix0, ix1, iy0, iy1 = lo, hi, lo, hi
    else:
        ix0 = max(lo, int(math.floor((cx - radius) / VOXEL)))
        ix1 = min(hi, int(math.ceil((cx + radius) / VOXEL)))
        iy0 = max(lo, int(math.floor((cy - radius) / VOXEL)))
        iy1 = min(hi, int(math.ceil((cy + radius) / VOXEL)))
    gx, gy = _ground_cells(ix0, ix1, iy0, iy1)
    kinds = [np.zeros(len(gx), dtype=np.int8)]
    aa = [gx]
    bb = [gy]
    cc = [np.zeros(len(gx))]
    iz0 = int(math.floor(GROUND_Z / VOXEL)) + 1
    izs = np.arange(iz0, iz0 + WALL_CELLS_H, dtype=np.int64)
    wall_cols = set(int(math.floor(c / VOXEL)) for c in scene.wall_coords)
    for c in scene.wall_coords:
        if radius is not None and abs(c - cx) > radius:
            pass
        else:
            # wall x = c : cells (iy, iz)
            iy, iz = np.meshgrid(np.arange(iy0, iy1, dtype=np.int64), izs, indexing="ij")
            kinds.append(np.full(iy.size, 1, dtype=np.int8)); aa.append(iy.ravel()); bb.append(iz.ravel()); cc.append(np.full(iy.size, c))
        if radius is not None and abs(c - cy) > radius:
            pass
        else:
            # wall y = c : cells (ix, iz); skip columns that an x-wall already occupies
            ixs = np.array([i for i in range(ix0, ix1) if i not in wall_cols], dtype=np.int64)
            ix, iz = np.meshgrid(ixs, izs, indexing="ij")
            kinds.append(np.full(ix.size, 2, dtype=np.int8)); aa.append(ix.ravel()); bb.append(iz.ravel()); cc.append(np.full(ix.size, c))
    kind = np.concatenate(kinds)
    a = np.concatenate(aa)
    b = np.concatenate(bb)
    c = np.concatenate(cc)
    if radius is not None:
        # horizontal position of the cell centre
        px = np.select([kind == 0, kind == 1, kind == 2], [(a + 0.5) * VOXEL, c, (a + 0.5) * VOXEL])
        py = np.select([kind == 0, kind == 1, kind == 2], [(b + 0.5) * VOXEL, (a + 0.5) * VOXEL, c])
        keep = (px - cx) ** 2 + (py - cy) ** 2 <= radius * radius
        kind, a, b, c = kind[keep], a[keep], b[keep], c[keep]
    return kind, a, b, c


def make_map(n_map: int, seed: int = 1):
    """n_map x 4 float32 (x, y, z, intensity), <= 1 point per VOXEL cell."""
    scene = _scene_for(n_map)
    rng = np.random.default_rng(seed)
    kind, a, b, c = _enumerate_cells(scene)
    assert len(kind) >= n_map, (len(kind), n_map)
    sel = rng.permutation(len(kind))[:n_map]
    sel.sort()
    xyz = _points_from_cells(rng, kind[sel], a[sel], b[sel], c[sel])
    pts = np.empty((n_map, 4), dtype=np.float32)
    pts[:, :3] = xyz.astype(np.float32)
    pts[:, 3] = rng.uniform(1.0, 100.0, n_map).astype(np.float32)
    pts = pts[rng.permutation(n_map)]          # the map arrives unordered
    return np.ascontiguousarray(pts), scene


def make_scan(scene: Scene, n_scan: int, x_true: np.ndarray, seed: int = 2, noise_sigma: float = 0.02, order: str = "voxelgrid"):
    """n_scan x 4 float32 body-frame points (x, y, z, intensity) of surfaces within range of
    the true sensor pose, one per VOXEL cell (the scan is voxel-filtered upstream,
    laserMapping.cpp:904-907), with `noise_sigma` range noise along the surface normal."""
    rng = np.random.default_rng(seed)
    pos = state_pos(x_true)
    radius = 20.0
    while True:
        kind, a, b, c = _enumerate_cells(scene, pos[0], pos[1], radius)
        if len(kind) >= int(1.3 * n_scan) or radius > 4 * scene.extent:
            break
        radius *= 1.25
    assert len(kind) >= n_scan, "scene too small for the requested scan"
    sel = rng.permutation(len(kind))[:n_scan]
    sel.sort()
    kind, a, b, c = kind[sel], a[sel], b[sel], c[sel]
    n = n_scan
    u = rng.uniform(0.0, VOXEL, size=(n, 2))
    nz = rng.normal(0.0, noise_sigma, size=n)
    w = np.empty((n, 3), dtype=np.float64)
    g = kind == 0
    w[g, 0] = a[g] * VOXEL + u[g, 0]; w[g, 1] = b[g] * VOXEL + u[g, 1]; w[g, 2] = GROUND_Z + nz[g]
    wx = kind == 1
    w[wx, 0] = c[wx] + nz[wx]; w[wx, 1] = a[wx] * VOXEL + u[wx, 0]; w[wx, 2] = b[wx] * VOXEL + u[wx, 1]
    wy = kind == 2
    w[wy, 0] = a[wy] * VOXEL + u[wy, 0]; w[wy, 1] = c[wy] + nz[wy]; w[wy, 2] = b[wy] * VOXEL + u[wy, 1]
    # world -> body:  p_b = R_LI^T ( R^T (p_w - pos) - t_LI )
    R = quat_to_mat(x_true[3:7])
    R_li = quat_to_mat(x_true[7:11])
    t_li = x_true[11:14]
    p_imu = (w - pos) @ R            # == (R^T (w-pos)^T)^T
    p_b = (p_imu - t_li) @ R_li
    scan = np.empty((n, 4), dtype=np.float32)
    scan[:, :3] = p_b.astype(np.float32)
    scan[:, 3] = rng.uniform(1.0, 100.0, n).astype(np.float32)
    if order == "random":
        scan = scan[rng.permutation(n)]
    else:
        # the update's input is the output of pcl::VoxelGrid (laserMapping.cpp:904-907), which emits one
        # centroid per occupied leaf sorted by leaf index  ix + iy*nx + iz*nx*ny  (body frame): reproduce
        # that ordering (x fastest, then y, then z)
        cell = np.floor(scan[:, :3].astype(np.float64) / VOXEL).astype(np.int64)
        cell -= cell.min(axis=0)
        nx, ny = int(cell[:, 0].max()) + 1, int(cell[:, 1].max()) + 1
        key = cell[:, 0] + cell[:, 1] * nx + cell[:, 2] * nx * ny
        scan = scan[np.argsort(key, kind="stable")]
    return np.ascontiguousarray(scan)


@dataclasses.dataclass
class RawScan:
    xyzi: np.ndarray         # n x 4 float32, body (LiDAR) frame AT EACH POINT'S OWN TIME, acquisition order
    offset_ms: np.ndarray    # n float32, PointType::curvature (offset from the first point, milliseconds)
    imu_pose: np.ndarray     # n_pose x 22 float64, IMUpose (msg/Pose6D.msg), offsets in seconds
    x_end: np.ndarray        # 26, state at the frame end
    truth_end: np.ndarray    # n x 3 float64: the same surface points in the LiDAR frame at the frame end


def make_raw_scan(scene: Scene, n_raw: int, x_end: np.ndarray, seed: int = 5, period_s: float = 0.1, imu_hz: float = 200.0,
                  omega=(0.3, -0.2, 0.8), accel=(0.4, -0.3, 0.1), noise_sigma: float = 0.0, shuffle: bool = True) -> RawScan:
    """A raw (not yet de-skewed, not yet down-sampled) scan of `scene` taken by a sensor that moves with constant
    body-frame angular velocity `omega` and constant world acceleration `accel` during `period_s`, ending in `x_end`.
    That is the motion model of UndistortPcl's backward pass (IMU_Processing.hpp:327-336), so compensating the
    points with the returned IMUpose list must reproduce `truth_end` up to float32 rounding.  Several points fall into
    one 0.5 m cell (raw scans are denser than the down-sampled cloud the update consumes)."""
    rng = np.random.default_rng(seed)
    omega = np.asarray(omega, dtype=np.float64)
    accel = np.asarray(accel, dtype=np.float64)
    T = float(period_s)
    R_end = quat_to_mat(x_end[3:7])
    p_end = np.array(x_end[0:3], dtype=np.float64)
    v_end = np.array(x_end[14:17], dtype=np.float64)
    R_li = quat_to_mat(x_end[7:11])
    t_li = np.array(x_end[11:14], dtype=np.float64)
    R0 = R_end @ quat_to_mat(quat_exp(-omega * T))
    v0 = v_end - accel * T
    p0 = p_end - v0 * T - 0.5 * accel * T * T

    def pose_at(t):
        return R0 @ quat_to_mat(quat_exp(omega * t)), p0 + v0 * t + 0.5 * accel * t * t, v0 + accel * t

    # surface points around the end pose, with replacement over cells -> several points per voxel
    radius = 15.0
    while True:
        kind, a, b, c = _enumerate_cells(scene, p_end[0], p_end[1], radius)
        if len(kind) * 3 >= n_raw or radius > 4 * scene.extent:
            break
        radius *= 1.25
    pick = rng.integers(0, len(kind), size=n_raw)
    w = _points_from_cells(rng, kind[pick], a[pick], b[pick], c[pick])
    if noise_sigma > 0:
        w += rng.normal(0.0, noise_sigma, size=w.shape)
    t = np.sort(rng.uniform(0.0, T, size=n_raw))
    t[0] = 0.0                                          # the first point defines the offset origin
    t_ms = (t * 1000.0).astype(np.float32)
    t_used = t_ms.astype(np.float64) / 1000.0           # what the de-skew will see
    xyz = np.empty((n_raw, 3), dtype=np.float64)
    for lo in range(0, n_raw, 4096):                    # per-point pose, vectorised through Rodrigues
        tt = t_used[lo:lo + 4096]
        th = np.linalg.norm(omega)
        k = omega / th if th > 0 else np.zeros(3)
        K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        ang = th * tt
        Rt = R0[None] @ (np.eye(3)[None] + np.sin(ang)[:, None, None] * K[None] + (1 - np.cos(ang))[:, None, None] * (K @ K)[None])
        pt = p0[None] + v0[None] * tt[:, None] + 0.5 * accel[None] * (tt * tt)[:, None]
        p_imu = np.einsum("nji,nj->ni", Rt, w[lo:lo + 4096] - pt)          # R(t)^T (w - p(t))
        xyz[lo:lo + 4096] = (p_imu - t_li) @ R_li
    truth = ((w - p_end) @ R_end - t_li) @ R_li
    xyzi = np.empty((n_raw, 4), dtype=np.float32)
    xyzi[:, :3] = xyz.astype(np.float32)
    xyzi[:, 3] = rng.uniform(1.0, 100.0, n_raw).astype(np.float32)
    if shuffle:                                          # drivers deliver points ring by ring, not by time
        perm = rng.permutation(n_raw)
        xyzi, t_ms, truth = xyzi[perm], t_ms[perm], truth[perm]
    # IMUpose: offset 0 first (IMU_Processing.hpp:241), then one entry per IMU sample, the last one at/after the frame end
    n_imu = int(math.ceil(T * imu_hz))
    offs = [0.0] + [min(T, (k + 1) / imu_hz) for k in range(n_imu)]
    poses = np.zeros((len(offs), 22), dtype=np.float64)
    for k, o in enumerate(offs):
        Rk, pk, vk = pose_at(o)
        poses[k, 0] = o
        poses[k, 1:4] = accel                           # acc: world-frame acceleration of the segment ENDING here (:327)
        poses[k, 4:7] = omega                           # gyr: unbiased body-frame rate of that segment (:328)
        poses[k, 7:10] = vk
        poses[k, 10:13] = pk
        poses[k, 13:22] = Rk.reshape(-1)
    return RawScan(np.ascontiguousarray(xyzi), np.ascontiguousarray(t_ms), poses, np.array(x_end, dtype=np.float64).copy(), truth)


@dataclasses.dataclass
class Problem:
    cfg: Config
    map_pts: np.ndarray      # N x 4 float32
    scan: np.ndarray         # Q x 4 float32 (body frame)
    x_true: np.ndarray       # 26
    x_prior: np.ndarray      # 26
    P_prior: np.ndarray      # 23 x 23
    scene: Scene
    R: float = 0.001         # LASER_POINT_COV, laserMapping.cpp:64
    limit: float = 0.001     # epsi, laserMapping.cpp:826-827
    extrinsic_est_en: int = 0


def make_problem(name_or_cfg, extrinsic_est_en: int = 0) -> Problem:
    cfg = CONFIGS[name_or_cfg] if isinstance(name_or_cfg, str) else name_or_cfg
    map_pts, scene = make_map(cfg.n_map, seed=cfg.seed)
    xt = true_state(cfg.lidar)
    scan = make_scan(scene, cfg.n_scan, xt, seed=cfg.seed + 1)
    xp, P = make_prior(xt, seed=cfg.seed + 2)
    return Problem(cfg, map_pts, scan, xt, xp, P, scene, extrinsic_est_en=extrinsic_est_en)
