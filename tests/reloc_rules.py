"""numpy restatements of the relocalisation (fl_reloc_expand_grid_device, fl_filter_relocalize_device): the grid of hypotheses,
the update's FP64 body->world transform of the screen, and the ranking of the survivors."""
import numpy as np


def offsets(i, n, step):
    return (np.asarray(i, np.float64) - (n - 1) / 2.0) * step


def qmul(a, b):
    """lie.cuh qmul over rows (x, y, z, w), in its order of operations."""
    ax, ay, az, aw = (a[..., k] for k in range(4))
    bx, by, bz, bw = (b[..., k] for k in range(4))
    return np.stack([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def expand(prior, n, step):
    """The (n0 n1 n2 n3, 26) hypotheses: h = ((i_yaw n2 + i_z) n1 + i_y) n0 + i_x; pos + offset; rot = q_yaw * rot_prior with
    q_yaw about u = -grav / |grav|; every other component the prior's."""
    prior = np.asarray(prior, np.float64)
    n0, n1, n2, n3 = (int(v) for v in n)
    h = np.arange(n0 * n1 * n2 * n3)
    idx = [h % n0, (h // n0) % n1, (h // (n0 * n1)) % n2, h // (n0 * n1 * n2)]
    X = np.tile(prior, (len(h), 1))
    for a in range(3):
        X[:, a] = prior[a] + offsets(idx[a], (n0, n1, n2)[a], step[a])
    gx, gy, gz = prior[23], prior[24], prior[25]
    gn = np.sqrt(gx * gx + gy * gy + gz * gz)
    half = 0.5 * offsets(idx[3], n3, step[3])
    s = np.sin(half)
    q = np.stack([-gx / gn * s, -gy / gn * s, -gz / gn * s, np.cos(half)], axis=-1)
    X[:, 3:7] = qmul(q, np.broadcast_to(prior[3:7], q.shape))
    return X


def assert_quat_ulp(got, want, ulps=4):
    """Each quaternion within `ulps` units in the last place of its largest component.  A component near zero comes out of
    qmul's cancellation, so a one-ulp difference between two libms' sin / cos of the yaw is many of its own ulps; the quaternion's
    scale is the fair unit."""
    tol = ulps * np.spacing(np.abs(want).max(axis=-1, keepdims=True))
    bad = np.abs(np.asarray(got) - want) > tol
    assert not bad.any(), (np.argwhere(bad)[:5], (np.abs(np.asarray(got) - want) / tol * ulps).max())


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _qrot(q, v):
    """QuaternionBase::_transformVector (lie.cuh qrot) of rows v by q, in its order of operations."""
    qv = np.broadcast_to(q[:3], v.shape)
    uv = _cross(qv, v)
    uv = uv + uv
    return (v + uv * q[3]) + _cross(qv, uv)


def world(x, body):
    """measure.cuh body_to_world in FP64, rounded to float32: the queries of the update and of the screen."""
    p = np.asarray(body, np.float32)[:, :3].astype(np.float64)
    p_this = _qrot(x[7:11], p) + x[11:14]
    return (_qrot(x[3:7], p_this) + x[0:3]).astype(np.float32)


def winner(rows, min_effct):
    """Index into rows of the winner (or -1): FL_OK and last-pass effct >= min_effct qualify; the largest effct, then the smallest
    res_sum / effct, then the earliest row."""
    best, key = -1, None
    for s, r in enumerate(rows):
        if r["status"] != 0 or r["passes"] < 1 or r["effct"] < min_effct:
            continue
        k = (-int(r["effct"]), float(r["res_sum"]) / float(r["effct"]) if r["effct"] else float("nan"))
        if best < 0 or k[0] < key[0] or (k[0] == key[0] and k[1] < key[1]):
            best, key = s, k
    return best
