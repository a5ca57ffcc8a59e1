"""The update's normal equations recomputed from its own outputs, point by point with the measurement model the kernels run
(measure.cuh through tests/kernels/manifold_harness.cu) and summed exactly, without the CPU oracle's looser tolerance.

For the last pass of an update: the state it ran at is x_after of the pass before it (or the prior), its planes are the
fits to the final Nearest_Points (the neighbours of the last searching pass; a pass that does not search reuses them), and
its rows are the points the update left selected.  On a searching last pass, `selected` must equal the model applied to
every point: the kNN gate on d^2 as map.cuh's sq_dist3 computes it, the plane fit, the score.  The problems' own
max_iter (4) converges before the last pass, which then reuses the neighbours; with max_iter = 1 the filter re-searches on
its last pass (esekfom.hpp's forced search on the pass before max_iter, SURVEY T2), so each problem runs both.

Bound on HtH, Hth and res_sum: each entry is a sum of n terms a_i b_i (n = effct) that the kernels form in FP64 along a
summation tree -- 32-row sums per warp in warp_accumulate, accumulated over a worker's tiles, the per-block partials and
sol_reduce's per-warp and cross-warp sums.  Any such tree has depth <= n, so with the product's rounding
|got - exact| <= gamma_{n+1} sum |a_i b_i|, gamma_k = k eps / (1 - k eps), eps = 2^-53.  The exact sums are formed with
error-free products (Veltkamp / Dekker) and math.fsum, which gives the correctly rounded exact sum.  At these sizes the
bound is ~1e-12 of sum |terms|, against the 1e-9 relative the oracle comparison allows; one dropped or doubled row moves
an entry by ~1 / n of it.
"""
import math

import numpy as np
import pytest

from fast_lio_b200 import api
from manifold_harness import Harness, compile_harness

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53
TRI = [(a, b) for a in range(12) for b in range(a, 12)]


@pytest.fixture(scope="module")
def hx(tmp_path_factory):
    return Harness(compile_harness(tmp_path_factory.mktemp("normal_equations_harness")))


def _split(a):
    c = a * 134217729.0                    # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    """p + e == a * b exactly (no FMA; |a b| far from overflow)"""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def _exact_sum(a, b):
    p, e = _two_prod(np.asarray(a, np.float64), np.asarray(b, np.float64))
    return math.fsum(np.concatenate([p, e])), math.fsum(np.abs(p))


def _sq_dist3(a, b):
    """map.cuh sq_dist3: float32, (dx^2 + dy^2) + dz^2, every operation rounded"""
    d = (a.astype(np.float32) - b.astype(np.float32)).astype(np.float32)
    s = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32)
    return (s + d[:, 2] * d[:, 2]).astype(np.float32)


def _run(form, pr, extr, max_iter=None):
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=max_iter or pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr),
                  **({"fused": 0} if form == "split" else {}))
    n = len(pr.scan)
    if form == "device":
        x, P = torch.from_numpy(pr.x_prior.copy()).cuda(), torch.from_numpy(np.ascontiguousarray(pr.P_prior)).cuda()
        f.update_device(torch.from_numpy(np.ascontiguousarray(pr.scan, dtype=np.float32)).cuda(), x, P, pr.R)
        pts, cnt = f.nearest_device(n)
        sel = f.selected_device(n)
        torch.cuda.synchronize()
        nearest, ncnt, selected = pts.cpu().numpy(), cnt.cpu().numpy(), sel.cpu().numpy()
    else:
        f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
        (nearest, ncnt), selected = f.nearest(n), f.selected(n)
    logs = f.pass_logs()
    f.close()
    t.close()
    return nearest, ncnt, selected, logs


def _model(hx, pr, x_at, nearest, ncnt, extr):
    """The harness's measure entry for every scan point at x_at, with d^2 of the 5th neighbour as the search computes it."""
    n = len(pr.scan)
    base = np.zeros((n, 47))
    base[:, :26] = x_at
    base[:, 26:29] = pr.scan[:, :3]
    base[:, 29:44] = nearest[:, :, :3].reshape(n, 15)
    base[:, 44] = ncnt
    base[:, 46] = extr
    world = hx.eval("measure", base, device=False)[:, :3]
    base[:, 45] = _sq_dist3(world, nearest[:, 4, :3])
    return hx.eval("measure", base, device=False)


@pytest.mark.parametrize("max_iter", [None, 1])
@pytest.mark.parametrize("form", ["fused", "split", "device"])
@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
def test_last_pass_normal_equations_are_the_exact_sums_of_its_rows(hx, problems, name, extr, form, max_iter):
    pr = problems(name)
    nearest, ncnt, selected, logs = _run(form, pr, extr, max_iter)
    last = logs[-1]
    assert last["valid"] == 1
    if max_iter == 1:                       # the case that checks the kNN gate, the fit and the score point by point
        assert last["searched"] == 1
    x_at = logs[-2]["x_after"] if len(logs) > 1 else pr.x_prior
    out = _model(hx, pr, x_at, nearest, ncnt, extr)
    sel = selected.astype(bool)
    if last["searched"]:
        want = (out[:, 3] == 1) & (out[:, 4] == 1) & (out[:, 5] == 1)
        assert np.array_equal(sel, want), (np.nonzero(sel != want)[0][:10], out[sel != want][:3, 3:6])
        assert (~want).any(), "the model rejected no point: the rejections were not exercised"
    else:                                   # the rows of a pass that does not search all passed the fit and the score
        assert np.all(out[sel, 4] == 1) and np.all(out[sel, 5] == 1)
    assert last["effct"] == int(sel.sum()) and last["effct"] > 0
    rows, z, absres = out[sel, 12:24], out[sel, 24], np.abs(out[sel, 10])
    k = len(rows)
    gamma = (k + 1) * EPS / (1 - (k + 1) * EPS)
    HtH, Hth = np.asarray(last["HtH"]).reshape(12, 12), np.asarray(last["Hth"])
    worst = 0.0
    for a, b in TRI:
        ex, mag = _exact_sum(rows[:, a], rows[:, b])
        err = abs(HtH[a, b] - ex)
        assert err <= gamma * mag, (a, b, HtH[a, b], ex, mag)
        worst = max(worst, err / mag if mag else 0.0)
    for a in range(12):
        ex, mag = _exact_sum(rows[:, a], z)
        assert abs(Hth[a] - ex) <= gamma * mag, (a, Hth[a], ex, mag)
    ex, mag = _exact_sum(absres, np.ones(k))
    assert abs(last["res_sum"] - ex) <= gamma * mag, (last["res_sum"], ex)
    print(f"{name} extr={extr} {form}: {k} rows, searched={last['searched']}, worst |err| / sum|terms| = {worst:.2e}")


# ------------------------------------------------------------------------------------------------ adversarial scenes
# Whole updates against the reference's own ikd-Tree and the restated update (tests/refcalls.py; answers recorded under
# tests/golden/ref/scene_*.npz), on maps built here where the per-point model meets its field cases:
#   far     the small scene and its state translated by (1500, -800, 20) m: planes fitted in float on kilometre coordinates
#   poles   the small scene plus vertical poles, columns of points at one (x, y) spaced 0.5 m, and scan points on them:
#           exactly collinear neighbour sets, which the fit handles as rank deficient
#   origin  the small scene with a wall x = 5e-4 m, passing within 1e-3 m of the world origin, and scan points on it
#   gate    isolated five-point clusters on z = 1 (a plane through the origin has no fit) at the identity pose, whose 5th neighbour lies at d^2 exactly 5.0f (the
#           kNN gate passes) or at the next float up (it does not)
SCENES = ["far", "poles", "origin", "gate"]
FAR = np.array([1500.0, -800.0, 20.0])
WALL_X = np.float32(5e-4)


def _to_body(x26, pw):
    """World points -> the body frame of state x26 (offset_R_L_I is the identity in these scenes)."""
    from fast_lio_b200 import synth
    R = synth.quat_to_mat(x26[3:7])
    return ((np.asarray(pw, np.float64) - x26[0:3]) @ R - x26[11:14]).astype(np.float32)


def _with_scan(x_true, scan, extra_world):
    body = _to_body(x_true, extra_world)
    return np.concatenate([scan, np.c_[body, np.ones(len(body), np.float32)]]).astype(np.float32)


def scene(problems, name):
    """(map (N, 4), scan (Q, 4), x_prior, P_prior, R, limit, max_iter)"""
    from fast_lio_b200 import synth
    pr = problems("small")
    m, scan, x0 = pr.map_pts.copy(), pr.scan.copy(), pr.x_prior.copy()
    if name == "far":
        m[:, :3] = (m[:, :3].astype(np.float64) + FAR).astype(np.float32)
        x0[0:3] += FAR
    elif name == "poles":
        c = pr.x_true[0:2]
        poles = [c + d for d in ([2.5, 1.5], [-2.0, 2.5], [3.0, -2.0], [-3.5, -1.5])]
        poles = [np.float32(p) for p in poles]
        for p in poles:
            m = m[np.hypot(m[:, 0] - p[0], m[:, 1] - p[1]) > 1.0]
        z = np.arange(-1.75, 4.3, 0.5, dtype=np.float32)
        col = [np.c_[np.full_like(z, p[0]), np.full_like(z, p[1]), z, np.ones_like(z)] for p in poles]
        m = np.concatenate([m] + col).astype(np.float32)
        zs = np.arange(-1.55, 3.5, 0.5)
        scan = _with_scan(pr.x_true, scan, [[p[0], p[1], h] for p in poles for h in zs])
    elif name == "origin":
        m = m[np.abs(m[:, 0]) > 0.6]
        y, z = np.meshgrid(np.arange(-8.0, 8.01, 0.5), np.arange(-1.75, 4.3, 0.5))
        wall = np.c_[np.full(y.size, WALL_X), y.ravel(), z.ravel(), np.ones(y.size)].astype(np.float32)
        m = np.concatenate([m, wall]).astype(np.float32)
        body_world = scan[:, :3].astype(np.float64) @ synth.quat_to_mat(pr.x_true[3:7]).T + pr.x_true[0:3]
        scan = scan[np.abs(body_world[:, 0]) > 0.6]
        ys, zs = np.meshgrid(np.arange(-5.9, 6.0, 0.7), np.arange(-1.4, 3.5, 0.7))
        scan = _with_scan(pr.x_true, scan, np.c_[np.full(ys.size, float(WALL_X)), ys.ravel(), zs.ravel()])
    elif name == "gate":
        up = np.float32(0.000625)          # dz^2 ~ 3.9e-7 lies between half an ulp and 1.5 ulps of 5.0f: 5 + dz^2 -> next float
        near = np.float32([[0.5, 0, 0], [0, 0.6, 0], [-0.7, 0, 0], [0, -0.8, 0]])
        pts, qs = [], []
        for i in range(12):
            for j in range(12):
                q = np.float32([8.0 * i - 44.0, 8.0 * j - 44.0, 1.0])
                fifth = np.float32([2.0, 1.0, up if (i + j) % 2 else 0.0])
                pts += list(q + near) + [q + fifth]
                qs.append(q)
        m = np.c_[np.array(pts, np.float32), np.ones(len(pts), np.float32)].astype(np.float32)
        scan = np.c_[np.array(qs, np.float32), np.ones(len(qs), np.float32)].astype(np.float32)
        x0 = synth.pack_state(np.zeros(3), [0, 0, 0, 1.0], [0, 0, 0, 1.0], np.zeros(3), np.zeros(3), np.zeros(3),
                              np.zeros(3), [0.0, 0.0, -9.809])
    return m, scan, x0, pr.P_prior, pr.R, pr.limit, pr.cfg.max_iter


def _reached(name, scan, nearest, ncnt, logs):
    """Each scene reached its case."""
    if name == "far":
        assert np.abs(nearest[:, :, :3]).max() > 1000.0 and logs[-1]["effct"] > 500
    elif name == "poles":
        same_xy = np.all(nearest[:, :, :2] == nearest[:, :1, :2], axis=(1, 2)) & (ncnt == 5)
        assert same_xy.sum() >= 20, same_xy.sum()          # exactly collinear neighbour sets, fitted
    elif name == "origin":
        on_wall = np.all(nearest[:, :, 0] == WALL_X, axis=1) & (ncnt == 5)
        assert on_wall.sum() >= 20, on_wall.sum()
    elif name == "gate":
        d2 = _sq_dist3(scan[:, :3], nearest[:, 4, :3])   # the first pass searches at the identity pose: world == body
        at, above = d2 == np.float32(5.0), d2 == np.nextafter(np.float32(5.0), np.float32(10.0))
        assert at.sum() == 72 and above.sum() == 72, (at.sum(), above.sum())
        assert logs[0]["searched"] == 1 and logs[0]["effct"] == 72


@pytest.mark.parametrize("form", ["fused", "split", "device"])
@pytest.mark.parametrize("name", SCENES)
def test_adversarial_scene_matches_reference(problems, name, form):
    from refcalls import RefTree, digest
    m, scan, x0, P0, R, limit, max_iter = scene(problems, name)
    o = RefTree(f"scene_{name}", m).update_iterated(scan, x0, P0, max_iter, R, limit, 0)
    if form == "device":
        t = api.KdTree(0, 0.5)
        t.Build(m)
        f = api.Esekf(t, max_points=len(scan), max_iter=max_iter, limit=limit)
        xd, Pd = torch.from_numpy(x0.copy()).cuda(), torch.from_numpy(np.ascontiguousarray(P0)).cuda()
        f.update_device(torch.from_numpy(scan).cuda(), xd, Pd, R)
        pts, cnt = f.nearest_device(len(scan))
        sel = f.selected_device(len(scan))
        torch.cuda.synchronize()
        nearest, ncnt, selected, x, logs = pts.cpu().numpy(), cnt.cpu().numpy(), sel.cpu().numpy(), xd.cpu().numpy(), f.pass_logs()
    else:
        t = api.KdTree(0, 0.5)
        t.Build(m)
        f = api.Esekf(t, max_points=len(scan), max_iter=max_iter, limit=limit, **({"fused": 0} if form == "split" else {}))
        x, _, _ = f.update_iterated_dyn_share_modified(scan, x0, P0, R)
        (nearest, ncnt), selected, logs = f.nearest(len(scan)), f.selected(len(scan)), f.pass_logs()
    assert len(logs) == len(o.passes)
    for lg, op in zip(logs, o.passes):
        assert (lg["searched"], lg["effct"], lg["converged"], lg["valid"]) == (op["searched"], op["effct"], op["converged"], op["valid"])
    assert digest(ncnt) == o.nearest_cnt_digest
    assert digest(nearest) == o.nearest_digest
    assert digest(selected) == o.selected_digest
    assert np.abs(x[0:3] - o.x[0:3]).max() <= 1e-4 and np.abs(x[3:7] - o.x[3:7]).max() <= 1e-4
    _reached(name, scan, nearest, ncnt, logs)
