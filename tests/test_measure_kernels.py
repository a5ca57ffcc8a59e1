"""The per-point measurement model (measure.cuh) on the host and the device, against the CPU oracle's restatement and a
60-digit restatement (tests/plane_mp.py), on the inputs where a float32 plane fit goes wrong: planes far from the origin
and through it, coincident, duplicated, collinear and nearly collinear neighbours, a zero column, every column order,
and the float on either side of each gate.

Plane-fit bound (float32, u = 2^-24).  esti_plane is Householder QR least squares with column pivoting, so (Higham,
Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm 19.13 / 20.3) the computed x^ solves exactly a problem
(A + dA) x = b + db with ||dA e_j|| <= g ||A e_j|| and ||db|| <= g ||b||, g = c m n u (m = 5, n = 3; we take c = 4, so
g = 60 u).  To first order the residual vector r = A x + 1 then moves by (Higham Thm 20.1, with the kappa^2 term of x
not reaching r except through ||r||):  ||dr|| <= g (||b|| + ||A||_F ||x|| + kappa(A) ||r||).  pd2_j = r_j / |x| and
d = 1 / |x| is the plane's distance from the origin, so the neighbour distances move by d ||dr||, and the normalisation
by |x^| instead of |x| adds |pd2_j| g kappa(A).  Rounding x^ / |x^| and 1 / |x^| to float adds 2 u (max|p| + d).  The
float check |n . p + d| > 0.1 evaluates four products and three sums of magnitude <= max|p| + d: 4 u (max|p| + d).
The bound applies while g kappa(A) < 0.1 and the fit found full rank; otherwise the problem has no unique answer and
only bit-equality with the oracle is asserted.

Row bound (FP64, eps = 2^-52).  The row is two quaternion rotations (Eigen's _transformVector, ~6 eps each of
|v|), a cross product with the lever arm p_this and, with extrinsic estimation, a 3x3 product with hat(p_be) (both up
to ~100 m): every entry is within 32 eps (1 + max(|p_this|, |p_be|)) of the exact value from the same float plane and
point.  z = -pd2 exactly.
"""
from __future__ import annotations

import itertools
import math

import mpmath as mpm
import numpy as np
import pytest

import plane_mp as PM
from manifold_harness import Harness, compile_harness
from oracle import bind

U = 2.0 ** -24
EPS = 2.0 ** -52
G = 60 * U


@pytest.fixture(scope="module")
def hx(tmp_path_factory):
    return Harness(compile_harness(tmp_path_factory.mktemp("measure_harness")))


# ------------------------------------------------------------------------------------------------ inputs
def _unit(rng):
    v = rng.standard_normal(3)
    return v / np.linalg.norm(v)


def _basis(n):
    a = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    u = np.cross(n, a)
    u /= np.linalg.norm(u)
    return u, np.cross(n, u)


def _plane(rng, center, normal, spread, noise):
    u, v = _basis(normal)
    a, b = rng.uniform(-spread, spread, (2, 5))
    return (center + a[:, None] * u + b[:, None] * v + noise * rng.standard_normal(5)[:, None] * normal).astype(np.float32)


def plane_families(seed=11):
    """name -> list of 5 x 3 float32 neighbour sets."""
    rng = np.random.default_rng(seed)
    F = {}
    F["well"] = [_plane(rng, dist * _unit(rng), _unit(rng), spread, noise)
                 for dist in (1.0, 10.0, 100.0, 1e3, 1e4) for spread in (0.1, 0.3, 1.0) for noise in (0.0, 0.01, 0.05)
                 for _ in range(2)]
    near = []
    for off in (1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 0.0):
        for _ in range(3):
            n = _unit(rng)
            u, _ = _basis(n)
            near.append(_plane(rng, off * n + 3.0 * u, n, 0.5, 0.0))
    near.append(np.array([[1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 3, 0], [-1, 2, 0]], np.float32))   # z = 0 exactly
    F["near_origin"] = near
    deg = [np.tile(np.float32([3, 0, 0]), (5, 1)), np.tile(rng.uniform(-20, 20, 3).astype(np.float32), (5, 1))]
    for k in (2, 3, 4):
        for _ in range(3):
            p = _plane(rng, 10 * _unit(rng), _unit(rng), 0.5, 0.01)
            p[1:k] = p[0]
            deg.append(p)
    for axis in range(3):                                            # axis-aligned lines
        p = np.tile(rng.uniform(-5, 5, 3).astype(np.float32), (5, 1))
        p[:, axis] = np.float32([0.0, 0.5, 1.0, 1.5, 2.0]) + p[0, axis]
        deg.append(p)
    for _ in range(6):                                               # general lines
        p0, d = rng.uniform(-20, 20, 3), _unit(rng)
        deg.append((p0 + np.linspace(-1, 1, 5)[:, None] * d).astype(np.float32))
    F["degenerate"] = deg
    nc = []
    for aspect in (1e-3, 1e-4, 1e-5, 1e-6, 1e-7):
        for _ in range(4):
            p0, d, e = rng.uniform(-20, 20, 3), _unit(rng), _unit(rng)
            t = np.linspace(-1, 1, 5)
            nc.append((p0 + t[:, None] * d + aspect * rng.standard_normal(5)[:, None] * e).astype(np.float32))
    F["near_collinear"] = nc
    zc = []
    for _ in range(4):
        p = _plane(rng, np.array([0.0, 4.0, 2.0]), np.array([1.0, 0.0, 0.0]), 1.0, 0.0)
        p[:, 0] = 0.0
        zc.append(p)
    F["zero_column"] = zc
    perms = []
    for base in (F["well"][7], F["well"][40], zc[0], nc[2], near[0]):
        perms += [np.ascontiguousarray(base[:, list(o)]) for o in itertools.permutations(range(3))]
    F["column_orders"] = perms
    F["origin"] = [np.zeros((5, 3), np.float32)]
    return F


def all_planes():
    return [p for ps in plane_families().values() for p in ps]


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def _same(a, b):
    """bit for bit, with every NaN equal to every NaN"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(both_nan | (_bits(a) == _bits(b))))


def _harness_planes(hx, planes, device, threshold=0.1):
    return hx.eval("esti_plane", [list(p.astype(np.float64).ravel()) + [threshold] for p in planes], device=device)


def _oracle_planes(planes, threshold=0.1):
    out, traces = [], []
    for p in planes:
        ok, pabcd, tr = bind.esti_plane_trace(p, threshold)
        out.append([float(ok)] + [float(t) for t in pabcd])
        traces.append(tr)
    return np.array(out), traces


# ------------------------------------------------------------------------------------------------ plane fit
def branch_counts(traces):
    c = {"swap": 0, "rank<3": 0, "tiny_tail": 0, "downdate": 0, "recompute": 0, "zero_norm_skip": 0}
    orders = set()
    for t in traces:
        c["swap"] += int(any(t["transp"][k] != k for k in range(3)))
        c["rank<3"] += int(t["nonzero_pivots"] < 3)
        c["tiny_tail"] += int(t["tiny_tail"].any())
        c["downdate"] += int((t["norm"] == 1).sum())
        c["recompute"] += int((t["norm"] == 2).sum())
        c["zero_norm_skip"] += int((t["norm"] == 3).sum())
        orders.add(tuple(int(v) for v in t["transp"]))
    return c, orders


# each traced branch of esti_plane, at least this often over the 187 sets of all_planes(); the counts are 157 sets with a
# column swap, 38 rank-deficient, 16 with a tiny Householder tail, 325 norm downdates, 206 recomputes, 30 zero-norm skips
MIN_BRANCH = {"swap": 100, "rank<3": 20, "tiny_tail": 8, "downdate": 200, "recompute": 100, "zero_norm_skip": 15}


def test_inputs_reach_every_plane_branch():
    _, traces = _oracle_planes(all_planes())
    c, orders = branch_counts(traces)
    for k, v in MIN_BRANCH.items():
        assert c[k] >= v, (k, c)
    # transposition patterns: transp[0] in {0,1,2}, transp[1] in {1,2}, transp[2] == 2 -- all six reached
    assert len(orders) == 6, orders


def test_host_plane_matches_oracle(hx):
    planes = all_planes()
    host, (orc, _) = _harness_planes(hx, planes, False), _oracle_planes(planes)
    bad = [i for i in range(len(planes)) if not _same(host[i], orc[i])]
    assert not bad, [(planes[i].tolist(), host[i], orc[i]) for i in bad[:3]]


@pytest.mark.gpu
def test_device_plane_matches_host_and_oracle(hx):
    planes = all_planes() + [e for e, _ in _plane_edge_inputs(hx)]
    dev, host = _harness_planes(hx, planes, True), _harness_planes(hx, planes, False)
    orc, traces = _oracle_planes(planes)
    for i in range(len(planes)):
        assert _same(dev[i], host[i]) and _same(dev[i], orc[i]), (planes[i].tolist(), dev[i], host[i], orc[i])
    c, _ = branch_counts(traces)
    print("esti_plane device branches:", c)
    for k, v in MIN_BRANCH.items():
        assert c[k] >= v, (k, c)


def plane_bound(p, x, pd2):
    """The float plane's error bound at each neighbour (module docstring); None where it does not apply."""
    A = p.astype(np.float64)
    s = np.linalg.svd(A, compute_uv=False)
    if s[-1] == 0.0:
        return None
    kappa = s[0] / s[-1]
    if G * kappa >= 0.1:
        return None
    xf = np.array([float(t) for t in x])
    nx = float(np.linalg.norm(xf))
    d = 1.0 / nx
    r = np.array([float(t) for t in pd2]) * nx
    pmax = float(np.abs(A).max()) * math.sqrt(3)
    dr = G * (math.sqrt(5) + np.linalg.norm(A) * nx + kappa * np.linalg.norm(r))
    return d * dr + np.abs(np.array([float(t) for t in pd2])) * G * kappa + 6 * U * (pmax + d)


def _full_rank_planes():
    out = []
    for name, ps in plane_families().items():
        for p in ps:
            ok, pabcd, tr = bind.esti_plane_trace(p)
            if tr["nonzero_pivots"] == 3 and np.all(np.isfinite(pabcd)):
                out.append((name, p, ok, pabcd))
    return out


def test_plane_within_bound_of_extended_precision():
    """|pd2_float - pd2_exact| at every neighbour within plane_bound, and the accept decision equals the exact one wherever
    the exact worst residual is farther than that bound from 0.1."""
    checked = decided = 0
    worst = 0.0
    for name, p, ok, pabcd in _full_rank_planes():
        x, pd2 = PM.plane_exact(p)
        b = plane_bound(p, x, pd2)
        if b is None:
            continue
        got = [PM.at_plane(pabcd, q) for q in p]
        err = np.array([float(abs(g - e)) for g, e in zip(got, pd2)])
        assert np.all(err <= b), (name, p.tolist(), err, b)
        worst = max(worst, float((err / b).max()))
        checked += 1
        w = max(float(abs(e)) for e in pd2)
        if abs(w - 0.1) > float(b.max()):
            assert ok == (w <= 0.1), (name, p.tolist(), w, b)
            decided += 1
    print(f"plane bound: {checked} fits, worst error / bound {worst:.3g}, {decided} decisions checked")
    assert checked >= 100 and decided >= 80


# ------------------------------------------------------------------------------------------------ threshold edges
def _last_true(pred, lo, hi):
    """lo (float32, pred true) < hi (pred false): the last float32 in [lo, hi) where pred holds, by bisection on the bits."""
    a, b = int(np.float32(lo).view(np.int32)), int(np.float32(hi).view(np.int32))
    assert a >= 0 and b >= 0 and pred(np.float32(lo)) and not pred(np.float32(hi))
    while b - a > 1:
        m = (a + b) // 2
        if pred(np.int32(m).view(np.float32)):
            a = m
        else:
            b = m
    return np.int32(a).view(np.float32)


def _ulps_around(v, ks=(1, 2)):
    out = [np.float32(v)]
    for k in ks:
        up = dn = np.float32(v)
        for _ in range(k):
            up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        out += [up, dn]
    return out


def _plane_edge_inputs(hx):
    """(5 x 3 points, edge value) at both sides of the 0.1 m acceptance: neighbour 0 moved along z (the planes are
    z ~ const) to the last float where the fit is accepted, and +-1, +-2 ulps."""
    rng = np.random.default_rng(5)
    out = []
    for dist in (1.0, 30.0, 1e3):
        for _ in range(2):
            base = _plane(rng, np.array([rng.uniform(-dist, dist), rng.uniform(-dist, dist), dist]), np.array([0.0, 0.0, 1.0]),
                          1.0, 0.0)

            def ok_at(z):
                q = base.copy()
                q[0, 2] = z
                return _harness_planes(hx, [q], False)[0][0] == 1.0
            z_edge = _last_true(ok_at, base[0, 2], base[0, 2] + np.float32(0.5))
            for z in _ulps_around(z_edge):
                q = base.copy()
                q[0, 2] = z
                out.append((q, z_edge))
    return out


def test_plane_threshold_edge_host_matches_oracle(hx):
    edges = _plane_edge_inputs(hx)
    planes = [e for e, _ in edges]
    host, (orc, _) = _harness_planes(hx, planes, False), _oracle_planes(planes)
    for i in range(len(planes)):
        assert _same(host[i], orc[i]), (planes[i].tolist(), host[i], orc[i])
    assert {h[0] for h in host} == {0.0, 1.0}


# ------------------------------------------------------------------------------------------------ per-point measure
def _quat(rng, angle):
    a = _unit(rng)
    return list(a * math.sin(angle / 2)) + [math.cos(angle / 2)]


def measure_inputs(seed=3):
    """47-wide harness inputs: x26, body point, 5 x 3 neighbours, count, 5th squared distance, extr."""
    rng = np.random.default_rng(seed)
    xs = []
    gates = [(5, 1.0), (5, 5.0), (5, float(np.nextafter(np.float32(5), np.float32(np.inf)))), (4, 1.0), (5, math.nan)]
    for i in range(80):
        x = np.zeros(26)
        x[0:3] = rng.uniform(-200, 200, 3)
        x[3:7] = _quat(rng, rng.uniform(0, math.pi))
        x[7:11] = _quat(rng, rng.uniform(0, 0.2))
        x[11:14] = rng.uniform(-0.3, 0.3, 3)
        x[23:26] = [0.0, 0.0, -9.809]
        r = 10 ** rng.uniform(-0.5, 2)
        pb = (_unit(rng) * r).astype(np.float32)
        # the world point, then a plane near it
        pw = np.zeros(3, np.float32)
        bind.lib().oracle_transform_point(x, np.ascontiguousarray(pb), pw)
        n = _unit(rng)
        off = rng.choice([0.0, 0.01, 0.05, 0.3]) * rng.choice([-1, 1])
        near = _plane(rng, pw.astype(np.float64) + off * n, n, 0.5, rng.choice([0.0, 0.01]))
        cnt, d5 = gates[i % len(gates)]
        for extr in (0, 1):
            xs.append(list(x) + list(pb.astype(np.float64)) + list(near.astype(np.float64).ravel()) + [cnt, d5, extr])
    return xs


def _oracle_measure(xs):
    return np.array([bind.measure_point(x[:26], x[26:29], x[29:44], int(x[44]), x[45], int(x[46])) for x in xs])


def _score_edge_inputs(hx):
    """At the identity pose the world point is the body point.  Neighbours on a plane z = c; the body point moved up
    from the plane to the last float z where the score gate passes, and +-1, +-2 ulps, with and without extr."""
    rng = np.random.default_rng(9)
    x = [0.0] * 26
    x[6] = x[10] = 1.0
    x[23:26] = [0.0, 0.0, -9.809]
    out = []
    for c in (0.5, 2.0, 7.0, 30.0):
        for _ in range(2):
            xy = rng.uniform(-20, 20, 2).astype(np.float32)
            near = _plane(rng, np.array([xy[0], xy[1], c]), np.array([0.0, 0.0, 1.0]), 0.5, 0.0)
            near[:, 2] = np.float32(c)

            def at(z, extr=0):
                return x + [float(xy[0]), float(xy[1]), float(z)] + list(near.astype(np.float64).ravel()) + [5, 1.0, extr]

            def passes(z):
                return hx.eval("measure", [at(z)], False)[0][5] == 1.0
            edge = _last_true(passes, np.float32(c), np.float32(c + 10.0))
            out += [at(z, extr) for z in _ulps_around(edge) for extr in (0, 1)]
    return out


def test_measure_host_matches_oracle(hx):
    xs = measure_inputs()
    host, orc = hx.eval("measure", xs, False), _oracle_measure(xs)
    for i in range(len(xs)):
        assert _same(host[i][:25], orc[i]), (i, host[i][:25], orc[i])
        assert _same(host[i][25:38], host[i][12:25]), i           # jacobian_row == jacobian_row_at
    flags = host[:, 3:6]
    for j in range(3):                                             # every gate both ways
        assert set(flags[:, j]) == {0.0, 1.0}, j


def test_score_edge_host_matches_oracle(hx):
    xs = _score_edge_inputs(hx)
    assert len(xs) >= 10
    host, orc = hx.eval("measure", xs, False), _oracle_measure(xs)
    for i in range(len(xs)):
        assert _same(host[i][:25], orc[i]), (i, host[i][:25], orc[i])
    assert set(host[:, 5]) == {0.0, 1.0}


def test_row_within_bound_of_extended_precision(hx):
    xs = measure_inputs()
    host = hx.eval("measure", xs, False)
    worst = 0.0
    for x, o in zip(xs, host):
        nv = list(o[6:9]) + [o[10]]
        row, z, lever = PM.jacobian_row(x[:26], x[26:29], nv, int(x[46]))
        scale = 32 * EPS * (1.0 + float(lever))
        err = max(float(abs(mpm.mpf(float(g)) - r)) for g, r in zip(o[12:24], row))
        assert err <= scale, (err, scale, x)
        assert o[24] == float(z)
        worst = max(worst, err / scale)
    print(f"row: worst error / bound {worst:.3g}")


@pytest.mark.gpu
def test_device_measure_matches_host_and_oracle(hx):
    xs = measure_inputs() + _score_edge_inputs(hx)
    dev, host, orc = hx.eval("measure", xs, True), hx.eval("measure", xs, False), _oracle_measure(xs)
    for i in range(len(xs)):
        assert _same(dev[i], host[i]), (i, dev[i], host[i])
        assert _same(dev[i][:25], orc[i]), (i, dev[i][:25], orc[i])
