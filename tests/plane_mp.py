"""The per-point measurement model restated in extended precision (mpmath, 60 digits): the exact least-squares plane of
five float neighbours and the Jacobian row of laserMapping.cpp:723-751 with the quaternion formulas lie.cuh takes from
Eigen (_transformVector, toRotationMatrix).  Inputs are the floats / doubles the kernels see; results are mpf.
"""
from __future__ import annotations

import mpmath as mpm

DPS = 60


def plane_exact(pts):
    """Least squares A x = -1 (A = the 5 x 3 points) by Householder QR at 60 digits; returns (x, pd2) with pd2[j] the signed
    distance of point j from the normalised plane n = x / |x|, d = 1 / |x| (common_lib.h:243-256)."""
    with mpm.workdps(DPS):
        A = mpm.matrix([[mpm.mpf(float(c)) for c in p] for p in pts])
        x, _ = mpm.qr_solve(A, mpm.matrix([-1] * len(pts)))
        nx = mpm.sqrt(sum(x[i] ** 2 for i in range(3)))
        pd2 = [(sum(A[j, i] * x[i] for i in range(3)) + 1) / nx for j in range(len(pts))]
        return [x[i] for i in range(3)], pd2


def at_plane(pabcd, p):
    """pabcd . (p, 1) evaluated exactly from the float coefficients."""
    with mpm.workdps(DPS):
        return sum(mpm.mpf(float(pabcd[i])) * mpm.mpf(float(p[i])) for i in range(3)) + mpm.mpf(float(pabcd[3]))


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _qrot(q, v):                                # Eigen _transformVector, exact in mp
    qv = q[:3]
    uv = _cross(qv, v)
    uv = [2 * t for t in uv]
    c = _cross(qv, uv)
    return [v[i] + q[3] * uv[i] + c[i] for i in range(3)]


def _qmat(q):                                   # Eigen toRotationMatrix
    x, y, z, w = q
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
            [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
            [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]


def _mv(m, v):
    return [sum(m[i][k] * v[k] for k in range(3)) for i in range(3)]


def _hat(v):
    return [[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]]


def jacobian_row(x26, pb, nv, extr):
    """Row (12) and z of laserMapping.cpp:723-751 for the flat state x26, body point pb and normvec nv = (n, pd2), and the
    largest lever arm the row multiplies: max |p_this|, |p_be| (p_be enters the extrinsic block)."""
    with mpm.workdps(DPS):
        M = lambda t: mpm.mpf(float(t))
        rot = [M(t) for t in x26[3:7]]
        offR = [M(t) for t in x26[7:11]]
        offT = [M(t) for t in x26[11:14]]
        p_be = [M(t) for t in pb]
        p_this = [a + b for a, b in zip(_qrot(offR, p_be), offT)]
        n = [M(t) for t in nv[:3]]
        C = _qrot([-rot[0], -rot[1], -rot[2], rot[3]], n)
        A = _mv(_hat(p_this), C)
        row = n + A + [mpm.mpf(0)] * 6
        if extr:
            R = _qmat([-offR[0], -offR[1], -offR[2], offR[3]])
            H = _hat(p_be)
            HR = [[sum(H[i][k] * R[k][j] for k in range(3)) for j in range(3)] for i in range(3)]
            row[6:9] = _mv(HR, C)
            row[9:12] = C
        return row, -M(nv[3]), max(abs(t) for t in p_this + p_be)
