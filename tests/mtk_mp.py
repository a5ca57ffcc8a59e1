"""The MTK manifold arithmetic of the filter restated in extended precision (mpmath, 60 digits).

Each function follows the formula of the reference's IKFoM / MTK toolkit that fast_lio_b200/csrc/lie.cuh follows
(include/IKFoM_toolkit/mtk/src/mtkmath.hpp, types/SOn.hpp, types/S2.hpp, S2_typ = 1, length 98090/10000),
with its quirks: the identity exp(.., scalar(1/2)) in S2_Mx (T4), the periodic log that uses atan rather than
atan2 (T7), 3.1415926 for antipodal S2 vectors, the degenerate S2_Bx below v.x + L <= tolerance and the
MTK::tolerance clamps.  Branches are decided in double on the double inputs, as the reference decides them;
the chosen formula is then evaluated in mpmath at 60 digits (mpmath's working precision is set inside each public
function, not for the process).  Inputs are Python floats; results are lists of mpf.
"""
from __future__ import annotations

import functools
import math

import mpmath as mpm

DPS = 60

TOL = 1e-11                                   # MTK::tolerance<double>(), mtkmath.hpp:121
L_D = 98090.0 / 10000.0                       # use-ikfom.hpp:8 (the double the reference stores)
TAYLOR_N_BOUND = math.sqrt(math.sqrt(2.0 ** -52))   # mtkmath.hpp:148-150, = 2^-13


def M(x):
    return mpm.mpf(x)


def L():
    return M(L_D)


def _hat(v):                                  # mtkmath.hpp:178-185
    return [[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]]


def _mm(a, b):
    return [[sum(a[i][k] * b[k][j] for k in range(len(b))) for j in range(len(b[0]))] for i in range(len(a))]


def _mv(a, v):
    return [sum(a[i][k] * v[k] for k in range(len(v))) for i in range(len(a))]


def _tr(a):
    return [list(r) for r in zip(*a)]


def _dot_d(a, b):                             # double, left to right (the reference's branch inputs)
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross_d(a, b):                           # hat(a) * b in double
    return [-a[2] * b[1] + a[1] * b[2], a[2] * b[0] - a[0] * b[2], -a[1] * b[0] + a[0] * b[1]]


# ---------------------------------------------------------------- mtkmath.hpp
def cos_sinc_sqrt(x2):
    """mtkmath.hpp:142-176: (cos sqrt(x2), sin sqrt(x2) / sqrt(x2)); the Taylor branch is the 3-term series.
    `x2` is a double (the branch input) or, inside a composite formula, an mpf decided on its double value."""
    xd = float(x2)
    x2 = M(x2)
    if xd >= TAYLOR_N_BOUND:
        x = mpm.sqrt(x2)
        return mpm.cos(x), mpm.sin(x) / x
    c = 1 - x2 / 2 + x2 ** 2 / 24 - x2 ** 3 / 720
    s = 1 - x2 / 6 + x2 ** 2 / 120 - x2 ** 3 / 5040
    return c, s


def mtk_exp(v, scale):
    """mtkmath.hpp:249-256 -> (x, y, z, w)."""
    v = [M(t) for t in v]
    c, sinc = cos_sinc_sqrt(M(scale) ** 2 * sum(t * t for t in v))
    mult = sinc * M(scale)
    return [mult * v[0], mult * v[1], mult * v[2], c]


def so3_exp(v):                               # SOn.hpp:284-288: exp(dvec, scale = 1) -> MTK::exp(.., scale / 2)
    return mtk_exp(v, 0.5)


def so3_log(q):
    """SOn.hpp:293-297 -> mtkmath.hpp:268-288 with scale 2 and plus_minus_periodicity = true (T7): atan, not atan2."""
    nv_d = math.sqrt(_dot_d(q[:3], q[:3]))
    v = [M(t) for t in q[:3]]
    w = M(q[3])
    nv = M(TOL) if nv_d < TOL else mpm.sqrt(sum(t * t for t in v))
    if q[3] == 0.0:                           # nv / w = +-inf in double: atan -> +-pi/2
        at = mpm.pi / 2 if math.copysign(1.0, q[3]) > 0 else -mpm.pi / 2
    else:
        at = mpm.atan(nv / w)
    s = 2 / nv * at
    return [s * t for t in v]


def A_matrix(v):
    """mtkmath.hpp:235-248, row-major 9."""
    n_d = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if n_d < TOL:
        return [M(1) if i % 4 == 0 else M(0) for i in range(9)]
    return _A_exact([M(t) for t in v])


def _A_matrix_mp(v):                          # A_matrix of an intermediate, decided on its double value
    return A_matrix([float(t) for t in v]) if math.sqrt(sum(float(t) ** 2 for t in v)) < TOL else _A_exact(v)


def _A_exact(v):
    sq = sum(t * t for t in v)
    n = mpm.sqrt(sq)
    h = _hat(v)
    hh = _mm(h, h)
    a, b = (1 - mpm.cos(n)) / sq, (1 - mpm.sin(n) / n) / sq
    return [(1 if i == j else 0) + a * h[i][j] + b * hh[i][j] for i in range(3) for j in range(3)]


def qmat(q):                                  # Eigen QuaternionBase::toRotationMatrix
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def qmul(a, b):                               # Eigen quat_product, (x, y, z, w)
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz]


# ---------------------------------------------------------------- S2.hpp, S2_typ = 1
def S2_Bx(v):
    """S2.hpp:214-239, 3x2 row-major 6."""
    if v[0] + L_D > TOL:
        x, y, z = (M(t) for t in v)
        Ln = L()
        r = [-y, -z, Ln - y * y / (Ln + x), -z * y / (Ln + x), -z * y / (Ln + x), Ln - z * z / (Ln + x)]
        return [t / Ln for t in r]
    return [M(0), M(0), M(0), M(-1), M(1), M(0)]


def _Bmat(B):
    return [[B[0], B[1]], [B[2], B[3]], [B[4], B[5]]]


def S2_boxplus(v, d0, d1):
    """S2.hpp:136-142: exp(Bx delta, 1/2) applied to v."""
    B = _Bmat(S2_Bx(v))
    Bu = _mv(B, [M(d0), M(d1)])
    return _mv(qmat(mtk_exp(Bu, 0.5)), [M(t) for t in v])


def S2_boxminus(s, o):
    """S2.hpp:144-167: self [-] other."""
    v_sin_d = math.sqrt(_dot_d(_cross_d(s, o), _cross_d(s, o)))
    v_cos_d = _dot_d(s, o)
    theta_d = math.atan2(v_sin_d, v_cos_d)
    if v_sin_d < TOL:
        return [M(3.1415926), M(0)] if abs(theta_d) > TOL else [M(0), M(0)]
    sm, om = [M(t) for t in s], [M(t) for t in o]
    cr = _mv(_hat(sm), om)
    v_sin = mpm.sqrt(sum(t * t for t in cr))
    v_cos = sum(a * b for a, b in zip(sm, om))
    theta = mpm.atan2(v_sin, v_cos)
    hv = _mv(_hat(om), sm)
    r = _mv(_tr(_Bmat(S2_Bx(o))), hv)
    return [theta / v_sin * t for t in r]


def S2_Nx_yy(v):
    """S2.hpp:262-267: 1/L/L * Bx^T hat(v), 2x3 row-major 6."""
    N = _mm(_tr(_Bmat(S2_Bx(v))), _hat([M(t) for t in v]))
    return [N[i][j] / L() / L() for i in range(2) for j in range(3)]


def S2_Mx(v, d0, d1):
    """S2.hpp:269-281, 3x2 row-major 6.  T4: exp(Bu, scalar(1/2)) has scale 0 -- the identity rotation."""
    B = _Bmat(S2_Bx(v))
    h = _hat([M(t) for t in v])
    if math.sqrt(d0 * d0 + d1 * d1) < TOL:
        T = h
    else:
        Bu = _mv(B, [M(d0), M(d1)])
        A = _A_matrix_mp(Bu)
        T = _mm(h, _tr([A[0:3], A[3:6], A[6:9]]))
    R = _mm(T, B)
    return [-R[i][j] for i in range(3) for j in range(2)]


def S2_congruence(g_now, g_prop, d0, d1):
    """esekfom.hpp:1686-1690: Nx(x.grav) * Mx(x_prop.grav, delta), 2x2."""
    N, Mx = S2_Nx_yy(g_now), S2_Mx(g_prop, d0, d1)
    return [sum(N[i * 3 + k] * Mx[k * 2 + j] for k in range(3)) for i in range(2) for j in range(2)]


# ---------------------------------------------------------------- the compound state, build_manifold.hpp:192-200
def state_boxplus(x, d):
    x = [M(t) for t in x]
    r = list(x)
    for i in range(3):
        for xo, do in ((0, 0), (11, 9), (14, 12), (17, 15), (20, 18)):
            r[xo + i] = x[xo + i] + M(d[do + i])
    r[3:7] = qmul(x[3:7], so3_exp(d[3:6]))
    r[7:11] = qmul(x[7:11], so3_exp(d[6:9]))
    r[23:26] = S2_boxplus([float(t) for t in x[23:26]], d[21], d[22])
    return r


def state_boxminus(a, b):
    r = [M(0)] * 23
    for i in range(3):
        for xo, do in ((0, 0), (11, 9), (14, 12), (17, 15), (20, 18)):
            r[do + i] = M(a[xo + i]) - M(b[xo + i])
    for xo, do in ((3, 3), (7, 6)):
        q = qmul([M(-t) for t in b[xo:xo + 3]] + [M(b[xo + 3])], [M(t) for t in a[xo:xo + 4]])
        # the reference logs the double product; its branch decision is taken on that product's rounding
        r[do:do + 3] = _so3_log_mp(q)
    r[21:23] = S2_boxminus(a[23:26], b[23:26])
    return r


def _so3_log_mp(q):
    nv = mpm.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2)
    if float(nv) < TOL:
        nv = M(TOL)
    s = 2 / nv * mpm.atan(nv / q[3])
    return [s * t for t in q[:3]]


def _at_dps(f):
    @functools.wraps(f)
    def g(*a, **k):
        with mpm.workdps(DPS):
            return f(*a, **k)
    return g


for _name in ("cos_sinc_sqrt", "mtk_exp", "so3_exp", "so3_log", "A_matrix", "qmat", "qmul", "S2_Bx", "S2_boxplus", "S2_boxminus",
              "S2_Nx_yy", "S2_Mx", "S2_congruence", "state_boxplus", "state_boxminus"):
    globals()[_name] = _at_dps(globals()[_name])
