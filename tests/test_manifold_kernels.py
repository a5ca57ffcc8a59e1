"""lie.cuh against an extended-precision restatement of the reference's MTK formulas (tests/mtk_mp.py), on the host and on
the device, at the magnitudes and branch thresholds where the series and the exact forms meet.

Errors are measured in units of eps = 2^-52 of the result's max-norm, ||ref||_inf, or of a stated floor where the
reference's own formula cancels (the error is then relative to the magnitude of the terms, not of the result).

Bounds (derived from the operation counts; device sin / cos / atan / atan2 are within 2 ulps and glibc's within 1):
  cos_sinc_sqrt  4   series: three Horner-like steps, each adding <= 1 ulp to a sum of size ~1; exact: sqrt (1/2) +
                     sin or cos (2) + one division (1/2)
  so3_exp        6   cos_sinc_sqrt (4) + mult = sinc * 0.5 (exact) + mult * v (1/2)
  so3_log        8   series: r2 (2), eight alternating Horner steps dominated by the last (1), 2 / w, * p, * v (3 x 1/2);
                     exact: norm (2), nv / w (1/2), atan (2), 2 / nv, * atan, * v (3 x 1/2)
  A_matrix      16   series: ~2.  Exact branch, |v| >= 0.2: (1 - cos n) / n^2 cancels -- a 2-ulp cos error divided by n^2
                     and multiplied by |hat v| = n is 2 / n <= 10 ulps of ||A|| ~ 1; (1 - sin n / n) / n^2 times |hat v|^2
                     adds 2 more
  S2_Bx          4   one reciprocal, then two products and one subtraction per entry, * invL
  S2_boxplus    16   S2_Bx (4) -> B d (1) -> so3-type exp (6) -> toRotationMatrix (2) -> R v (2), |v| = L
  S2_boxminus    8   floor theta / v_sin * L^2: hat(other) self cancels for nearly aligned and nearly opposed vectors, an
                     absolute error of ~2 eps L^2 that f = theta / v_sin multiplies (~1 / L^2 when aligned, ~pi / v_sin
                     when opposed), whatever |result|; plus f itself (8 ulps)
  S2_Nx_yy       6   floor 1 / L: B^T hat(v) sums three products of size ~1, then * (1 / L / L)
  S2_Mx         24   floor L: A_matrix (16) times hat(v) B (2 x 3-term sums of size L)
  S2_congruence 32   floor 1: Nx (6) times Mx (24), 3-term sums
  state_boxplus 24   floor 1: the S2 block (16) and two quaternion products (4) on unit quaternions
  state_boxminus 16  per block, floor 1: the conjugate product of two unit quaternions rounds each component by ~2 eps
                     absolute, which the log carries through with a factor ~2; the gravity block as S2_boxminus, with its
                     own floor
"""
from __future__ import annotations

import math

import mpmath as mpm
import numpy as np
import pytest

import mtk_mp as R
from manifold_harness import Harness, compile_harness

EPS = 2.0 ** -52
TOL = 1e-11
L = R.L_D

BOUND = {"cos_sinc_sqrt": 4, "so3_exp": 6, "so3_log": 8, "A_matrix": 16, "S2_Bx": 4, "S2_boxplus": 16, "S2_boxminus": 8,
         "S2_Nx_yy": 6, "S2_Mx": 24, "S2_congruence": 32, "state_boxplus": 24, "state_boxminus": 16}
FLOOR = {"S2_Nx_yy": 1.0 / L, "S2_Mx": L, "S2_congruence": 1.0, "state_boxplus": 1.0, "state_boxminus": 1.0}
# device vs host on the branches that call sin / cos / atan / atan2: each call differs by <= 3 ulps of its value (2 + 1);
# carried through the formula with the amplification named above
DEV_HOST = {"cos_sinc_sqrt": 4, "so3_exp": 4, "so3_log": 6, "A_matrix": 16, "S2_boxplus": 8, "S2_boxminus": 6, "S2_Mx": 16,
            "S2_congruence": 20, "state_boxplus": 12, "state_boxminus": 8}
THRESHOLDS = [1.220703125e-4, 2.5e-3, 0.04, TOL * TOL]


@pytest.fixture(scope="module")
def hx(tmp_path_factory):
    return Harness(compile_harness(tmp_path_factory.mktemp("manifold_harness")))


# ------------------------------------------------------------------------------------------------ inputs
def _around(x, ks=(1, 2, 1000)):
    out = [x]
    for k in ks:
        up, dn = x, x
        for _ in range(k):
            up, dn = math.nextafter(up, math.inf), math.nextafter(dn, -math.inf)
        out += [up, dn]
    return out


def _unit(rng, n=3):
    v = rng.standard_normal(n)
    return v / np.linalg.norm(v)


def _mags(rng, k):
    return np.concatenate([10.0 ** rng.uniform(-12, 0.497, k), [1e-12, 1e-6, math.pi - 1e-6, 3.0, 0.2, 0.1, 0.022]])


def _quat(axis, angle, sign=1.0):
    s = math.sin(angle / 2)
    return [sign * axis[0] * s, sign * axis[1] * s, sign * axis[2] * s, sign * math.cos(angle / 2)]


def _s2(u):
    return list(np.asarray(u) / np.linalg.norm(u) * L)


def make_inputs(fn, seed=7, k=60):
    rng = np.random.default_rng(seed)
    th = [t for x in THRESHOLDS for t in _around(x)]
    if fn == "cos_sinc_sqrt":
        return [[x] for x in list(_mags(rng, k) ** 2) + th]
    if fn in ("so3_exp", "A_matrix"):
        sc = 2.0 if fn == "so3_exp" else 1.0          # so3_exp decides on |v/2|^2
        return [list(_unit(rng) * m) for m in _mags(rng, k)] + [list(_unit(rng) * math.sqrt(x) * sc) for x in th] + \
            [[math.sqrt(x) * sc, 0.0, 0.0] for x in th] + [[0.0, 0.0, 0.0]]
    if fn == "so3_log":
        qs = []
        for m in _mags(rng, k):
            a = _unit(rng)
            qs += [_quat(a, m), _quat(a, m, -1.0)]             # w > 0 and w < 0
        for r2 in th:                                           # r2 = nv^2 / w^2 at the thresholds
            a = _unit(rng)
            w = 1.0 / math.sqrt(1.0 + r2)
            qs += [list(a * math.sqrt(r2) * w) + [w], list(a * math.sqrt(r2) * w) + [-w]]
        qs += [list(_unit(rng)) + [0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0], [3e-12, 0.0, 0.0, 1.0]]
        return qs
    if fn in ("S2_Bx", "S2_Nx_yy"):
        vs = [_s2(_unit(rng)) for _ in range(k)] + [[L, 0.0, 0.0], [-L, 0.0, 0.0]]
        for d in (1e-13, 5e-12, 1e-11, 2e-11, 1e-9, 1e-6):      # near (-L, 0, 0), straddling v.x + L = MTK_TOL
            x = -L + d
            y = math.sqrt(max(L * L - x * x, 0.0))
            vs += [[x, y, 0.0], [x, 0.0, y], [x, y * 0.6, y * 0.8]]
        return vs
    if fn in ("S2_boxplus", "S2_Mx"):
        out = []
        for m in list(_mags(rng, k // 2)) + [TOL * 0.5, TOL, math.nextafter(TOL, 0), math.nextafter(TOL, 1), 2 * TOL, 0.0]:
            d = _unit(rng, 2) * m
            out.append(_s2(_unit(rng)) + list(d))
        out += [[-L + 1e-6, math.sqrt(L * L - (L - 1e-6) ** 2), 0.0, 0.3, -0.2], [L, 0.0, 0.0, 0.5, 0.5]]
        return out
    if fn == "S2_boxminus":
        out = []
        for m in _mags(rng, k):                                 # other rotated by m away from self
            s = _unit(rng)
            ax = np.cross(s, _unit(rng))
            ax /= np.linalg.norm(ax)
            o = _rot(ax, m) @ s
            out.append(_s2(s) + _s2(o))
        s = _unit(rng)
        out += [_s2(s) + _s2(s), _s2(s) + _s2(-s), _s2(s) + _s2(-s + 1e-9 * _unit(rng)), _s2(s) + _s2(-s + 1e-4 * _unit(rng))]
        for t2 in _around(2.5e-3):                             # tan^2 of the angle at the series threshold
            a = math.atan(math.sqrt(t2))
            ax = np.cross(s, [0.0, 0.0, 1.0])
            ax /= np.linalg.norm(ax)
            out.append(_s2(s) + _s2(_rot(ax, a) @ s))
        return out
    if fn == "S2_congruence":
        out = []
        for m in list(_mags(rng, k // 2)) + [TOL * 0.5, 2 * TOL]:
            g0 = _unit(rng)
            ax = np.cross(g0, _unit(rng))
            ax /= np.linalg.norm(ax)
            out.append(_s2(_rot(ax, min(m, 3.0)) @ g0) + _s2(g0) + list(_unit(rng, 2) * m))
        return out
    if fn in ("state_boxplus", "state_boxminus"):
        out = []
        for m in list(_mags(rng, k // 2)):
            x = _state(rng)
            if fn == "state_boxplus":
                d = rng.standard_normal(23) * 0.1
                d[3:6] = _unit(rng) * m
                d[6:9] = _unit(rng) * min(m, 1.0)
                d[21:23] = _unit(rng, 2) * m
                out.append(list(x) + list(d))
            else:
                y = _state(rng)
                y[3:7] = np.array(R.qmul([R.M(t) for t in x[3:7]], [R.M(t) for t in _quat(_unit(rng), m)]), dtype=float)
                y[7:11] = np.array(R.qmul([R.M(t) for t in x[7:11]], [R.M(t) for t in _quat(_unit(rng), m, -1.0)]), dtype=float)
                g = x[23:26] / L
                ax = np.cross(g, _unit(rng))
                y[23:26] = _s2(_rot(ax / np.linalg.norm(ax), min(m, 3.0)) @ g)
                out.append(list(y) + list(x))
        return out
    raise KeyError(fn)


def _rot(axis, ang):
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K


def _state(rng):
    x = rng.standard_normal(26)
    x[3:7] = _quat(_unit(rng), rng.uniform(0, 3))
    x[7:11] = _quat(_unit(rng), rng.uniform(0, 0.5))
    x[23:26] = _s2(_unit(rng))
    return x


# ------------------------------------------------------------------------------------------------ reference and branches
def reference(fn, x):
    x = [float(t) for t in x]
    if fn == "cos_sinc_sqrt":
        return list(R.cos_sinc_sqrt(x[0]))
    if fn in ("so3_exp", "so3_log", "A_matrix", "S2_Bx", "S2_Nx_yy"):
        return getattr(R, fn)(x)
    if fn in ("S2_boxplus", "S2_Mx"):
        return getattr(R, fn)(x[:3], x[3], x[4])
    if fn == "S2_boxminus":
        return R.S2_boxminus(x[:3], x[3:6])
    if fn == "S2_congruence":
        return R.S2_congruence(x[:3], x[3:6], x[6], x[7])
    if fn == "state_boxplus":
        return R.state_boxplus(x[:26], x[26:])
    return R.state_boxminus(x[:26], x[26:])


def transcendental(fn, x, host_bx=None):
    """Whether lie.cuh calls sin / cos / atan / atan2 on input x (its own branch tests, in double)."""
    def exp_x2(v):
        return 0.5 * 0.5 * (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) >= 1.220703125e-4

    def log_exact(q):
        nv2, ww = q[0] * q[0] + q[1] * q[1] + q[2] * q[2], q[3] * q[3]
        return ww == 0.0 or not (nv2 / ww < 2.5e-3) or nv2 < TOL * TOL

    def a_exact(v):
        return not (v[0] * v[0] + v[1] * v[1] + v[2] * v[2] < 0.04)

    def bm_exact(s, o):
        cr = R._cross_d(s, o)
        vs2, vc = R._dot_d(cr, cr), R._dot_d(s, o)
        return not (vs2 < TOL * TOL) and not (vc > 0.0 and vs2 / (vc * vc) < 2.5e-3)

    def bu(v, d0, d1):
        B = R.S2_Bx(v)
        return [float(B[0]) * d0 + float(B[1]) * d1, float(B[2]) * d0 + float(B[3]) * d1, float(B[4]) * d0 + float(B[5]) * d1]

    x = [float(t) for t in x]
    if fn == "cos_sinc_sqrt":
        return x[0] >= 1.220703125e-4
    if fn == "so3_exp":
        return exp_x2(x)
    if fn == "so3_log":
        return log_exact(x)
    if fn == "A_matrix":
        return a_exact(x)
    if fn in ("S2_Bx", "S2_Nx_yy"):
        return False
    if fn == "S2_boxplus":
        return exp_x2(bu(x[:3], x[3], x[4]))
    if fn == "S2_Mx":
        return a_exact(bu(x[:3], x[3], x[4]))
    if fn == "S2_congruence":
        return a_exact(bu(x[3:6], x[6], x[7]))
    if fn == "S2_boxminus":
        return bm_exact(x[:3], x[3:6])
    return True                                   # the compound state: decided per block; compared within DEV_HOST


def branch(fn, x):
    """The lie.cuh branch an input of `fn` takes, by name (for the coverage counts)."""
    x = [float(t) for t in x]
    if fn == "cos_sinc_sqrt":
        return "cos_sinc_exact" if x[0] >= 1.220703125e-4 else "series"
    if fn == "so3_exp":
        return "cos_sinc_exact" if transcendental(fn, x) else "series"
    if fn == "so3_log":
        nv2 = x[0] * x[0] + x[1] * x[1] + x[2] * x[2]
        if nv2 < TOL * TOL:
            return "so3_log_exact(clamp)"
        return "so3_log_exact" if transcendental(fn, x) else "series"
    if fn == "A_matrix":
        sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2]
        return "A_matrix_exact" if not sq < 0.04 else ("identity" if sq < TOL * TOL else "series")
    if fn in ("S2_Bx", "S2_Nx_yy"):
        return "regular" if x[0] + L > TOL else "degenerate"
    if fn == "S2_boxminus":
        cr = R._cross_d(x[:3], x[3:6])
        vs2, vc = R._dot_d(cr, cr), R._dot_d(x[:3], x[3:6])
        if vs2 < TOL * TOL:
            return "antipodal" if vc < 0.0 else "aligned"
        return "atan2" if transcendental(fn, x) else "series"
    if fn in ("S2_Mx", "S2_boxplus"):
        if fn == "S2_Mx" and not math.sqrt(x[3] * x[3] + x[4] * x[4]) < TOL:
            return "A_matrix_exact" if transcendental(fn, x) else "A_series"
        if fn == "S2_Mx":
            return "negligible_delta"
        return "cos_sinc_exact" if transcendental(fn, x) else "series"
    return "-"


def _boxminus_floor(s, o):
    cr = R._cross_d(s, o)
    v_sin = math.sqrt(R._dot_d(cr, cr))
    return math.atan2(v_sin, R._dot_d(s, o)) / v_sin * L * L if v_sin >= TOL else 1.0


def floor(fn, x):
    x = [float(t) for t in x]
    if fn == "S2_boxminus":
        return _boxminus_floor(x[:3], x[3:6])
    return FLOOR.get(fn, 0.0)


def ulps(fn, got, ref, x):
    if fn == "state_boxminus":                    # per block: the S2 floor applies to the gravity block alone
        x = [float(t) for t in x]
        return max(_ulps(got[:21], ref[:21], 1.0), _ulps(got[21:], ref[21:], max(1.0, _boxminus_floor(x[23:26], x[49:52]))))
    return _ulps(got, ref, floor(fn, x))


def _ulps(got, ref, floor_):
    ref_f = max(abs(t) for t in ref)
    scale = max(float(ref_f), floor_)
    if scale == 0.0:
        return 0.0 if all(g == 0.0 for g in got) else math.inf
    return float(max(abs(mpm.mpf(float(g)) - r) for g, r in zip(got, ref)) / scale) / EPS


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("fn", list(BOUND))
def test_host_within_bound_of_extended_precision(hx, fn):
    xs = make_inputs(fn)
    got = hx.eval(fn, xs, device=False)
    worst = max((ulps(fn, g, reference(fn, x), x), i) for i, (g, x) in enumerate(zip(got, xs)))
    assert worst[0] <= BOUND[fn], (fn, worst, xs[worst[1]])


@pytest.mark.gpu
@pytest.mark.parametrize("fn", list(BOUND))
def test_device_within_bound_of_extended_precision(hx, fn):
    xs = make_inputs(fn)
    got = hx.eval(fn, xs, device=True)
    worst = max((ulps(fn, g, reference(fn, x), x), i) for i, (g, x) in enumerate(zip(got, xs)))
    counts = {}
    for x in xs:
        counts[branch(fn, x)] = counts.get(branch(fn, x), 0) + 1
    print(f"{fn}: branches {counts}, worst {worst[0]:.2f} ulps")
    assert worst[0] <= BOUND[fn], (fn, worst, xs[worst[1]])


@pytest.mark.gpu
@pytest.mark.parametrize("fn", list(BOUND))
def test_device_matches_host(hx, fn):
    """Bit for bit where lie.cuh uses only + - * / sqrt (--fmad=false, correctly rounded / and sqrt); within DEV_HOST where
    it calls sin, cos, atan or atan2."""
    xs = make_inputs(fn)
    dev, host = hx.eval(fn, xs, device=True), hx.eval(fn, xs, device=False)
    trans = np.array([transcendental(fn, x) for x in xs])
    exact = ~trans
    assert np.array_equal(dev[exact].view(np.int64), host[exact].view(np.int64)), \
        [(xs[i], dev[i], host[i]) for i in np.nonzero(exact & np.any(dev != host, axis=1))[0][:3]]
    if trans.any():
        d = [ulps(fn, dv, [mpm.mpf(float(t)) for t in hv], x) for dv, hv, x in zip(dev[trans], host[trans], np.asarray(xs)[trans])]
        assert max(d) <= DEV_HOST[fn], (fn, max(d))


def test_inputs_reach_every_branch():
    """The generator reaches every branch of lie.cuh the functions have."""
    want = {"cos_sinc_sqrt": {"series", "cos_sinc_exact"}, "so3_exp": {"series", "cos_sinc_exact"},
            "so3_log": {"series", "so3_log_exact", "so3_log_exact(clamp)"}, "A_matrix": {"series", "A_matrix_exact", "identity"},
            "S2_Bx": {"regular", "degenerate"}, "S2_boxminus": {"series", "atan2", "aligned", "antipodal"},
            "S2_Mx": {"negligible_delta", "A_series", "A_matrix_exact"}, "S2_boxplus": {"series", "cos_sinc_exact"}}
    for fn, branches in want.items():
        assert {branch(fn, x) for x in make_inputs(fn)} == branches, fn


# ------------------------------------------------------------------------------------------------ the CPU oracle's restatement
ORACLE_FNS = ["so3_exp", "so3_log", "S2_Bx", "S2_boxminus", "S2_Nx_yy", "S2_Mx"]


def _oracle(fn, xs):
    import ctypes as C
    from oracle import bind
    L_ = bind.lib()
    f = getattr(L_, "oracle_" + fn)
    f.argtypes = [np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")] * 2
    f.restype = None
    nout = {"so3_exp": 4, "so3_log": 3, "S2_Bx": 6, "S2_boxminus": 2, "S2_Nx_yy": 6, "S2_Mx": 6}[fn]
    out = np.zeros((len(xs), nout))
    for i, x in enumerate(xs):
        o = np.zeros(nout)
        f(np.ascontiguousarray(x, dtype=np.float64), o)
        out[i] = o
    return out


# oracle (double, the reference's operation order) vs lie.cuh, in ulps of the result's max-norm.  S2_Bx, entry by entry:
# lie.cuh rounds r = 1 / (L + v.x), v.y * v.y, * r, L - yy, * invL and invL itself (<= 6 half-ulps, ~1.5 ulps of max|B|
# since the rounded terms are at most max|B| in size); the reference rounds L + v.x, v.y * v.y, / (L + v.x), L - ., / L
# (<= 5 half-ulps, ~1.25) -- apart by at most ~2.75, so 3.  Measured: 2.10 (host), the entries within 1.7 ulps of the exact
# value on both sides.  S2_Nx_yy and S2_Mx carry B through one more product and stay within the same 3.  The transcendental
# branches add the device's 2-ulp calls.
ORACLE_ULPS = {"S2_Bx": 3, "S2_Nx_yy": 3, "S2_Mx": 3, "so3_exp": 2, "so3_log": 2, "S2_boxminus": 2}


@pytest.mark.parametrize("fn", ORACLE_FNS)
def test_host_matches_oracle(hx, fn):
    xs = [x for x in make_inputs(fn) if not transcendental(fn, x)]
    host, orc = hx.eval(fn, xs, device=False), _oracle(fn, xs)
    d = max(ulps(fn, h, [mpm.mpf(float(t)) for t in o], x) for h, o, x in zip(host, orc, xs))
    assert d <= ORACLE_ULPS[fn], (fn, d)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ORACLE_FNS)
def test_device_matches_oracle(hx, fn):
    xs = make_inputs(fn)
    dev, orc = hx.eval(fn, xs, device=True), _oracle(fn, xs)
    trans = [transcendental(fn, x) for x in xs]
    d = [ulps(fn, h, [mpm.mpf(float(t)) for t in o], x) for h, o, x in zip(dev, orc, xs)]
    assert max([v for v, t in zip(d, trans) if not t] or [0.0]) <= ORACLE_ULPS[fn], (fn, d)
    assert max(d) <= ORACLE_ULPS[fn] + DEV_HOST.get(fn, 0), (fn, max(d))
