"""The Gauss-Jordan routines of gj.cuh against extended precision, on the shapes the update solves: the 23 x 46 inverse,
the small-m systems (mr = 1..22 rows, ld = mr + 13) and the 6 x 13 / 12 x 25 lemma systems [I + H^T H P11 / R | H^T h | H^T H].

Forward error:  ||X - X*||_inf <= C n kappa_inf(A) eps ||X*||_inf  with C = 4 (Gauss-Jordan with partial pivoting has
the forward error of LU with partial pivoting times a small constant; the systems here have no element growth to speak of).
"""
from __future__ import annotations

import functools

import mpmath as mpm
import numpy as np
import pytest

from manifold_harness import Harness, compile_harness

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52
C = 4
THREADS = [32, 64, 160, 192, 256, 512]
KINDS = ["random", "graded", "cond1e2", "cond1e6", "cond1e10", "zero_pivot", "single_row", "singular"]


@pytest.fixture(scope="module")
def hx(tmp_path_factory):
    return Harness(compile_harness(tmp_path_factory.mktemp("gj_harness")))


def _cond(rng, n, kappa):
    u, _ = np.linalg.qr(rng.standard_normal((n, n)))
    v, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return u @ np.diag(np.logspace(0, -np.log10(kappa), n)) @ v.T


def make_system(kind, n, m, seed):
    """[A | B], n x (n + m)."""
    rng = np.random.default_rng(seed)
    B = rng.standard_normal((n, m))
    if kind == "random":
        A = rng.standard_normal((n, n)) + 2 * np.sqrt(n) * np.eye(n)
    elif kind == "graded":                                   # rows of P mix metres and radians
        g = np.where(np.arange(n) < min(6, n), 1e5, 1.0)
        A = (rng.uniform(-0.5, 0.5, (n, n)) + 3 * np.eye(n)) * g[:, None]
        B = B * g[:, None]
    elif kind.startswith("cond"):
        A = _cond(rng, n, float(kind[4:])) if n > 1 else np.array([[1.0]])
    elif kind == "zero_pivot":
        A = rng.standard_normal((n, n)) + 2 * np.sqrt(n) * np.eye(n)
        A[0, 0] = 0.0
        if n == 1:
            A[0, 0] = 1.0                                    # a 1 x 1 system with a zero pivot is singular
    elif kind == "single_row":                               # I + h^T h P11 / R from one Jacobian row (m = 1)
        h = rng.standard_normal(n)
        P = _cond(rng, n, 1e3)
        P = P @ P.T * 1e-4
        A = np.eye(n) + np.outer(h, h) @ P / 0.001
    elif kind == "singular":
        A = rng.standard_normal((n, n))
        A[:, n // 2] = 0.0
    return np.hstack([A, B])


@functools.lru_cache(maxsize=None)
def _reference(kind, n, m, seed):
    S = make_system(kind, n, m, seed)
    with mpm.workdps(50):
        A = mpm.matrix(S[:, :n].tolist())
        Ai = mpm.inverse(A)
        X = Ai * mpm.matrix(S[:, n:].tolist())
        nrm = lambda M: max(sum(abs(M[i, j]) for j in range(M.cols)) for i in range(M.rows))
        kappa = float(nrm(A) * nrm(Ai))
        return np.array(X.tolist(), dtype=float), kappa, X


def check(hx, variant, n, m, threads, kinds=KINDS, seeds=(1, 2)):
    cases = [(k, s) for k in kinds for s in seeds]
    systems = np.stack([make_system(k, n, m, s) for k, s in cases])
    X, rmap, ok = hx.gj(variant, systems, n, n + m, threads)
    for (kind, seed), x, r, o in zip(cases, X, rmap, ok):
        tag = (variant, n, m, threads, kind, seed)
        if kind == "singular":
            assert not o, tag
            continue
        assert o, tag
        assert sorted(r.tolist()) == list(range(n)), (tag, r)
        xr, kappa, xm = _reference(kind, n, m, seed)
        err = max(abs(mpm.mpf(float(x[i, j])) - xm[i, j]) for i in range(n) for j in range(m))
        bound = C * n * kappa * EPS * np.abs(xr).max()
        assert err <= bound, (tag, float(err), bound, kappa)


@pytest.mark.parametrize("threads", THREADS)
def test_gj_eliminate_inverse_23(hx, threads):
    """The 23 x 46 system [P / R | I] (solver 0) at every block size, including 160 threads (5 warps: warp 0 owns five rows)."""
    check(hx, "gj_eliminate", 23, 23, threads)


@pytest.mark.parametrize("threads", THREADS)
def test_gj_eliminate_small_m(hx, threads):
    """[H P H^T / R + I | h_x | h] of the small-m gain, mr = 1..22 rows, 13 right-hand sides."""
    for mr in range(1, 23):
        check(hx, "gj_eliminate", mr, 13, threads, seeds=(mr,))


@pytest.mark.parametrize("variant, n", [("gj_eliminate", 6), ("gj_eliminate", 12), ("gj_warp", 6), ("gj_warp", 12),
                                        ("gj_warp_reg6", 6), ("gj_warp_reg12", 12), ("gj_cols6", 6), ("gj_cols12", 12)])
def test_lemma_systems(hx, variant, n):
    """[I + H^T H P11 / R | H^T h | H^T H] of the one-right-hand-side lemma form, ne = 6 and 12."""
    check(hx, variant, n, n + 1, 32 if variant != "gj_eliminate" else 256)


def test_gj_eliminate_160_equals_256(hx):
    """The update at any block size computes the same numbers: the elimination order does not depend on blockDim."""
    systems = np.stack([make_system(k, 23, 23, s) for k in KINDS[:-1] for s in (1, 2)])
    a = hx.gj("gj_eliminate", systems, 23, 46, 160)
    for t in (32, 64, 192, 256, 512):
        b = hx.gj("gj_eliminate", systems, 23, 46, t)
        assert np.array_equal(a[0].view(np.int64), b[0].view(np.int64)) and np.array_equal(a[1], b[1]), t
