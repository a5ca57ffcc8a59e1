"""CPU: the map's maintenance rules (fast_lio_b200/csrc/map_rules.h), run through a g++-built harness
(tests/kernels/map_rules_harness.cpp), equal every copy of them the host forms and the device forms' one-thread kernels
carried before they were gathered there (fast_lio_b200/csrc/map.cu at commit 0084864; the lines are cited below): the
overflow-chain limit, re-pack due, re-list due, the headroom of a batch, and the growth after a directory error and for a
batch.  Boundary inputs (the 64 and 1024 thresholds, exactly 90 % table load, leaf_used + n == leaf_cap, n_main 1, counts
near INT_MAX) and a seeded random sweep, over the inputs the callers can pass."""
from __future__ import annotations

import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "kernels", "map_rules_harness.cpp")

INT_MAX = 2**31 - 1
UINT_MAX = 2**32 - 1
LEAF = 32                                  # slots per leaf (map.cuh)
LEAF_LIMIT = 0x7fffffff // LEAF            # Map::ensure_capacity refuses more leaves than this (map.cu:1250-1251)
HALO_NEW_CAP = 64                          # map.cuh:43
FRAC = 0.05                                # Map::rebuild_overflow_frac_ (map.h:122), the only value the map uses
SWEEP = 4000


# ------------------------------------------------------------------------------------------------ C arithmetic
def i32(v):
    """An int expression.  Signed overflow is undefined in C, so no input of a copy may cause it."""
    assert -2**31 <= v <= INT_MAX, v
    return v


def i64(v):
    assert -2**63 <= v < 2**63, v
    return v


def u64(v):
    """A size_t expression: arithmetic modulo 2^64."""
    return v % 2**64


def cdiv(a, b):
    """C's integer division, truncating toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def f32_times_int(frac, n):
    """(int)(float * int): the int converted to float, a float product (no excess precision on x86-64 or the GPU), truncated."""
    p = np.float32(frac) * np.float32(n)
    assert abs(float(p)) < 2**31
    return int(p)


# ------------------------------------------------------------------------------------------------ the copies at 0084864
def chain_limit_0084864(frac, n_main):
    """std::max(64, (int)(rebuild_overflow_frac_ * v_.n_main)), the same text in Map::maybe_rebuild (map.cu:1930),
    Map::enqueue_delete (map.cu:1525, the argument of k_delete_account) and Map::enqueue_add (map.cu:2196, of k_async_account)."""
    return max(64, f32_times_int(frac, n_main))


CHAIN_LIMIT = {"maybe_rebuild map.cu:1930": chain_limit_0084864, "enqueue_delete map.cu:1525": chain_limit_0084864,
               "enqueue_add map.cu:2196": chain_limit_0084864}


def repack_maybe_rebuild(leaf_used, n_main, frac, tombs, valid):
    """Map::maybe_rebuild, map.cu:1929-1932."""
    overflow = i32(leaf_used - n_main)
    too_chained = overflow > max(64, f32_times_int(frac, n_main))
    too_sparse = tombs > 1024 and tombs > valid
    return too_chained or too_sparse


def repack_k_delete_account(leaf_used, n_main, frac, tombs, valid):
    """k_delete_account, map.cu:573-574, its chain_limit from Map::enqueue_delete, map.cu:1525."""
    chain_limit = chain_limit_0084864(frac, n_main)
    return (tombs > 1024 and tombs > valid) or i32(leaf_used - n_main) > chain_limit


def repack_k_async_account(leaf_used, n_main, frac, tombs, valid):
    """k_async_account, map.cu:967-968, less the `|| counters[C_ERROR]` it ORs in; chain_limit from Map::enqueue_add, :2196."""
    chain_limit = chain_limit_0084864(frac, n_main)
    return i32(leaf_used - n_main) > chain_limit or (tombs > 1024 and tombs > valid)


REPACK = {"maybe_rebuild map.cu:1929": repack_maybe_rebuild, "k_delete_account map.cu:573": repack_k_delete_account,
          "k_async_account map.cu:967": repack_k_async_account}


def relist_host(dir_error, crowded, cells):
    """Map::insert_device, map.cu:1970-1975, and Map::settle, map.cu:2061-2066 (the same text):
    crowded = C_DIR_CROWDED > std::max(64, C_DIR_CELLS / 1024), then C_DIR_ERROR || crowded."""
    is_crowded = crowded > max(64, cdiv(cells, 1024))
    return bool(dir_error) or is_crowded


def relist_k_async_account(dir_error, crowded, cells):
    """k_async_account, map.cu:965: C_DIR_ERROR || C_DIR_CROWDED > max(64, C_DIR_CELLS / 1024)."""
    return bool(dir_error) or crowded > max(64, cdiv(cells, 1024))


RELIST = {"insert_device map.cu:1970": relist_host, "settle map.cu:2061": relist_host,
          "k_async_account map.cu:965": relist_k_async_account}


def fits_insert_device(leaf_used, leaf_cap, cells, cap, n):
    """Map::insert_device, map.cu:1939 and 1943-1947 (n an int): (no re-pack, no re-list) before the inserts."""
    leaves = not i64(leaf_used + n) > leaf_cap
    if not cap:
        return leaves, True
    c = u64(u64(cells) + u64(n * 27))
    return leaves, not u64(c * 10) > u64(cap * 9)


def fits_async_grow(leaf_used, leaf_cap, cells, cap, n):
    """Map::async_grow, map.cu:2096-2097 and 2101-2103, for its n = std::max(n_max, 1) >= 1."""
    leaves = not i64(leaf_used + n) > leaf_cap
    if not cap:
        return leaves, True
    c = i64(cells + 27 * n)
    return leaves, not i64(c * 10) > i64(cap * 9)


def fits_async_fits(leaf_used, leaf_cap, cells, cap, n):
    """Map::async_fits, map.cu:2087-2089, for its n = ub_n_ + n_max."""
    if i64(leaf_used + n) > leaf_cap:
        return False
    return not cap or i64(i64(cells + 27 * n) * 10) <= i64(cap * 9)


def fits_k_plan(leaf_used, leaf_cap, cells, cap, n):
    """k_plan, map.cu:935-938, for its n = C_RA + C_RB (the list-pool check that follows is the plan's own)."""
    ok = i64(leaf_used + n) <= leaf_cap
    if cap:
        ok = ok and i64(i64(cells + 27 * n) * 10) <= i64(cap * 9)
    return ok


def grow_insert_device(min_pool, min_cap, cells, n):
    """Map::insert_device, map.cu:1940 and 1946-1948: min_pool_ (no clamp, n + 1024 in int) and dir_min_cap_."""
    pool = max(min_pool, i32(n + 1024))
    c = u64(u64(cells) + u64(n * 27))
    return pool, max(min_cap, u64(c * 2 + 16384))


def grow_async_grow(min_pool, min_cap, cells, n):
    """Map::async_grow, map.cu:2098, 2102 and 2106."""
    pool = min(max(min_pool, n + 1024), INT_MAX // 2)
    c = i64(cells + 27 * n)
    return pool, max(min_cap, u64(u64(c) * 2 + 16384))


def after_error_host(min_cap, min_pool, cap):
    """Map::insert_device, map.cu:1971-1974, and Map::settle, map.cu:2062-2065 (the same text)."""
    return max(min_cap, u64(cap + cap // 2)), max(u64(min_pool * 2), HALO_NEW_CAP * 262144)


def pool_build_directory(min_pool):
    """Map::build_directory, map.cu:1391: the list pool after the re-list itself ran out of it."""
    return max(u64(min_pool * 2), HALO_NEW_CAP * 262144)


def pool_async_grow(min_pool, need):
    """Map::async_grow, map.cu:2104 and 2107: the list pool after a refused call, need = max(C_NEED, 0)."""
    return max(u64(min_pool * 2), u64(2 * need))


# ------------------------------------------------------------------------------------------------ harness
@pytest.fixture(scope="module")
def rules(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("map_rules") / "libmap_rules.so")
    res = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC", SRC, "-o", out],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    lib = C.CDLL(out)
    i, ll, sz = C.c_int, C.c_longlong, C.c_size_t
    sig = {"mr_chain_limit": ([C.c_float, i], i), "mr_repack_due": ([i] * 5, i), "mr_relist_due": ([i] * 3, i),
           "mr_leaves_fit": ([ll] * 3, i), "mr_table_fits": ([ll] * 3, i), "mr_batch_fits": ([ll] * 5, i),
           "mr_pool_min_for_batch": ([i, ll], i), "mr_dir_cap_min_for_batch": ([sz, ll, ll], sz),
           "mr_dir_cap_min_after_error": ([sz, sz], sz), "mr_list_pool_min_grown": ([sz, sz], sz)}
    for name, (args, res_t) in sig.items():
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = res_t
    return lib


def _near(*centres, lo=0, hi=INT_MAX, d=(-1, 0, 1)):
    return sorted({c + k for c in centres for k in d if lo <= c + k <= hi})


def _draw(rng, lo, hi, size):
    """Half uniform on [lo, hi], half log-uniform, so small and large magnitudes both come up (hi < 2^63)."""
    u = rng.integers(lo, hi, size=size, endpoint=True)
    g = np.exp(rng.uniform(0, np.log(hi - lo + 1), size=size))
    return [int(a) if p else min(hi, lo + int(b) - 1) for a, b, p in zip(u, g, rng.random(size) < 0.5)]


def _frac(rng, size):
    return [FRAC if r < 0.5 else float(np.float32(f)) for r, f in zip(rng.random(size), rng.uniform(0, 1, size))]


# ------------------------------------------------------------------------------------------------ tests
def test_chain_limit(rules):
    fracs = [FRAC, 0.0, 0.01, 0.5, 1.0]
    n_mains = {1, 2, 63, 64, 65, LEAF_LIMIT - 1, LEAF_LIMIT}
    for f in fracs:                               # where (int)(f * n_main) passes 64
        if f > 0:
            n_mains.update(_near(int(64 / f), int(65 / f), lo=1, hi=LEAF_LIMIT, d=range(-2, 3)))
    rng = np.random.default_rng(1)
    cases = list(itertools.product(fracs, sorted(n_mains))) + list(zip(_frac(rng, SWEEP), _draw(rng, 1, LEAF_LIMIT, SWEEP)))
    for name, copy in CHAIN_LIMIT.items():
        for f, n_main in cases:
            assert rules.mr_chain_limit(f, n_main) == copy(f, n_main), (name, f, n_main)
    assert rules.mr_chain_limit(FRAC, 1280) == 64 and rules.mr_chain_limit(FRAC, 1300) == 65


def test_repack_due(rules):
    """The chain limit of the map's own fraction and of others, each side of it; tombs each side of 1024 and of valid."""
    cases = []
    for f, n_main in itertools.product([FRAC, 0.5], [1, 1300, 20000, LEAF_LIMIT // 2]):
        lim = chain_limit_0084864(f, n_main)
        for over in _near(lim, 0, hi=LEAF_LIMIT):
            if n_main + over <= LEAF_LIMIT:
                cases += [(n_main + over, n_main, f, t, v) for t in (0, 1024, 1025)
                          for v in (0, t - 1, t, t + 1) if v >= 0]
    for tombs in _near(1024, 2048, INT_MAX - 1):
        cases += [(1, 1, FRAC, tombs, v) for v in _near(tombs, 0, 1024, INT_MAX)]
    cases += [(0, 1, FRAC, INT_MAX, INT_MAX), (LEAF_LIMIT, 1, FRAC, 0, 0), (0, LEAF_LIMIT, FRAC, 0, 0)]
    rng = np.random.default_rng(2)
    n_main = _draw(rng, 1, LEAF_LIMIT, SWEEP)
    over = [int(v) for v in rng.integers(-100, 5000, SWEEP)]
    leaf_used = [min(max(m + o, 0), LEAF_LIMIT) for m, o in zip(n_main, over)]
    cases += list(zip(leaf_used, n_main, _frac(rng, SWEEP), _draw(rng, 0, INT_MAX, SWEEP), _draw(rng, 0, INT_MAX, SWEEP)))
    seen = set()
    for name, copy in REPACK.items():
        for leaf_used, n_main, f, tombs, valid in cases:
            got = rules.mr_repack_due(leaf_used, n_main, rules.mr_chain_limit(f, n_main), tombs, valid)
            assert bool(got) == copy(leaf_used, n_main, f, tombs, valid), (name, leaf_used, n_main, f, tombs, valid)
            seen.add(bool(got))
    assert seen == {False, True}


def test_relist_due(rules):
    """Cells each side of 64 * 1024 (where cells / 1024 passes 64) and of every multiple of 1024 tried, crowded each side of
    the limit, with and without a directory error."""
    cases = []
    for cells in _near(0, 1023, 1024, 65535, 65536, 66559, 66560, 2**20, INT_MAX - 1024, INT_MAX):
        lim = max(64, cells // 1024)
        cases += [(e, c, cells) for e in (0, 1) for c in _near(0, lim, INT_MAX)]
    rng = np.random.default_rng(3)
    cells = _draw(rng, 0, INT_MAX, SWEEP)
    crowded = [max(0, min(INT_MAX, max(64, c // 1024) + int(d))) for c, d in zip(cells, rng.integers(-3, 4, SWEEP))]
    crowded[::3] = _draw(rng, 0, INT_MAX, len(crowded[::3]))
    cases += list(zip([int(v) for v in rng.integers(0, 2, SWEEP)], crowded, cells))
    for name, copy in RELIST.items():
        for e, c, cells in cases:
            assert bool(rules.mr_relist_due(e, c, cells)) == copy(e, c, cells), (name, e, c, cells)


def _fit_cases(rng, n_hi):
    """(leaf_used, leaf_cap, cells, cap, n): leaf_used + n == leaf_cap +- 1, (cells + 27 n) * 10 == cap * 9 +- 1 and +- 10
    (exactly 90 % load), no directory, and counts near INT_MAX; then a sweep with n in [1, n_hi]."""
    cases = []
    for n in (1, 2, 1000, INT_MAX // 27, INT_MAX - 1, INT_MAX, n_hi):
        if n > n_hi:
            continue
        for leaf_cap in (1, 65536 + 1, LEAF_LIMIT):
            cases += [(u, leaf_cap, 0, 0, n) for u in _near(leaf_cap - n, 0, hi=leaf_cap)]
        for cells in (0, 5, 65536, INT_MAX):
            load = cells + 27 * n                     # cap * 9 == load * 10 when cap = load * 10 / 9
            for cap in _near(load * 10 // 9, (load * 10 + 8) // 9, hi=UINT_MAX, d=range(-2, 3)):
                cases += [(0, LEAF_LIMIT, cells, cap, n)]
            cases += [(0, LEAF_LIMIT, cells, 0, n), (0, LEAF_LIMIT, cells, UINT_MAX, n)]
    m = SWEEP
    n = _draw(rng, 1, n_hi, m)
    leaf_cap = _draw(rng, 1, LEAF_LIMIT, m)
    leaf_used = [max(0, min(c, c - k + int(d))) for c, k, d in zip(leaf_cap, n, rng.integers(-5, 5, m))]
    leaf_used[::2] = [min(u, c) for u, c in zip(_draw(rng, 0, LEAF_LIMIT, len(leaf_used[::2])), leaf_cap[::2])]
    cells = _draw(rng, 0, INT_MAX, m)
    cap = [min(UINT_MAX, (c + 27 * k) * 10 // 9 + int(d)) for c, k, d in zip(cells, n, rng.integers(-3, 4, m))]
    cap[::2] = _draw(rng, 0, UINT_MAX, len(cap[::2]))
    cap[::7] = [0] * len(cap[::7])
    return cases + list(zip(leaf_used, leaf_cap, cells, cap, n))


def test_batch_fits(rules):
    rng = np.random.default_rng(4)
    seen = set()
    # insert_device (n an int) and async_grow (n = max(n_max, 1), n_max an int): the two parts, each deciding a growth
    for name, copy in (("insert_device map.cu:1939", fits_insert_device), ("async_grow map.cu:2097", fits_async_grow)):
        for case in _fit_cases(rng, INT_MAX):
            leaf_used, leaf_cap, cells, cap, n = case
            got = (bool(rules.mr_leaves_fit(leaf_used, leaf_cap, n)), bool(rules.mr_table_fits(cells, cap, n)))
            assert got == copy(*case), (name, case)
            seen.add(got)
    # async_fits (n = ub_n_ + n_max, every device-form call since the last settle and this one) and k_plan (two lists)
    for name, copy, n_hi in (("async_fits map.cu:2087", fits_async_fits, 2**40), ("k_plan map.cu:935", fits_k_plan, 2 * INT_MAX)):
        for case in _fit_cases(rng, n_hi):
            assert bool(rules.mr_batch_fits(*case)) == copy(*case), (name, case)
    assert seen == set(itertools.product((False, True), repeat=2))


def _grow_cases(rng, n_hi):
    cases = []
    for n in _near(1, INT_MAX // 2 - 1024, LEAF_LIMIT - 1024, INT_MAX - 1024, lo=1, hi=n_hi):
        for min_pool in (65536, n + 1023, n + 1024, n + 1025, LEAF_LIMIT, INT_MAX // 2, INT_MAX):
            if min_pool <= INT_MAX:
                cases += [(min_pool, mc, cells, n) for mc in (0, 2**40) for cells in (0, 12345, INT_MAX)]
    m = SWEEP
    n = _draw(rng, 1, n_hi, m)
    min_pool = [max(65536, v) for v in _draw(rng, 0, INT_MAX, m)]
    min_pool[::3] = [min(INT_MAX, max(65536, k + 1024 + int(d))) for k, d in zip(n[::3], rng.integers(-2, 3, len(n[::3])))]
    cells = _draw(rng, 0, INT_MAX, m)
    min_cap = [min(2**62, v * 64) for v in _draw(rng, 0, INT_MAX, m)]
    min_cap[::3] = [2 * (c + 27 * k) + 16384 + int(d) for c, k, d in zip(cells[::3], n[::3], rng.integers(-2, 3, len(n[::3])))]
    return cases + list(zip(min_pool, min_cap, cells, n))


def test_growth_for_a_batch(rules):
    """dir_min_cap_ as both copies grew it.  min_pool_ as async_grow grew it, clamped to INT_MAX / 2; insert_device did not
    clamp.  The two differ only when the minimum passes INT_MAX / 2, and then both are above LEAF_LIMIT - 1, where
    Map::ensure_capacity refuses every re-pack whatever n_main (want = n_main + max(n_main / 2, min_pool_) > LEAF_LIMIT,
    map.cu:1250-1251).  min_pool_ only ever grows, so the clamp never changes a re-pack that can succeed."""
    rng = np.random.default_rng(5)
    clamped = 0
    for name, copy, n_hi in (("insert_device map.cu:1940", grow_insert_device, INT_MAX - 1024),
                             ("async_grow map.cu:2098", grow_async_grow, INT_MAX)):
        for case in _grow_cases(rng, n_hi):
            min_pool, min_cap, cells, n = case
            pool, cap = copy(*case)
            assert rules.mr_dir_cap_min_for_batch(min_cap, cells, n) == cap, (name, case)
            got = rules.mr_pool_min_for_batch(min_pool, n)
            if copy is grow_async_grow or got == pool:
                assert got == pool, (name, case)
                continue
            clamped += 1
            assert got == INT_MAX // 2 < pool, (name, case)
            for n_main in (1, 2, LEAF_LIMIT):
                assert n_main + max(n_main // 2, got) > LEAF_LIMIT and n_main + max(n_main // 2, pool) > LEAF_LIMIT
    assert clamped > 0


def test_growth_after_a_directory_error(rules):
    """The table 1.5 times the current one and the list pool doubled, at least HALO_NEW_CAP * 262144 (insert_device and
    settle after inserts, build_directory after its own re-list) or twice the plan's need (async_grow after a refusal);
    size_t arithmetic, so values near 2^64 wrap alike."""
    rng = np.random.default_rng(6)
    floor = HALO_NEW_CAP * 262144
    edges = [0, 1, floor // 2 - 1, floor // 2, floor // 2 + 1, 2**32, 2**63 - 1, 2**63, 2**64 - 1]
    caps = [0, 1, 2, 16384, 2**31, UINT_MAX]
    cases = list(itertools.product(edges, edges, caps))
    cases += list(zip(_draw(rng, 0, 2**63 - 1, SWEEP), _draw(rng, 0, 2**63 - 1, SWEEP), _draw(rng, 0, UINT_MAX, SWEEP)))
    for min_cap, min_pool, cap in cases:
        want = after_error_host(min_cap, min_pool, cap)
        got = (rules.mr_dir_cap_min_after_error(min_cap, cap), rules.mr_list_pool_min_grown(min_pool, floor))
        assert got == want, ("insert_device map.cu:1971 / settle map.cu:2062", min_cap, min_pool, cap)
        assert got[1] == pool_build_directory(min_pool), ("build_directory map.cu:1391", min_pool)
    for min_pool, need in itertools.chain(itertools.product(edges, _near(0, floor // 4, INT_MAX)),
                                          zip(_draw(rng, 0, 2**63 - 1, SWEEP), _draw(rng, 0, INT_MAX, SWEEP))):
        assert rules.mr_list_pool_min_grown(min_pool, 2 * need) == pool_async_grow(min_pool, need), ("async_grow map.cu:2107", min_pool, need)
