"""CPU: the batched preprocess (fl_preprocess_batch_*) is exported, declared and bound, fl_preprocess_raw_t is 16 bytes, its kernels
do not spill, preprocess.cu's single-frame kernels compile to the SASS they had before the batch was added, and a numpy model of
the slot-prefixed ring sort, the scan by key and the global scans less each slot's base gives every slot the single form's
answer."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import sass_functions, spills
from test_map_async_build import cubin, stable_sort_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_preprocess_batch_create", "fl_preprocess_batch_destroy", "fl_preprocess_batch_run_device",
               "fl_preprocess_batch_get_outputs", "fl_preprocess_batch_download"]


def test_symbols_exported_declared_and_bound():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def test_preprocess_raw_layout(tmp_path):
    """fl_preprocess_raw_t: raw at 0, n_raw at 8, 16 bytes, in C and in the binding."""
    assert api.C.sizeof(api.PreprocessRaw) == 16
    assert (api.PreprocessRaw.raw.offset, api.PreprocessRaw.n_raw.offset) == (0, 8)
    src = tmp_path / "raw.c"
    src.write_text('#include "fastlio_b200.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(fl_preprocess_raw_t) == 16, "size");\n'
                   '_Static_assert(offsetof(fl_preprocess_raw_t, raw) == 0, "raw");\n'
                   '_Static_assert(offsetof(fl_preprocess_raw_t, n_raw) == 8, "n_raw");\n'
                   "int main(void) { return 0; }\n")
    res = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "raw")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


@pytest.fixture(scope="module")
def pp_cubin(tmp_path_factory):
    return cubin("preprocess.cu", tmp_path_factory)


def test_new_kernels_do_not_spill(pp_cubin):
    sp = spills(pp_cubin[0])
    fresh = [k for k in sp if re.search(r"k_ppb_(mark|avia_keep|velo_head|velo_tri|velo_out|scatter|commit)", k)]
    assert len(fresh) == 7, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}


def anon(text):
    """preprocess.cu's kernels live in an anonymous namespace, whose mangled name depends on the file: replaced by ANON."""
    return re.sub(r"\d+_GLOBAL__N__\w*?_preprocess_cu_[0-9a-f]{8}", "ANON", text)


def test_single_frame_kernels_compile_to_the_same_sass(pp_cubin):
    """k_pp_mark, k_pp_avia_keep, the three Velodyne kernels and k_pp_scatter: the batch shares their device helpers."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_preprocess_kernels_sm90a.json")))
    _, sass, ver = pp_cubin
    if ver != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {ver}")
    got = {anon(k): v for k, v in sass_functions(sass).items()}
    assert len(want["functions"]) == 6
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256(anon("\n".join(got[name])).encode()).hexdigest() == digest, name


def key_bits(n_scans):
    """PpParams.key_bits: the bits of the ring keys 0 .. n_scans (n_scans is the padding key)."""
    b = 1
    while (1 << b) <= n_scans:
        b += 1
    return b


def slot_bits(n):
    b = 0
    while (1 << b) < n:
        b += 1
    return b


def tri_scan(keys, t, a, b, first):
    """cub::DeviceScan::InclusiveScanByKey with TriCompose: the aggregate restarts where the key changes (or at `first`);
    returns the scanned maps applied to 0 (k_pp_velo_out's time)."""
    out = np.zeros(len(keys), np.float32)
    acc = None
    for p in range(len(keys)):
        x = (t[p], a[p], b[p])
        if acc is None or first[p] or keys[p] != keys[p - 1]:
            acc = x
        else:
            app = lambda f, c: f[2] if f[0] < c else f[1]          # noqa: E731
            acc = (acc[0], app(x, acc[1]), app(x, acc[2]))
        out[p] = acc[2] if acc[0] < 0.0 else acc[1]
    return out


@pytest.mark.parametrize("seed", range(8))
def test_slot_prefixed_ring_sort_and_scans_equal_the_single_form(seed):
    """k_ppb_mark keys row i of slot s (count c) as (s << key_bits) | ring for a yaw row and (s << key_bits) | n_scans otherwise
    (rows past c, rings >= n_scans), one stable sort on key_bits + slot_bits(n_slots_max) bits runs over every slot, one scan by
    key restarts at every (slot, ring), and the Avia and compaction sums run once over all rows less the slot's base.  Each slot
    must come out as the single form's n_max-row frame: rows in its region, in the single sort's order, the Tri composition
    restarted at the slot's first row, and positions equal to its own scans."""
    rng = np.random.default_rng(seed)
    n_scans = int(rng.choice([6, 16, 32, 64, 128]))
    kb = key_bits(n_scans)
    S = int(rng.integers(1, 10))
    S_max = S + int(rng.integers(0, 40))
    n_max = int(rng.integers(1, 200))
    counts = rng.integers(0, n_max + 1, S)
    for c in (0, 1, n_max):
        counts[rng.integers(0, S)] = c
    end_bit = kb + slot_bits(S_max)
    assert end_bit <= 32 and key_bits(128) + slot_bits(65535) <= 32
    keys, rings = [], []
    for s in range(S):
        ring = rng.integers(0, n_scans + 8, n_max)                # some rings >= n_scans: dropped rows
        ring[rng.random(n_max) < 0.3] = ring[0]
        k = np.where((np.arange(n_max) < counts[s]) & (ring < n_scans), ring, n_scans).astype(np.uint64)
        rings.append(k)
        keys.append((np.uint64(s) << np.uint64(kb)) | k)
    got_k, got_v = stable_sort_bits(np.concatenate(keys), np.arange(S * n_max, dtype=np.uint64), end_bit)
    # the maps of the sorted rows: a run's first row (and padding) the constant 0, the others (lo, lo, hi)
    lo = rng.uniform(0, 100, S * n_max).astype(np.float32)
    hi = (lo + np.float32(99.7)).astype(np.float32)
    lo_ring = got_k & np.uint64((1 << kb) - 1)
    head = np.r_[True, got_k[1:] != got_k[:-1]]
    zero = head | (lo_ring >= n_scans)
    t, a, b = np.where(zero, 0, lo), np.where(zero, 0, lo), np.where(zero, 0, hi)
    batch_tm = tri_scan(got_k, t, a, b, np.zeros(S * n_max, bool))
    keep = (rng.random(S * n_max) < 0.6).astype(np.int64)
    valid = (rng.random(S * n_max) < 0.7).astype(np.int64)
    for s in range(S):
        keep[s * n_max + counts[s]:(s + 1) * n_max] = 0
        valid[s * n_max + counts[s]:(s + 1) * n_max] = 0
        valid[s * n_max] = 0                                      # Avia's row 0 is never valid
    pos = np.concatenate([[0], np.cumsum(keep)[:-1]])              # one exclusive sum over every slot
    vsum = np.cumsum(valid)                                        # one inclusive sum
    for s in range(S):
        region = slice(s * n_max, (s + 1) * n_max)
        want_k, want_v = stable_sort_bits(rings[s], np.arange(n_max, dtype=np.uint64), kb)
        assert (got_k[region] >> np.uint64(kb) == s).all()
        assert np.array_equal(got_k[region] & np.uint64((1 << kb) - 1), want_k)
        assert np.array_equal(got_v[region] - np.uint64(s * n_max), want_v)
        # the single form's scan over the slot's own sorted rows, restarting at its first row
        first = np.zeros(n_max, bool)
        first[0] = True
        want_tm = tri_scan(want_k, t[region], a[region], b[region], first)
        assert batch_tm[region].tobytes() == want_tm.tobytes()
        kp, vp = keep[region], valid[region]
        assert np.array_equal(pos[region] - pos[s * n_max], np.concatenate([[0], np.cumsum(kp)[:-1]]))
        assert np.array_equal(vsum[region] - (vsum[s * n_max] - valid[s * n_max]), np.cumsum(vp))
        assert pos[s * n_max + n_max - 1] + keep[s * n_max + n_max - 1] - pos[s * n_max] == kp.sum()
