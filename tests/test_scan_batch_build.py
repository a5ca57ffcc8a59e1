"""CPU: the batched scan front end (fl_scan_batch_*) is exported, declared and bound, fl_scan_raw_t is 48 bytes, its kernels do not
spill, the one slot-prefixed time sort it runs orders each slot's rows as the single form's padded sort orders the scan's, and
scan.cu's single-scan kernels compile to the SASS they had before the batch was added."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import sass_functions, spills
from test_frontend_device_build import PAD_TIME, twiddle_f32
from test_map_async_build import cubin, stable_sort_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_scan_batch_create", "fl_scan_batch_destroy", "fl_scan_batch_reserve", "fl_scan_batch_run_device",
               "fl_scan_batch_get_refs", "fl_scan_batch_download"]
FIELDS = ["xyzi", "offset_ms", "n", "imu_pose22", "n_pose", "x26_end"]


def test_symbols_exported_declared_and_bound():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def test_scan_raw_layout(tmp_path):
    """fl_scan_raw_t: six device pointers, 48 bytes, in the order of the header, in C and in the binding."""
    assert api.C.sizeof(api.ScanRaw) == 48
    assert [getattr(api.ScanRaw, f).offset for f in FIELDS] == [8 * i for i in range(6)]
    asserts = "".join(f"_Static_assert(offsetof(fl_scan_raw_t, {f}) == {8 * i}, \"{f}\");\n" for i, f in enumerate(FIELDS))
    src = tmp_path / "raw.c"
    src.write_text('#include "fastlio_b200.h"\n#include <stddef.h>\n_Static_assert(sizeof(fl_scan_raw_t) == 48, "size");\n' + asserts +
                   "int main(void) { return 0; }\n")
    res = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "raw")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


@pytest.fixture(scope="module")
def scan_cubin(tmp_path_factory):
    return cubin("scan.cu", tmp_path_factory)


def test_new_kernels_do_not_spill(scan_cubin):
    sp = spills(scan_cubin[0])
    fresh = [k for k in sp if re.search(r"k_batch_(gather|undistort|minmax|keys|heads|centroid|commit)", k)]
    assert len(fresh) == 7, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}


def anon(text):
    """scan.cu's kernels live in an anonymous namespace, whose mangled name depends on the file: replaced by ANON."""
    return re.sub(r"\d+_GLOBAL__N__\w*?_scan_cu_[0-9a-f]{8}", "ANON", text)


def test_single_scan_kernels_compile_to_the_same_sass(scan_cubin):
    """k_upload_n, k_undistort, the voxel-grid kernels, k_frame and the cube kernels: the batch shares their device helpers."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_scan_kernels_sm90a.json")))
    _, sass, ver = scan_cubin
    if ver != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {ver}")
    got = {anon(k): v for k, v in sass_functions(sass).items()}
    assert len(want["functions"]) == 11
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256(anon("\n".join(got[name])).encode()).hexdigest() == digest, name


def awkward_times(rng, n):
    t = rng.uniform(-5, 100, n).astype(np.float32)
    t[rng.random(n) < 0.2] = t[0]
    t[rng.random(n) < 0.05] = 0.0
    t[rng.random(n) < 0.05] = -0.0
    t[rng.random(n) < 0.03] = np.inf
    t[rng.random(n) < 0.03] = -np.inf
    nan_bits = rng.choice(np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, 0x7FFFFFFF, 0x7FFFFFFE], np.uint32), n)
    pick = rng.random(n) < 0.1
    t[pick] = nan_bits[pick].view(np.float32)
    return t


@pytest.mark.parametrize("seed", range(6))
def test_slot_prefixed_sort_orders_each_slot_as_the_single_padded_sort(seed):
    """k_batch_gather keys row i of slot s (count c) as (s << 32) | twiddle(t), the padding rows [c, n_max) as (s << 32) |
    0xFFFFFFFF, and one stable sort on bits [0, 32 + ceil(log2 S)) runs over every slot.  Each slot's rows must come out in its
    own region, ordered as the single form's stable 32-bit sort of its n_max padded rows orders them -- ties, +-0.0, +-inf, NaNs of
    various payloads and real times equal to the padding pattern included."""
    rng = np.random.default_rng(seed)
    S = int(rng.integers(1, 9))
    n_max = int(rng.integers(1, 300))
    counts = rng.integers(0, n_max + 1, S)
    counts[rng.integers(0, S)] = n_max
    keys, times = [], []
    for s in range(S):
        t = np.concatenate([awkward_times(rng, int(counts[s])), np.full(n_max - counts[s], PAD_TIME, np.float32)])
        times.append(t)
        keys.append((np.uint64(s) << np.uint64(32)) | twiddle_f32(t))
    end_bit = 32 + int(np.ceil(np.log2(S))) if S > 1 else 32
    got_k, got_v = stable_sort_bits(np.concatenate(keys), np.arange(S * n_max, dtype=np.uint32), end_bit)
    for s in range(S):
        want_k, want_v = stable_sort_bits(twiddle_f32(times[s]), np.arange(n_max, dtype=np.uint32), 32)
        region = slice(s * n_max, (s + 1) * n_max)
        assert (got_k[region] >> np.uint64(32) == s).all()
        assert np.array_equal(got_k[region] & np.uint64(0xFFFFFFFF), want_k)
        assert np.array_equal(got_v[region] - s * n_max, want_v)
        assert (want_v[counts[s]:] >= counts[s]).all()          # the padding rows sort last in the slot
