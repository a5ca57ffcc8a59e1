"""CPU: the device forms of Add_Points and map_incremental (fl_map_add_points_async, fl_map_maintain,
fl_filter_map_incremental_device) are exported and declared, their kernels do not spill, the kernels pinned by the SASS goldens
are unchanged, and the padding-key sort they run over n_max rows orders the real rows as the host form's sort of n rows."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import sass_functions, spills

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_map_add_points_async", "fl_map_maintain", "fl_filter_map_incremental_device"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def cubin(src, tmp_path_factory):
    nvcc = build._nvcc()
    out = tmp_path_factory.mktemp("cubin") / (os.path.basename(src) + ".cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared",)]
    res = subprocess.run([nvcc, *flags, "-ccbin", "/usr/bin/g++", "-cubin", os.path.join(build.CSRC, src), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", str(out)], capture_output=True, text=True, check=True).stdout
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout).group(0)
    return res.stdout + res.stderr, sass, ver


@pytest.fixture(scope="module")
def cubins(tmp_path_factory):
    return {src: cubin(src, tmp_path_factory) for src in ("map.cu", "filter.cu")}


def test_new_kernels_do_not_spill(cubins):
    sp = spills(cubins["map.cu"][0])
    fresh = [k for k in sp if re.search(r"k_plan|k_async_|k_set_counts", k)]
    assert len(fresh) == 7, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}
    # the Add_Points kernels that now take a device count: no local memory beyond the 8 bytes k_downsample_resolve always had
    for pat in (r"k_voxel_keys", r"k_group_heads", r"k_insert", r"k_halo_claim", r"k_halo_append", r"k_downsample_resolve"):
        k = next(k for k in sp if re.search(pat, k))
        assert sp[k] <= 8, (k, sp[k])


@pytest.mark.parametrize("src, golden", [("map.cu", "sass_existing_kernels_sm90a.json"), ("filter.cu", "sass_update_kernels_sm90a.json")])
def test_pinned_kernels_compile_to_the_same_sass(cubins, src, golden):
    """k_update, k_map_incremental and the query kernels, which the device forms run unchanged."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", golden)))
    log, sass, ver = cubins[src]
    if ver != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {ver}")
    got = sass_functions(sass)
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256("\n".join(got[name]).encode()).hexdigest() == digest, name


PAD = np.uint64(1 << 63)


def stable_sort_bits(keys, vals, end_bit):
    """An LSD radix sort over bits [0, end_bit), 8 bits a pass, as cub::DeviceRadixSort::SortPairs (stable)."""
    keys, vals = keys.copy(), vals.copy()
    for lo in range(0, end_bit, 8):
        width = min(8, end_bit - lo)
        digit = (keys >> np.uint64(lo)) & np.uint64((1 << width) - 1)
        order = np.argsort(digit, kind="stable")
        keys, vals = keys[order], vals[order]
    return keys, vals


@pytest.mark.parametrize("seed", range(6))
def test_padded_sort_orders_the_real_rows_as_the_unpadded_sort(seed):
    """k_voxel_keys gives rows n .. n_max - 1 the key 2^63 and the device forms sort bits 0-63 of n_max rows; the host form sorts
    bits 0-62 of n rows.  The first n rows must agree, keys and values, including real keys at 2^63 - 1 (clamped coordinates)."""
    rng = np.random.default_rng(seed)
    n, n_max = int(rng.integers(1, 400)), 0
    n_max = n + int(rng.integers(0, 300))
    cells = rng.integers(0, 1 << 21, size=(n, 3), dtype=np.uint64)
    cells[rng.random(n) < 0.3] = cells[0]                                 # shared voxels: equal keys must keep their order
    cells[rng.random(n) < 0.1] = (1 << 21) - 1                            # clamped at the top: key 2^63 - 1
    cells[rng.random(n) < 0.05] = 0
    keys = (cells[:, 0] << np.uint64(42)) | (cells[:, 1] << np.uint64(21)) | cells[:, 2]
    assert keys.max() <= np.uint64((1 << 63) - 1)
    vals = np.arange(n, dtype=np.uint32)
    want_k, want_v = stable_sort_bits(keys, vals, 63)
    pk = np.concatenate([keys, np.full(n_max - n, PAD, dtype=np.uint64)])
    pv = np.arange(n_max, dtype=np.uint32)
    got_k, got_v = stable_sort_bits(pk, pv, 64)
    assert np.array_equal(got_k[:n], want_k) and np.array_equal(got_v[:n], want_v)
    assert (got_k[n:] == PAD).all() and (got_v[n:] >= n).all()
    # group heads over the real prefix are those of the unpadded rows, and no group runs into the padding
    heads = lambda k: [r for r in range(len(k)) if r == 0 or k[r] != k[r - 1]]  # noqa: E731
    assert heads(got_k[:n]) == heads(want_k)
    if n_max > n:
        assert got_k[n] != got_k[n - 1]
