"""CPU: the device forms of the scan front end and of the update on it (fl_scan_reserve, fl_scan_*_device,
fl_filter_update_scan_device) are exported and declared, their kernels do not spill, and the padded sorts they run over n_max
rows order the real rows as the host forms' sorts of n rows."""
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import spills
from test_map_async_build import cubin, stable_sort_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_scan_reserve", "fl_scan_upload_device", "fl_scan_undistort_device", "fl_scan_voxel_downsample_device",
               "fl_filter_update_scan_device"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


@pytest.fixture(scope="module")
def logs(tmp_path_factory):
    return {src: cubin(src, tmp_path_factory)[0] for src in ("scan.cu", "filter.cu")}


def frames(log):
    """{kernel: (stack frame bytes, registers, shared memory bytes)} from ptxas -v."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame", line)
        if m and cur:
            out[cur] = [int(m.group(1)), 0, 0]
        m = re.search(r"Used (\d+) registers.*?(?:(\d+) bytes smem)?$", line)
        if m and cur in out:
            out[cur][1], out[cur][2] = int(m.group(1)), int(m.group(2) or 0)
    return out


def test_new_kernels_do_not_spill(logs):
    sp = spills(logs["scan.cu"])
    for pat in ("k_upload_n", "k_undistort", "k_vg_reset", "k_vg_minmax", "k_vg_keys", "k_vg_heads", "k_vg_centroid"):
        k = next(k for k in sp if re.search(pat, k))
        assert sp[k] == 0, (k, sp[k])
    sp = spills(logs["filter.cu"])
    k = next(k for k in sp if "k_flags_clear" in k)
    assert sp[k] == 0, (k, sp[k])


@pytest.mark.parametrize("extr", ["0", "1"])
@pytest.mark.parametrize("pair", ["1", "2"])
def test_k_update_n_keeps_k_updates_footprint(logs, extr, pair):
    """k_update_n is k_update's body with the count read from memory: the same registers, shared memory and stack frame
    (k_update itself keeps a few values on the stack under its 128-register cap), so it fits the same co-resident grid."""
    fr = frames(logs["filter.cu"])
    base = fr[f"_ZN2fl8k_updateILb{extr}ELi{pair}EEEvNS_7UpdArgsE"]
    new = fr[f"_ZN2fl10k_update_nILb{extr}ELi{pair}EEEvNS_7UpdArgsEPKi"]
    assert new == base, (new, base)


def twiddle_f32(t):
    """cub's radix key for float32: -0.0 folded onto +0.0, then the sign-dependent flip (cub/util_type.cuh TwiddleIn)."""
    bits = np.ascontiguousarray(t, np.float32).view(np.uint32).astype(np.uint64)
    bits[bits == 0x80000000] = 0
    neg = (bits & 0x80000000) != 0
    return np.where(neg, bits ^ 0xFFFFFFFF, bits ^ 0x80000000).astype(np.uint64)


PAD_TIME = np.array([0x7FFFFFFF], np.uint32).view(np.float32)[0]


@pytest.mark.parametrize("seed", range(8))
def test_padded_time_sort_orders_the_real_rows_as_the_unpadded_sort(seed):
    """k_upload_n gives rows n .. n_max - 1 the offset time 0x7FFFFFFF; the stable sort of n_max rows must order the first n rows as
    the sort of n rows, with ties, +-0.0, +-inf, NaNs of various payloads and real times equal to the padding pattern."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 500))
    n_max = n + int(rng.integers(0, 300))
    t = rng.uniform(-5, 100, n).astype(np.float32)
    t[rng.random(n) < 0.2] = t[0]
    t[rng.random(n) < 0.05] = 0.0
    t[rng.random(n) < 0.05] = -0.0
    t[rng.random(n) < 0.03] = np.inf
    t[rng.random(n) < 0.03] = -np.inf
    nan_bits = rng.choice(np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, 0x7FFFFFFF, 0x7FFFFFFE], np.uint32), n)
    pick = rng.random(n) < 0.1
    t[pick] = nan_bits[pick].view(np.float32)
    vals = np.arange(n, dtype=np.uint32)
    want_k, want_v = stable_sort_bits(twiddle_f32(t), vals, 32)
    pt = np.concatenate([t, np.full(n_max - n, PAD_TIME, np.float32)])
    got_k, got_v = stable_sort_bits(twiddle_f32(pt), np.arange(n_max, dtype=np.uint32), 32)
    assert np.array_equal(got_k[:n], want_k) and np.array_equal(got_v[:n], want_v)
    assert (got_v[n:] >= n).all()
    assert twiddle_f32(np.array([PAD_TIME]))[0] == 0xFFFFFFFF       # the largest key there is


@pytest.mark.parametrize("seed", range(6))
def test_padded_voxel_sort_orders_the_real_rows_as_the_unpadded_sort(seed):
    """k_vg_keys gives rows n .. n_max - 1 the key 0xFFFFFFFF, k_vg_heads makes them no heads: the first n rows of the sort, the
    heads and their exclusive scan equal the n-row ones, also with real keys at 0xFFFFFFFF."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 500))
    n_max = n + int(rng.integers(0, 300))
    keys = rng.integers(0, 1 << 31, n, dtype=np.uint64)
    keys[rng.random(n) < 0.4] = keys[0]
    keys[rng.random(n) < 0.05] = 0xFFFFFFFF
    want_k, want_v = stable_sort_bits(keys, np.arange(n, dtype=np.uint32), 32)
    pk = np.concatenate([keys, np.full(n_max - n, 0xFFFFFFFF, np.uint64)])
    got_k, got_v = stable_sort_bits(pk, np.arange(n_max, dtype=np.uint32), 32)
    assert np.array_equal(got_k[:n], want_k) and np.array_equal(got_v[:n], want_v)

    def heads(k, count):
        return np.array([1 if r < count and (r == 0 or k[r] != k[r - 1]) else 0 for r in range(len(k))], np.int64)
    hw, hg = heads(want_k, n), heads(got_k, n)
    assert np.array_equal(hg[:n], hw) and not hg[n:].any()
    assert np.array_equal((np.cumsum(hg) - hg)[:n], np.cumsum(hw) - hw)
