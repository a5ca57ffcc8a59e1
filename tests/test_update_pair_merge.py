"""CPU: the paired halo-list search of k_update<EXTR, 2> gives the answer of the one-thread scan, and its kernels spill no more
than the one-thread kernels.

Merge rule (update.cuh, knn_block_pair): the owner scans the first ceil(n / 2) 8-candidate chunks of a halo list into a TBest,
the partner the remaining chunks into its own, and the owner then inserts the partner's entries, in order, into its list.  The
model below states TBest (cell_consider + TBest::insert) and checks that rule against one sequential scan of the whole list, on
lists with slots listed twice, deleted slots and many equal distances."""
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import build

K = 5


class TBest:
    def __init__(self):
        self.d = [np.float32(np.inf)] * K
        self.idx = [-1] * K

    def consider(self, d, i):
        """cell_consider: only a distance strictly below the k-th enters; a held slot is refused; ties keep arrival order."""
        if not d < self.d[K - 1] or i in self.idx:
            return
        j = K - 1
        while j > 0 and d < self.d[j - 1]:
            j -= 1
        self.d.insert(j, d); self.idx.insert(j, i)
        self.d.pop(); self.idx.pop()


def sequential(d2, slots, valid):
    kb = TBest()
    for d, s, v in zip(d2, slots, valid):
        if v:
            kb.consider(d, s)
    return kb


def paired(d2, slots, valid):
    n = len(slots)
    h = ((n + 7) // 8 + 1) // 2 * 8                 # the owner's share: the first ceil(chunks / 2) chunks
    a = sequential(d2[:h], slots[:h], valid[:h])
    b = sequential(d2[h:], slots[h:], valid[h:])
    for d, s in zip(b.d, b.idx):
        if s >= 0:
            a.consider(d, s)
    return a


def lists(rng, count):
    for _ in range(count):
        n = int(rng.integers(1, 90))
        pool = int(rng.integers(max(1, n // 3), n + 8))
        slots = rng.integers(0, pool, n)            # a slot may be listed twice (or more)
        dist_of_slot = rng.integers(0, int(rng.integers(1, 12)), pool).astype(np.float32) * np.float32(0.25)   # many ties
        d2 = dist_of_slot[slots]
        valid = rng.random(pool) > 0.15             # deleted points keep their listings
        yield d2, slots.tolist(), valid[slots].tolist()


def test_paired_scan_equals_the_sequential_scan():
    rng = np.random.default_rng(11)
    for d2, slots, valid in lists(rng, 20000):
        s, p = sequential(d2, slots, valid), paired(d2, slots, valid)
        assert s.idx == p.idx and s.d == p.d, (d2, slots, valid)


def test_model_keeps_the_first_of_equal_distances_and_each_slot_once():
    d2 = np.array([1, 1, 0.5, 1, 0.5, 2, 1], np.float32)
    slots = [7, 3, 9, 7, 4, 1, 2]
    kb = sequential(d2, slots, [True] * 7)
    assert kb.idx == [9, 4, 7, 3, 2]


@pytest.fixture(scope="module")
def filter_log(tmp_path_factory):
    """ptxas -v of filter.cu with build.py's flags."""
    nvcc = build._nvcc()
    out = tmp_path_factory.mktemp("cubin") / "filter.cubin"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared",)]
    res = subprocess.run([nvcc, *flags, "-ccbin", "/usr/bin/g++", "-cubin", os.path.join(build.CSRC, "filter.cu"), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return res.stdout + res.stderr


def kernel_info(log, pattern):
    cur, info = None, {}
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and re.search(pattern, cur):
            info[cur] = int(m.group(1)) + int(m.group(2))
    assert len(info) == 1, (pattern, info)
    return next(iter(info.values()))


def test_paired_update_spills_no_more_than_the_single_thread_update(filter_log):
    """The flagship form (no extrinsic estimation): k_update<false, 2> at 512 threads keeps the 128-register cap of
    k_update<false, 1> and spills no more."""
    assert kernel_info(filter_log, r"k_updateILb0ELi2E") <= kernel_info(filter_log, r"k_updateILb0ELi1E")
