"""CPU: the batched update (fl_filter_reserve_batch, fl_filter_batch_plan, fl_filter_update_batch_device) is exported, declared
and bound, k_update_batch keeps the co-resident footprint of the one-thread k_update it runs, and its state kernels do not spill.
The SASS pins of k_update and k_map_incremental are checked, unchanged, by test_filter_device_build.py."""
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import spills
from test_frontend_device_build import frames
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_filter_reserve_batch", "fl_filter_batch_plan", "fl_filter_update_batch_device"]


def test_symbols_exported_declared_and_bound():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


@pytest.fixture(scope="module")
def filter_log(tmp_path_factory):
    return cubin("filter.cu", tmp_path_factory)[0]


@pytest.mark.parametrize("extr", ["0", "1"])
def test_batch_kernel_keeps_the_co_resident_footprint(filter_log, extr):
    """The registers and the shared memory of k_update<EXTR, 1>, so one k_update_batch block per k_update block fits on an SM.
    The slot's offset pointers live in registers rather than in the parameter bank, so ptxas spills a little more: stack and
    spill bytes may exceed k_update's by at most 128 and 384 bytes (measured with nvcc 12.9: +48 / +104 bytes of stack and
    +156 / +220 bytes spilled for EXTR 0 / 1)."""
    fr = frames(filter_log)
    base = fr[f"_ZN2fl8k_updateILb{extr}ELi1EEEvNS_7UpdArgsE"]
    new = fr[f"_ZN2fl14k_update_batchILb{extr}EEEvNS_7UpdArgsEi"]
    assert new[1:] == base[1:], (new, base)
    assert base[0] <= new[0] <= base[0] + 128, (new, base)
    sp = spills(filter_log)
    b, n = sp[f"_ZN2fl8k_updateILb{extr}ELi1EEEvNS_7UpdArgsE"], sp[f"_ZN2fl14k_update_batchILb{extr}EEEvNS_7UpdArgsEi"]
    assert n <= b + 384, (n, b)


def test_batch_state_kernels_do_not_spill(filter_log):
    sp = spills(filter_log)
    fresh = [k for k in sp if re.search(r"k_batch_state_(in|out)", k)]
    assert len(fresh) == 2, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}


def test_pass_log_decoder_reads_the_abi_layout():
    """decode_pass_logs reads fl_pass_log_t rows as pass_logs() returns them."""
    n = api.C.sizeof(api.PassLog)
    assert n == 4 * 4 + 8 * (1 + 144 + 12 + 26)
    rows = []
    for i in range(3):
        l = api.PassLog()
        l.searched, l.valid, l.effct, l.converged, l.res_sum = i, 1, 10 * i, i % 2, 0.5 * i
        for j in range(144):
            l.HtH[j] = i + j / 7.0
        for j in range(12):
            l.Hth[j] = -j - i
        for j in range(26):
            l.x_after[j] = j * 0.25 + i
        rows.append(np.frombuffer(bytes(l), np.uint8))
    raw = np.stack(rows)
    logs = api.decode_pass_logs(raw, 2)
    assert len(logs) == 2
    assert logs[1]["effct"] == 10 and logs[1]["res_sum"] == 0.5 and logs[1]["HtH"].shape == (12, 12)
    assert logs[1]["HtH"][0, 1] == 1 + 1 / 7.0 and logs[0]["x_after"][4] == 1.0
    with pytest.raises(ValueError):
        api.decode_pass_logs(raw, 4)
