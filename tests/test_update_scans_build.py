"""CPU: the batched update over many scans (fl_scan_get_ref, fl_filter_update_scans_device) is exported, declared and bound,
fl_scan_ref_t is 16 bytes, k_update_scans(_det) keeps the co-resident footprint of the one-thread k_update it runs, and its
state kernels do not spill.  The SASS pins of k_update and k_map_incremental are checked, unchanged, by
test_filter_device_build.py and test_map_async_build.py."""
import os
import re
import subprocess

import pytest

from fast_lio_b200 import api, build
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_scan_get_ref", "fl_filter_update_scans_device"]


def test_symbols_exported_declared_and_bound():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def test_scan_ref_layout(tmp_path):
    """fl_scan_ref_t: two device pointers, 16 bytes, the body at offset 0, in C and in the binding."""
    assert api.C.sizeof(api.ScanRef) == 16 and api.ScanRef.n.offset == 8
    src = tmp_path / "ref.c"
    src.write_text('#include "fastlio_b200.h"\n#include <stddef.h>\n'
                   "_Static_assert(sizeof(fl_scan_ref_t) == 16, \"size\");\n"
                   "_Static_assert(offsetof(fl_scan_ref_t, n) == 8, \"n\");\nint main(void) { return 0; }\n")
    res = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "ref")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


@pytest.fixture(scope="module")
def filter_log(tmp_path_factory):
    return cubin("filter.cu", tmp_path_factory)[0]


def footprint(log):
    """{kernel: (stack frame bytes, spill store + load bytes, registers, shared memory bytes)} from ptxas -v.  Only the properties
    block of the entry function itself counts (ptxas also lists the non-inlined device functions an entry calls)."""
    out, cur, props = {}, None, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur, props = m.group(1), None
            out[cur] = [0, 0, 0, 0]
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            props = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and props == cur:
            out[cur][0], out[cur][1] = int(m.group(1)), int(m.group(2)) + int(m.group(3))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m and cur:
            out[cur][2], out[cur][3] = int(m.group(1)), int(m.group(2))
    return out


def one(table, pat):
    hits = [k for k in table if re.search(pat, k)]
    assert len(hits) == 1, (pat, hits)
    return hits[0]


@pytest.mark.parametrize("det", ["", "_det"])
@pytest.mark.parametrize("extr", ["0", "1"])
def test_scans_kernel_keeps_the_co_resident_footprint(filter_log, extr, det):
    """The registers (128) and the shared memory of k_update<EXTR, 1>, so one k_update_scans block per k_update_batch block fits on
    an SM and UK_BATCH's plan holds.  Like k_update_batch it keeps the slot's pointers in registers rather than in the parameter
    bank, so it spills more than k_update; its stack and spills may exceed k_update_batch's by at most 128 and 384 bytes.
    Measured with nvcc 12.9 for sm_90a (stack bytes / spill stores + loads bytes): k_update_scans<0> 336 / 508 and
    k_update_scans<1> 432 / 1016, against 336 / 508 and 392 / 716 for k_update_batch and 288 / 352 and 288 / 496 for
    k_update<EXTR, 1>; the _det forms 328 / 544 and 392 / 792, the figures of k_update_batch_det."""
    fp = footprint(filter_log)
    base = fp[f"_ZN2fl8k_updateILb{extr}ELi1EEEvNS_7UpdArgsE"]
    batch = fp[one(fp, rf"\dk_update_batch{det}ILb{extr}E")]
    name = one(fp, rf"\dk_update_scans{det}ILb{extr}E")
    new = fp[name]
    print(f"{name}: stack {new[0]}, spills {new[1]}, registers {new[2]}, smem {new[3]}; k_update_batch{det}: {batch}; k_update: {base}")
    assert new[2] == base[2] == 128 and new[3] == base[3] > 0, (new, base)
    assert new[0] <= batch[0] + 128 and new[1] <= batch[1] + 384, (new, batch)


def test_scans_state_kernels_do_not_spill(filter_log):
    fp = footprint(filter_log)
    fresh = [k for k in fp if re.search(r"k_scans_state_(in|out)", k)]
    assert len(fresh) == 2, fresh
    assert all(fp[k][0] == 0 and fp[k][1] == 0 for k in fresh), {k: fp[k] for k in fresh}
