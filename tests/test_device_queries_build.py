"""CPU: the device-buffer map queries are exported and declared, their new kernels do not spill beyond the kernels they reuse,
and the kernels they share code with compile to the same SASS as before."""
import hashlib
import json
import os
import re
import subprocess

import pytest

from fast_lio_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_map_nearest_search_device", "fl_map_range_workspace_bytes", "fl_map_box_search_device",
               "fl_map_radius_search_device", "fl_map_build_device", "fl_map_add_points_device"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s


def sass_functions(text):
    out, name, buf = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = buf
            name, buf = m.group(1), []
        elif name:
            s = re.sub(r"/\*[0-9a-f]{4}\*/", "", line)
            s = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", s).strip()
            if s:
                buf.append(s)
    if name:
        out[name] = buf
    return out


@pytest.fixture(scope="module")
def map_cubin(tmp_path_factory):
    """map.cu alone, with build.py's flags, as a cubin; returns (ptxas -v log, SASS text, nvcc version)."""
    nvcc = build._nvcc()
    out = tmp_path_factory.mktemp("cubin") / "map.cubin"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared",)]
    res = subprocess.run([nvcc, *flags, "-ccbin", "/usr/bin/g++", "-cubin", os.path.join(build.CSRC, "map.cu"), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", str(out)], capture_output=True, text=True, check=True).stdout
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout).group(0)
    return res.stdout + res.stderr, sass, ver


def spills(log):
    """{kernel: spill store + load bytes} from ptxas -v."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = int(m.group(1)) + int(m.group(2))
    return out


def test_new_kernels_do_not_spill(map_cubin):
    sp = spills(map_cubin[0])
    fresh = [k for k in sp if re.search(r"k_dscan_|k_range_(plan|status|offsets_dev|count_dev|fill_dev)", k)]
    assert len(fresh) == 10, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}
    # the kernels that run an existing kernel's body: no more local memory than that kernel already uses
    by = lambda pat: next(sp[k] for k in sp if re.search(pat, k))  # noqa: E731
    assert by(r"k_knn_batch_gated") <= by(r"k_knn_batchENS") + 8
    assert by(r"k_range_leaves_boundedILb0") <= by(r"k_range_leavesILb0") + 8
    assert by(r"k_range_leaves_boundedILb1") <= by(r"k_range_leavesILb1") + 8


def test_kept_kernels_compile_to_the_same_sass(map_cubin):
    """k_knn_batch, k_knn_k and k_range_leaves, whose bodies the device-buffer queries reuse, compile to the SASS recorded
    before those queries were added."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_existing_kernels_sm90a.json")))
    if map_cubin[2] != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {map_cubin[2]}")
    got = sass_functions(map_cubin[1])
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256("\n".join(got[name]).encode()).hexdigest() == digest, name


def test_host_range_search_has_no_kernels_of_its_own(map_cubin):
    """The host-buffer range search runs the device-buffer pipeline: its former kernels are gone from the cubin."""
    names = sass_functions(map_cubin[1])
    gone = [n for n in names if re.search(r"k_range_(count|fill)ILb|k_range_offsetsE", n)]
    assert not gone, gone
    assert any("k_range_count_dev" in n for n in names) and any("k_range_offsets_dev" in n for n in names)
