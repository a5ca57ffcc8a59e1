"""CPU: the device-buffer update (fl_filter_update_device and its two getters) is exported and declared, its two kernels do not
spill, and k_update and k_map_incremental, which it runs unchanged, compile to the same SASS as before it was added."""
import hashlib
import json
import os
import re
import subprocess

import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import sass_functions, spills

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_filter_update_device", "fl_filter_get_nearest_device", "fl_filter_get_selected_device"]


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
def filter_cubin(tmp_path_factory):
    """filter.cu alone, with build.py's flags, as a cubin; returns (ptxas -v log, SASS text, nvcc version)."""
    nvcc = build._nvcc()
    out = tmp_path_factory.mktemp("cubin") / "filter.cubin"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared",)]
    res = subprocess.run([nvcc, *flags, "-ccbin", "/usr/bin/g++", "-cubin", os.path.join(build.CSRC, "filter.cu"), "-o", str(out)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", str(out)], capture_output=True, text=True, check=True).stdout
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout).group(0)
    return res.stdout + res.stderr, sass, ver


def test_state_kernels_do_not_spill(filter_cubin):
    sp = spills(filter_cubin[0])
    fresh = [k for k in sp if re.search(r"k_state_(in|out)", k)]
    assert len(fresh) == 2, fresh
    assert all(sp[k] == 0 for k in fresh), {k: sp[k] for k in fresh}


def test_update_kernels_compile_to_the_same_sass(filter_cubin):
    """The four k_update instantiations and k_map_incremental compile to the SASS recorded before the device-buffer update."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_update_kernels_sm90a.json")))
    if filter_cubin[2] != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {filter_cubin[2]}")
    got = sass_functions(filter_cubin[1])
    assert len(want["functions"]) == 5
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256("\n".join(got[name]).encode()).hexdigest() == digest, name
