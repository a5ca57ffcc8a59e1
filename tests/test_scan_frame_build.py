"""CPU: the scan's clouds in a frame (fl_scan_frame, fl_scan_frame_device) are exported, declared with the FL_FRAME_* values and
bound; the new kernels do not spill; and the kernels pinned by the SASS goldens in map.cu and filter.cu are unchanged."""
import hashlib
import json
import os
import re
import subprocess

import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import sass_functions, spills
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_scan_frame", "fl_scan_frame_device"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s
    frames = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define FL_FRAME_(\w+)\s+(\d+)", hdr)}
    assert frames == {"LIDAR": 0, "IMU": 1, "WORLD": 2}
    assert (api.FRAME_LIDAR, api.FRAME_IMU, api.FRAME_WORLD) == (0, 1, 2)


@pytest.fixture(scope="module")
def cubins(tmp_path_factory):
    return {src: cubin(src, tmp_path_factory) for src in ("scan.cu", "map.cu", "filter.cu")}


def test_new_kernels_do_not_spill(cubins):
    sp = spills(cubins["scan.cu"][0])
    ours = [k for k in sp if re.search(r"k_frame", k)]
    assert len(ours) == 2, ours
    assert all(sp[k] == 0 for k in ours), {k: sp[k] for k in ours}


@pytest.mark.parametrize("src, golden", [("map.cu", "sass_existing_kernels_sm90a.json"), ("filter.cu", "sass_update_kernels_sm90a.json")])
def test_pinned_kernels_compile_to_the_same_sass(cubins, src, golden):
    want = json.load(open(os.path.join(ROOT, "tests", "golden", golden)))
    _, sass, ver = cubins[src]
    if ver != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {ver}")
    got = sass_functions(sass)
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256("\n".join(got[name]).encode()).hexdigest() == digest, name
