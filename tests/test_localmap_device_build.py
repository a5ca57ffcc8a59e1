"""CPU: the device forms of lasermap_fov_segment and Delete_Point_Boxes (fl_localmap_segment_device, fl_map_delete_boxes_async)
are exported and declared, the new and changed kernels do not spill, the kernels pinned by the SASS goldens are unchanged, and
the host form of the segment still runs the restated lasermap_fov_segment through the cube arithmetic it shares with the
device form."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from oracle import bind
from test_device_queries_build import sass_functions, spills
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_map_delete_boxes_async", "fl_localmap_segment_device"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s
    # the per-scan chain no longer leaves the segment on the host
    assert "lasermap_fov_segment stay on the host" not in hdr


@pytest.fixture(scope="module")
def cubins(tmp_path_factory):
    return {src: cubin(src, tmp_path_factory) for src in ("map.cu", "scan.cu", "filter.cu")}


def test_new_and_changed_kernels_do_not_spill(cubins):
    for src, pats in (("map.cu", ("k_delete_plan", "k_delete_boxes", "k_delete_account", "k_delete_status", "k_refit_leaves",
                                  "k_refit_level")), ("scan.cu", ("k_seg_slide", "k_seg_commit"))):
        sp = spills(cubins[src][0])
        for pat in pats:
            k = next(k for k in sp if pat in k)
            assert sp[k] == 0, (k, sp[k])


@pytest.mark.parametrize("src, golden", [("map.cu", "sass_existing_kernels_sm90a.json"), ("filter.cu", "sass_update_kernels_sm90a.json")])
def test_pinned_kernels_compile_to_the_same_sass(cubins, src, golden):
    """k_update x4, k_map_incremental, k_knn_batch, k_knn_k and k_range_leaves."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", golden)))
    _, sass, ver = cubins[src]
    if ver != want["nvcc"]:
        pytest.skip(f"digests recorded with nvcc {want['nvcc']}, this is {ver}")
    got = sass_functions(sass)
    for name, digest in want["functions"].items():
        assert name in got, name
        assert hashlib.sha256("\n".join(got[name]).encode()).hexdigest() == digest, name


@pytest.mark.parametrize("cube_len, det_range", [(40.0, 8.0), (3.0, 0.5), (200.0, 300.0)])
def test_host_form_without_a_map_is_the_restated_segment(cube_len, det_range):
    ours, ref = api.LocalMap(cube_len, det_range), bind.LocalMap(cube_len, det_range)
    rng = np.random.default_rng(int(cube_len))
    pos = np.zeros(3)
    moved = 0
    for _ in range(300):
        pos = pos + cube_len / 30.0 * rng.normal(0.3, 1.0, 3)
        b_ref = ref.segment(pos)
        b, n = ours.segment(pos, None)
        assert n == 0 and b.tobytes() == np.ascontiguousarray(b_ref, np.float32).tobytes()
        assert ours.box().tobytes() == ref.box().tobytes()
        moved += len(b_ref)
    assert moved > 0
