"""CPU: the sensor-preprocessing entry points (fl_preprocess_*) are exported, declared and bound, and the kernels of
preprocess.cu do not spill.  The SASS pins of map.cu and filter.cu are checked, unchanged, by test_map_async_build.py."""
import os
import re
import subprocess

import pytest

from fast_lio_b200 import api, build
from test_device_queries_build import spills
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_preprocess_create", "fl_preprocess_destroy", "fl_preprocess_device", "fl_preprocess"]


def test_symbols_exported_and_declared():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def test_params_struct_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    body = re.search(r"typedef struct fl_preprocess_params \{(.*?)\} fl_preprocess_params_t;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [n for decl in body.split(";") if decl.strip() for n in re.findall(r"(\w+)\s*(?:,|$)", decl.strip().split(None, 1)[1])]
    assert names == [f for f, _ in api.PreprocessParams._fields_]


@pytest.fixture(scope="module")
def log(tmp_path_factory):
    return cubin("preprocess.cu", tmp_path_factory)[0]


def test_new_kernels_do_not_spill(log):
    sp = spills(log)
    ours = [k for k in sp if re.search(r"k_pp_", k)]
    assert len(ours) == 6, ours
    assert all(sp[k] == 0 for k in ours), {k: sp[k] for k in ours}


def test_default_layouts_are_the_reference_structs():
    """CustomPoint 20 bytes, velodyne_ros::Point 32, ouster_ros::Point 48 (PCL's 16-byte alignment), pcl::PointXYZI 32."""
    assert [api.DEFAULT_LAYOUT[t].itemsize for t in (1, 2, 3, 4)] == [20, 32, 48, 32]
    assert api.layout_offsets(api.CUSTOM_POINT, api.LIDAR_AVIA) == [4, 8, 12, 16, 0, -1, 17, 18]
    assert api.layout_offsets(api.VELODYNE_POINT, api.LIDAR_VELO16) == [0, 4, 8, 16, 20, 24, -1, -1]
    assert api.layout_offsets(api.OUSTER_POINT, api.LIDAR_OUST64)[:5] == [0, 4, 8, 16, 20]
