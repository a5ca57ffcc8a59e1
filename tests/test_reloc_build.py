"""CPU: the relocalisation (fl_reloc_expand_grid_device, fl_filter_reserve_reloc, fl_filter_relocalize_device) is exported,
declared and bound, its ctypes structs have the header's layout, its kernels' registers and spills are what ptxas reported when
they were written, and the numpy restatement of the grid agrees with a host build of the formula k_reloc_expand runs.  The pinned
SASS of the existing kernels is checked, unchanged, by test_map_async_build.py."""
import os
import re
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build
from reloc_rules import assert_quat_ulp, expand
from test_device_queries_build import spills
from test_frontend_device_build import frames
from test_map_async_build import cubin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fl_reloc_expand_grid_device", "fl_filter_reserve_reloc", "fl_filter_relocalize_device"]


def test_symbols_exported_declared_and_bound():
    assert os.path.exists(build.LIB), "run `python -m fast_lio_b200.build` first"
    out = subprocess.run(["nm", "-D", "--defined-only", build.LIB], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (fl_\w+)", out))
    hdr = open(os.path.join(ROOT, "include", "fastlio_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert s in exported, s
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in api.SYMBOLS, s


def test_ctypes_structs_match_the_header(tmp_path):
    """sizeof and offsetof of every field, from a C program compiled against the header."""
    import ctypes as C
    structs = {"fl_reloc_grid_t": (api.RelocGrid, ["n", "step"]),
               "fl_reloc_params_t": (api.RelocParams, ["keep", "stride", "r_inlier", "min_effct"]),
               "fl_reloc_row_t": (api.RelocRow, ["hyp", "inliers", "status", "passes", "effct", "pad", "res_sum"])}
    lines = []
    for name, (_, fields) in structs.items():
        lines.append(f'printf("{name} size %zu\\n", sizeof({name}));')
        lines += [f'printf("{name} {f} %zu\\n", offsetof({name}, {f}));' for f in fields]
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"fastlio_b200.h\"\nint main(void) {\n" + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    got = dict((" ".join(l.split()[:2]), int(l.split()[2])) for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                                       check=True).stdout.splitlines())
    for name, (cls, fields) in structs.items():
        assert got[f"{name} size"] == C.sizeof(cls), name
        for f in fields:
            assert got[f"{name} {f}"] == getattr(cls, f).offset, (name, f)
    assert api.RELOC_ROW.itemsize == C.sizeof(api.RelocRow)
    for f in api.RELOC_ROW.names:
        assert api.RELOC_ROW.fields[f][1] == getattr(api.RelocRow, f).offset, f


def test_row_decoder():
    import ctypes as C
    rows = []
    for s in range(3):
        r = api.RelocRow(7 * s, 100 - s, -4 * (s % 2), s + 1, 50 + s, 0, 0.25 * s)
        rows.append(np.frombuffer(bytes(r), np.uint8))
    got = api.decode_reloc_rows(np.stack(rows))
    assert list(got["hyp"]) == [0, 7, 14] and list(got["status"]) == [0, -4, 0] and list(got["res_sum"]) == [0.0, 0.25, 0.5]
    assert list(got["inliers"]) == [100, 99, 98] and list(got["passes"]) == [1, 2, 3] and list(got["effct"]) == [50, 51, 52]
    assert C.sizeof(api.RelocRow) == 32


@pytest.fixture(scope="module")
def reloc_log(tmp_path_factory):
    return cubin("reloc.cu", tmp_path_factory)[0]


def test_kernel_footprint(reloc_log):
    """Registers and spills of the new kernels as ptxas -v reports them (nvcc 12.9).  k_reloc_screen inlines knn_block -- the
    cell-directory search and the BVH walk of k_knn_batch -- whose walk state ptxas spills in part; the others spill nothing."""
    sp, fr = spills(reloc_log), frames(reloc_log)
    names = {k: n for n in ("k_reloc_expand", "k_reloc_screen", "k_reloc_keys", "k_reloc_gather", "k_reloc_rank") for k in sp if n in k}
    assert sorted(names.values()) == sorted(["k_reloc_expand", "k_reloc_screen", "k_reloc_keys", "k_reloc_gather", "k_reloc_rank"]), names
    for k, n in names.items():
        if n == "k_reloc_screen":
            assert sp[k] <= 344 + 64, (k, sp[k])
            assert fr[k][1] <= 64, (k, fr[k])
        else:
            assert sp[k] == 0, (k, sp[k])


def test_numpy_grid_equals_the_host_build_of_the_formula(tmp_path):
    exe = tmp_path / "reloc_expand_harness"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "kernels", "reloc_expand_harness.cpp"), "-o", str(exe)], check=True)
    rng = np.random.default_rng(4)
    from fast_lio_b200 import synth
    for case in range(4):
        prior = synth.make_prior(synth.true_state("avia"), seed=case)[0]
        if case >= 2:                                           # gravity off the world z axis
            g = rng.normal(0, 1, 3)
            prior[23:26] = 9.809 * g / np.linalg.norm(g)
        n = np.array([(3, 2, 1, 5), (1, 1, 1, 36), (4, 3, 2, 3), (2, 5, 1, 7)][case], np.int32)
        step = np.array([0.5, 0.25, 0.1, np.radians(10.0)] if case != 3 else [0.0, 0.3, 0.0, 0.2], np.float64)
        raw = subprocess.run([str(exe)], input=prior.tobytes() + n.tobytes() + step.tobytes(), capture_output=True, check=True).stdout
        host = np.frombuffer(raw, np.float64).reshape(-1, 26)
        want = expand(prior, n, step)
        assert host.shape == want.shape
        assert host[:, :3].tobytes() == want[:, :3].tobytes(), case
        assert host[:, 7:].tobytes() == want[:, 7:].tobytes(), case
        assert_quat_ulp(host[:, 3:7], want[:, 3:7])
