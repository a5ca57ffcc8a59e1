"""The drop-in boundary, EXECUTED on a GPU from C++ and from C (not through ctypes): tests/facade/facade_run.cpp drives the
KD_TREE<PointType> and esekf facades the way src/laserMapping.cpp does; examples/pipeline.c walks a scan through the plain-C ABI.
The C++ run must give the same state as the ctypes path bit for bit (same library, same inputs) and match the CPU oracle."""
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth
from refcalls import RefTree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build_facade(tmp_path):
    exe = tmp_path / "facade_run"
    cmd = ["/usr/bin/g++", "-O1", "-std=c++14", "-Wall", "-Wno-unused",
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "facade"), "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(ROOT, "tests", "facade", "facade_run.cpp"), "-o", str(exe), build.LIB, "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


@pytest.mark.parametrize("name", ["small", "avia_2k_50k"])
def test_cpp_facades_run_on_the_gpu(problems, tmp_path, name):
    pr = problems(name)
    exe = _build_facade(tmp_path)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", len(pr.map_pts), len(pr.scan), pr.cfg.max_iter, 0))
        f.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes()); f.write(np.ascontiguousarray(pr.scan, np.float32).tobytes())
        f.write(np.ascontiguousarray(pr.x_prior, np.float64).tobytes()); f.write(np.ascontiguousarray(pr.P_prior, np.float64).tobytes())
        f.write(struct.pack("d", pr.R))
    run = subprocess.run([str(exe), str(fin), str(fout)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    raw = open(fout, "rb").read()
    x = np.frombuffer(raw, np.float64, 26, 0); P = np.frombuffer(raw, np.float64, 529, 26 * 8).reshape(23, 23)
    off = (26 + 529 + 1) * 8
    size, validnum, add_ret, del_ret, n_removed, nearest_total, n_knn = struct.unpack_from("7i", raw, off)
    off += 28
    knn_d2 = np.frombuffer(raw, np.float32, n_knn * 5, off).reshape(n_knn, 5); off += n_knn * 20
    knn_pts = np.frombuffer(raw, np.float32, n_knn * 20, off).reshape(n_knn, 5, 4)
    # ---- the same calls through the ctypes harness
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    q = pr.map_pts[(np.arange(n_knn) * 7) % len(pr.map_pts)].copy()
    q[:, 0] += np.float32(0.11); q[:, 1] -= np.float32(0.07)
    gp, gd, gc = t.Nearest_Search(q, 5)
    assert np.array_equal(gd, knn_d2) and np.array_equal(gp, knn_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    xa, Pa, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert np.array_equal(xa, x) and np.array_equal(Pa, P)                     # same library, same inputs: same bits
    assert int(f.nearest(len(pr.scan))[1].sum()) == nearest_total
    t.acquire_removed_points()
    to_add = pr.map_pts[:500].copy(); to_add[:, 0] += np.float32(0.05); to_add[:, 2] += np.float32(0.02)
    assert t.Add_Points(to_add, True) == add_ret
    assert t.Delete_Point_Boxes(np.array([[-3, -3, -3, 3, 3, 3]], np.float32)) == del_ret
    assert len(t.acquire_removed_points()) == n_removed == del_ret
    assert (t.size(), t.validnum()) == (size, validnum)
    # ---- and the CPU oracle (north-star tolerance)
    o = RefTree(f"update_{name}_e0", pr.map_pts).update_iterated(pr.scan, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, 0)
    assert np.abs(x[:3] - o.x[:3]).max() <= 1e-4 and np.abs(x[3:7] - o.x[3:7]).max() <= 1e-4
    assert np.abs(x[11:] - o.x[11:]).max() <= 1e-4


def test_c_example_runs_on_the_gpu(tmp_path):
    exe = tmp_path / "pipeline_example"
    cmd = ["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "examples", "pipeline.c"), build.LIB, "-lm", "-o", str(exe), "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "map_incremental" in run.stdout and "down-sampled" in run.stdout
    # the floor was 3 cm off: the update must have pulled the state towards it
    z = float(run.stdout.split("state z =")[1].split("m")[0])
    assert abs(abs(z) - 0.03) < 0.01


def test_facade_reports_failures(tmp_path):
    """k > 5 is an error, not a silent clamp (ADVICE r1); the device is selectable."""
    src = tmp_path / "k.cpp"
    src.write_text('''#include <ikd-Tree/ikd_Tree.h>
int main() {
    KD_TREE<pcl::PointXYZINormal>::set_default_device(0);
    KD_TREE<pcl::PointXYZINormal> t(0.5f, 0.6f, 0.5f);
    if (!t.ok() || t.device() != 0) return 1;
    KD_TREE<pcl::PointXYZINormal>::PointVector v(40), out;
    for (int i = 0; i < 40; i++) { v[i].x = 0.3f * i; v[i].y = 0.1f * (i % 7); v[i].z = 0.f; }
    t.Build(v);
    std::vector<float> d;
    t.Nearest_Search(v[3], 5, out, d);
    if (out.size() != 5 || t.failed()) return 2;
    t.Nearest_Search(v[3], 8, out, d);
    if (!out.empty() || !t.failed()) return 3;
    return 0;
}''')
    exe = tmp_path / "k"
    cmd = ["/usr/bin/g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle", "shim"), str(src), "-o", str(exe),
           build.LIB, "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "not supported" in run.stderr
