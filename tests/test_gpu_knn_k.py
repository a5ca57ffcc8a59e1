"""KD_TREE::Nearest_Search(point, k, .., max_dist) on the device map (fl_map_nearest_search): any 1 <= k <= 32 and a
device-side max_dist.  Distances and counts equal the numpy rule (knn_rules.py) and the reference bit for bit on every row;
the neighbours equal both on every decided row (the reference's own rules fix them there)."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import knn_rules
from fast_lio_b200 import api, build
from refcalls import digest, row_digests
from refknn import GATED_KS, KS, MAX_DISTS, KnnRefTree, gated_queries, mutation_run, world_queries
from semantics import sort_rows

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_rule(got, rule):
    """Bit for bit: counts and distances on every row, neighbours (and their order) on decided rows."""
    gp, gd, gc = got
    p, d, c, decided = rule
    assert np.array_equal(gc, c)
    assert gd.tobytes() == d.tobytes()
    assert np.array_equal(gp[decided], p[decided])
    for i in np.flatnonzero(~decided):                               # zero past the count there too
        assert (gp[i, gc[i]:] == 0).all()


def check_ref(got, ref, decided):
    gp, gd, gc = got
    rows, d, c = ref
    assert np.array_equal(gc, c)
    assert digest(gd) == d
    assert np.array_equal(row_digests(gp)[decided], rows[decided])


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k"])
def test_matches_reference_and_rule_on_scan_queries(problems, name):
    pr = problems(name)
    q = world_queries(pr)
    r = KnnRefTree(f"knnk_{name}", pr.map_pts)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for k in KS:
        got = t.Nearest_Search_K(q, k)
        rule = knn_rules.nearest(q, pr.map_pts, k)
        check_rule(got, rule)
        check_ref(got, r.nearest_search(q, k), rule[3])


def lattice_map():
    rng = np.random.default_rng(17)
    g = np.arange(-6, 6.01, 0.5, dtype=np.float32)
    X, Y, Z = np.meshgrid(g, g, g[:9], indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel(), np.arange(X.size, dtype=np.float32)], axis=1).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    q = np.zeros((600, 4), dtype=np.float32)
    q[:, :3] = np.round(rng.uniform(-5, 5, (600, 3)) * 8) / 8
    q[:300, 0] += rng.uniform(-0.05, 0.05, 300).astype(np.float32)
    return pts, q


def planted_x_ties():
    """Each query has mirrored pairs of neighbours (x - a, x + a: exactly equidistant) among otherwise distinct ones."""
    rng = np.random.default_rng(19)
    qs, ps = [], []
    for i in range(10):
        for j in range(10):
            c = np.array([10.0 * i - 50, 10.0 * j - 50, float(rng.integers(-3, 4))])
            qs.append(c)
            for m in range(12):
                a = rng.integers(1, 40) / 64.0
                y, z = rng.integers(-40, 41, 2) / 64.0
                ps += [c + [-a, y, z], c + [a, y, z]]
            for m in range(20):
                ps.append(c + rng.uniform(0.3, 4.5, 3) * rng.choice([-1, 1], 3))
    pts = np.zeros((len(ps), 4), dtype=np.float32); pts[:, :3] = np.array(ps, dtype=np.float32); pts[:, 3] = np.arange(len(ps))
    q = np.zeros((len(qs), 4), dtype=np.float32); q[:, :3] = np.array(qs, dtype=np.float32)
    return pts[rng.permutation(len(pts))], q


@pytest.mark.parametrize("which", ["lattice", "planted_x_ties"])
def test_ties_follow_the_rule_on_both_routes(which):
    pts, q = lattice_map() if which == "lattice" else planted_x_ties()
    for cell_dir in (True, False):
        t = api.KdTree(0, 0.5, cell_directory=cell_dir); t.Build(pts)
        inner = 0
        for k in KS:
            rule = knn_rules.nearest(q, pts, k)
            got = t.Nearest_Search_K(q, k)
            check_rule(got, rule)
            d = rule[1][rule[3]]
            inner += int((np.diff(d, axis=1) == 0).any(axis=1).sum())
        assert inner >= 50                                                # the x rule is exercised on decided rows


def test_max_dist_against_rule_and_reference(problems):
    pr = problems("small")
    q = gated_queries(pr)
    r = KnnRefTree("knnk_maxdist_small", pr.map_pts)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for md in MAX_DISTS:
        for k in GATED_KS:
            got = t.Nearest_Search_K(q, k, md)
            rule = knn_rules.nearest(q, pr.map_pts, k, md)
            check_rule(got, rule)
            check_ref(got, r.nearest_search(q, k, md), rule[3])


def test_small_k_is_fl_map_knn_cut_at_max_dist(problems):
    pr = problems("small")
    q = gated_queries(pr)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for k in range(1, 6):
        p5, d5, c5 = t.Nearest_Search(q, k)
        for md in MAX_DISTS:
            md2 = np.float32(np.float32(md) * np.float32(md))
            keep = np.zeros_like(d5, dtype=bool)
            for i in range(len(q)):
                n = 0
                while n < c5[i] and d5[i, n] <= md2:
                    n += 1
                keep[i, :n] = True
            wp = np.where(keep[..., None], p5, 0).astype(np.float32)
            wd = np.where(keep, d5, np.inf).astype(np.float32)
            gp, gd, gc = t.Nearest_Search_K(q, k, md)
            assert gp.tobytes() == wp.tobytes() and gd.tobytes() == wd.tobytes() and np.array_equal(gc, keep.sum(1))


def test_directory_on_and_off(problems):
    pr = problems("avia_2k_50k")
    q = world_queries(pr)
    on = api.KdTree(0, 0.5); on.Build(pr.map_pts)
    off = api.KdTree(0, 0.5, cell_directory=False); off.Build(pr.map_pts)
    on.dir_stats()
    for k in KS:
        a, b = on.Nearest_Search_K(q, k), off.Nearest_Search_K(q, k)
        if k == 8:
            walked = on.dir_stats()["walked"]
            print(f"k = 8: the directory proved {1 - walked / len(q):.3f} of {len(q)} queries")
            assert 0 < walked < len(q)
        assert np.array_equal(a[2], b[2]) and a[1].tobytes() == b[1].tobytes()
        rule = knn_rules.nearest(q, pr.map_pts, k)
        assert np.array_equal(a[0][rule[3]], b[0][rule[3]])                # decided rows: no boundary tie, no equal-x tie
        check_rule(a, rule)
    # far from the map and crowded cells: the walk answers them
    rng = np.random.default_rng(23)
    dense = rng.uniform(-1, 1, (4000, 4)).astype(np.float32)
    sparse = rng.uniform(-60, 60, (3000, 4)).astype(np.float32)
    pts = np.concatenate([dense, sparse + np.float32([0, 0, 200, 0])])
    q2 = np.concatenate([rng.uniform(-2, 2, (200, 4)), rng.uniform(-80, 80, (200, 4)) + [0, 0, 200, 0],
                         rng.uniform(-500, 500, (100, 4))]).astype(np.float32)
    t = api.KdTree(0, 0.5); t.Build(pts)
    for k, md in ((8, np.inf), (32, np.inf), (32, 3.0)):
        check_rule(t.Nearest_Search_K(q2, k, md), knn_rules.nearest(q2, pts, k, md))


def test_edge_cases():
    L = api.load()
    three = np.array([[0, 0, 0, 1], [1, 0, 0, 2], [0, 1, 0, 3]], dtype=np.float32)
    q = np.array([[0.1, 0, 0, 0], [np.nan, 0, 0, 0], [0, np.inf, 0, 0], [0, 0, -np.inf, 0], [5, 5, 5, 0]], dtype=np.float32)
    unbuilt = api.KdTree(0, 0.5)
    for k in (3, 8, 32):
        gp, gd, gc = unbuilt.Nearest_Search_K(q, k)
        assert (gc == 0).all() and (gp == 0).all() and np.isinf(gd).all()
    empty = api.KdTree(0, 0.5); empty.Build(np.zeros((0, 4), np.float32))
    assert (empty.Nearest_Search_K(q, 8)[2] == 0).all()
    t = api.KdTree(0, 0.5); t.Build(three)
    for k in (3, 5, 8, 32):
        gp, gd, gc = t.Nearest_Search_K(q, k)
        assert list(gc) == [3, 0, 0, 0, 3]
        assert np.array_equal(gp[0, 0], three[0]) and np.isinf(gd[0, 3:]).all() and (gp[0, 3:] == 0).all()
        check_rule((gp, gd, gc), knn_rules.nearest(q, three, k))
    out_p, out_d, out_c = np.zeros((5, 33, 4), np.float32), np.zeros((5, 33), np.float32), np.zeros(5, np.int32)
    for k in (0, 33, -1):
        assert L.fl_map_nearest_search(t.h, q, 5, k, np.inf, out_p, out_d, out_c) == -2
        assert b"[1, 32]" in L.fl_last_error()
    raw = ctypes.CDLL(build.LIB).fl_map_nearest_search
    raw.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float] + [ctypes.c_void_p] * 3
    assert raw(t.h, None, 1, 8, np.inf, out_p.ctypes.data, out_d.ctypes.data, out_c.ctypes.data) == -2
    assert raw(t.h, q.ctypes.data, 1, 8, np.inf, out_p.ctypes.data, None, out_c.ctypes.data) == -2
    assert raw(t.h, None, 0, 8, np.inf, None, None, None) == 0


def test_after_map_mutation(problems):
    pr = problems("tiny")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for live, q, answers in mutation_run(pr, t):
        assert np.array_equal(sort_rows(t.flatten()), live)
        for (k, md), ref in answers.items():
            got = t.Nearest_Search_K(q, k, md)
            rule = knn_rules.nearest(q, live, k, md)
            check_rule(got, rule)
            check_ref(got, ref, rule[3])


def test_identical_calls_give_identical_bytes(problems):
    pr = problems("small")
    q = world_queries(pr)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for k, md in ((8, np.inf), (32, 1.0), (5, 0.5)):
        a, b = t.Nearest_Search_K(q, k, md), t.Nearest_Search_K(q, k, md)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_config2_scale_k32(problems):
    pr = problems("velodyne_30k_1m")
    q = np.zeros((len(pr.scan), 4), np.float32)
    rng = np.random.default_rng(41)
    from oracle.bind import lib
    L = lib()
    tmp = np.zeros(3, dtype=np.float32)
    rows = np.sort(rng.choice(len(q), 2000, replace=False))
    for i in range(len(q)):
        L.oracle_transform_point(pr.x_prior, np.ascontiguousarray(pr.scan[i, :3]), tmp)
        q[i, :3] = tmp
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    k = 32
    gp, gd, gc = t.Nearest_Search_K(q, k)
    assert len(q) == 30000 and (gc == k).all()
    _, cand = cKDTree(pr.map_pts[:, :3].astype(np.float64)).query(q[rows, :3].astype(np.float64), k + 16)
    check_rule((gp[rows], gd[rows], gc[rows]), knn_rules.nearest(q[rows], pr.map_pts, k, cand=cand))


def test_cpp_facade_runs_on_the_gpu(problems, tmp_path):
    pr = problems("small")
    exe = tmp_path / "facade_knn_k"
    cmd = ["/usr/bin/g++", "-O1", "-std=c++14", "-Wall", "-Wno-unused",
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "facade"), "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(ROOT, "tests", "facade", "facade_knn_k.cpp"), "-o", str(exe), build.LIB, "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    q = world_queries(pr)[:300]
    pairs = [(8, np.inf), (32, 1.0), (5, 0.7), (16, np.nan)]
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("3i", len(pr.map_pts), len(q), len(pairs)))
        f.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes() + q.tobytes())
        for k, md in pairs:
            f.write(struct.pack("if", k, md))
    run = subprocess.run([str(exe), str(fin), str(fout)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    raw, at = open(fout, "rb").read(), 0
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for k, md in pairs:
        wp, wd, wc = t.Nearest_Search_K(q, k, md)
        for _ in range(2):
            cnt = np.frombuffer(raw, np.int32, len(q), at); at += 4 * len(q)
            assert np.array_equal(cnt, wc)
            for i in range(len(q)):
                n = int(cnt[i])
                p = np.frombuffer(raw, np.float32, 4 * n, at).reshape(-1, 4); at += 16 * n
                d = np.frombuffer(raw, np.float32, n, at); at += 4 * n
                assert p.tobytes() == wp[i, :n].tobytes() and d.tobytes() == wd[i, :n].tobytes()
    assert at == len(raw)
