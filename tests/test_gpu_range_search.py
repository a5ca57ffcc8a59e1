"""KD_TREE::Box_Search / Radius_Search on the device map (fl_map_box_search / fl_map_radius_search): the answer is the literal
per-point rule (range_rules.py) bit for bit, boxes equal the reference's answers, and spheres differ from the reference only
on points of the band B = {d2 > fl(r * r) and sqrtf(d2) <= r}, where the reference decides by the shape of its tree."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

import range_rules as rr
from fast_lio_b200 import api, build
from refcalls import rows_digest
from refrange import RangeRefTree
from semantics import sort_rows

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_batch(rng, base_pts, n):
    """New points: most near existing map points (they compete in their voxel), a fifth in fresh space."""
    b = base_pts[rng.integers(0, len(base_pts), n)].copy()
    b[:, :3] += rng.normal(0, 0.3, (n, 3)).astype(np.float32)
    far = rng.random(n) < 0.2
    b[far, :3] += rng.uniform(5, 30, (int(far.sum()), 3)).astype(np.float32)
    b[:, 3] = rng.uniform(100, 200, n).astype(np.float32)
    return np.ascontiguousarray(b.astype(np.float32))


def assert_literal(offsets, pts, want):
    got = rr.split(offsets, pts)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.tobytes() == w.tobytes(), f"query {i}: {len(g)} points, the rule gives {len(w)}"
    return got


def check_radius_against_reference(got, ref, band):
    """device xor reference lies in the band, query by query; returns how many band points the two answers disagree on."""
    differ = 0
    for g, r, b in zip(got, ref, band):
        only_g = g[~rr.members(g, r)]
        only_r = r[~rr.members(r, g)]
        extra = np.concatenate([only_g, only_r])
        assert rr.members(extra, b).all(), "device and reference differ outside the band"
        differ += len(extra)
    return differ


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_box_search_matches_rule_and_reference(problems, name):
    pr = problems(name)
    boxes, _ = rr.make_queries(pr.map_pts, np.random.default_rng(5), 1000)
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    off, pts = g.Box_Search(boxes)
    got = assert_literal(off, pts, rr.box_sets(boxes, pr.map_pts))
    r = RangeRefTree(f"range_box_{name}", pr.map_pts)
    cnt, dig = r.box_search(boxes)
    assert list(np.diff(off)) == list(cnt)
    assert [rows_digest(x) for x in got] == dig


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_radius_search_matches_rule_and_reference_outside_the_band(problems, name):
    pr = problems(name)
    _, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(6), 1000)
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    off, pts = g.Radius_Search(spheres[:, :3], spheres[:, 3])
    lit, band = rr.radius_sets(spheres, pr.map_pts)
    got = assert_literal(off, pts, lit)
    ref = RangeRefTree(f"range_radius_{name}", pr.map_pts).radius_search(spheres, pr.map_pts)
    differ = check_radius_against_reference(got, ref, band)
    print(f"{name}: |B| = {sum(len(b) for b in band)} (query, point) pairs, device and reference differ on {differ}")


def test_degenerate_queries_find_nothing():
    rng = np.random.default_rng(8)
    pts = rng.uniform(-5, 5, (3000, 4)).astype(np.float32)
    boxes = np.array([[np.nan, -5, -5, 5, 5, 5], [-5, -5, -5, 5, np.nan, 5], [1, -5, -5, -1, 5, 5], [0, 0, 0, 0, 0, 0],
                      [-5, -5, -5, 5, 5, 5]], dtype=np.float32)
    spheres = np.array([[0, 0, 0, -1], [np.nan, 0, 0, 3], [0, 0, 0, np.nan], [0, 0, 0, 3]], dtype=np.float32)
    unbuilt = api.KdTree(0, 0.5)
    assert list(unbuilt.Box_Search(boxes)[0]) == [0] * 6
    assert list(unbuilt.Radius_Search(spheres[:, :3], spheres[:, 3])[0]) == [0] * 5
    g = api.KdTree(0, 0.5); g.Build(pts)
    off, _ = g.Box_Search(boxes)
    assert list(np.diff(off)) == [0, 0, 0, 0, len(pts)]
    off, got = g.Radius_Search(spheres[:, :3], spheres[:, 3])
    assert_literal(off, got, rr.radius_sets(spheres, pts)[0])
    assert list(np.diff(off)[:3]) == [0, 0, 0] and off[4] > off[3]
    assert list(g.Box_Search(np.zeros((0, 6), np.float32))[0]) == [0]


def test_points_on_the_sphere_and_on_the_faces():
    c = np.array([1.0, 2.0, 3.0], dtype=np.float32)
    pts = np.array([[*(c + [0.5, 0, 0]), 1], [*(c - [0, 0.5, 0]), 2], [*(c + [0, 0, 0.5]), 3], [*(c + [0.5, 0.5, 0]), 4],
                    [*c, 5]], dtype=np.float32)
    g = api.KdTree(0, 0.5); g.Build(pts)
    r = RangeRefTree("range_exact_boundary", pts)
    off, got = g.Radius_Search(c[None], 0.5)
    want = sort_rows(pts[[0, 1, 2, 4]])                       # d2 == r * r exactly: on the sphere is inside
    assert np.array_equal(sort_rows(got), want)
    assert np.array_equal(r.radius_search(np.array([[*c, 0.5]], dtype=np.float32), pts)[0], want)
    box = np.array([[1.0, 2.0, 3.0, 1.5, 2.5, 4.0]], dtype=np.float32)
    off, got = g.Box_Search(box)                              # min faces are in, max faces are out
    assert np.array_equal(sort_rows(got), sort_rows(pts[[2, 4]]))
    assert r.box_search(box)[1][0] == rows_digest(pts[[2, 4]])


def test_whole_map_box_is_flatten(problems):
    pr = problems("small")
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    g.Delete_Point_Boxes(np.array([[-5, -5, -5, 5, 5, 5]], dtype=np.float32))
    off, pts = g.Box_Search(np.array([[-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf]], dtype=np.float32))
    assert np.array_equal(sort_rows(pts), sort_rows(g.flatten())) and off[1] == g.validnum()


def test_range_search_after_map_mutation(problems):
    """Add_Points(.., true) / Add_Points(.., false) / Delete_Point_Boxes on both maps: the answers keep matching, and deleted or
    down-sampled-away points never appear."""
    pr = problems("small")
    rng = np.random.default_rng(12)
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    r = RangeRefTree("range_mutation", pr.map_pts)
    everything = np.array([[-1e9, -1e9, -1e9, 1e9, 1e9, 1e9]], dtype=np.float32)
    for step in range(3):
        batch = make_batch(rng, pr.map_pts, 1500)
        assert g.Add_Points(batch[:1000], True) == r.add(batch[:1000], True)
        assert g.Add_Points(batch[1000:], False) == r.add(batch[1000:], False)
        c = pr.map_pts[rng.integers(0, len(pr.map_pts)), :3]
        box = np.array([[*(c - 6), *(c + 6)]], dtype=np.float32)
        assert g.Delete_Point_Boxes(box) == r.delete_boxes(box)
        live = sort_rows(g.flatten())                                   # sorted: the queries below must not depend on slot order
        assert rows_digest(live) == r.flatten_digest()
        boxes, spheres = rr.make_queries(live, rng, 300)
        boxes = np.concatenate([boxes, box, everything])
        off, pts = g.Box_Search(boxes)
        got = assert_literal(off, pts, rr.box_sets(boxes, live))
        assert len(got[-2]) == 0 and len(got[-1]) == len(live)         # nothing of the deleted box; no dead slot anywhere
        assert [rows_digest(x) for x in got] == r.box_search(boxes)[1]
        off, pts = g.Radius_Search(spheres[:, :3], spheres[:, 3])
        lit, band = rr.radius_sets(spheres, live)
        check_radius_against_reference(assert_literal(off, pts, lit), r.radius_search(spheres, live), band)


def test_identical_calls_give_identical_bytes(problems):
    pr = problems("small")
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    boxes, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(3), 2000)
    for call in (lambda: g.Box_Search(boxes), lambda: g.Radius_Search(spheres[:, :3], spheres[:, 3])):
        o1, p1 = call()
        o2, p2 = call()
        assert o1.tobytes() == o2.tobytes() and p1.tobytes() == p2.tobytes()


def test_small_cap_reports_the_total_and_the_retry_fills(problems):
    pr = problems("small")
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    boxes, _ = rr.make_queries(pr.map_pts, np.random.default_rng(4), 200)
    full_off, full = g.Box_Search(boxes)
    total = int(full_off[-1])
    assert total > 100
    L = api.load()
    off = np.full(len(boxes) + 1, -7, dtype=np.int32)
    out = np.zeros((100, 4), dtype=np.float32)
    assert L.fl_map_box_search(g.h, boxes, len(boxes), off, out, 100) == total
    assert np.array_equal(off, full_off) and np.array_equal(out, full[:100])     # offsets in full, the first cap points
    assert L.fl_map_box_search(g.h, boxes, len(boxes), off, np.zeros((1, 4), np.float32), 0) == total
    o2, p2 = g.Box_Search(boxes, cap=10)                                            # the binding retries once
    assert np.array_equal(o2, full_off) and np.array_equal(p2, full)
    raw = ctypes.CDLL(build.LIB)                                                    # null buffers are refused
    fn = raw.fl_map_radius_search
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    q = np.zeros((1, 4), np.float32)
    assert fn(g.h, q.ctypes.data, 1, None, out.ctypes.data, 100) == -2
    assert fn(g.h, None, 1, off.ctypes.data, out.ctypes.data, 100) == -2
    assert fn(g.h, q.ctypes.data, 1, off.ctypes.data, None, 100) == -2


def test_one_whole_map_query_among_ten_thousand_small_ones(problems):
    """Work is spread over (query, leaf) pairs: one query that covers the whole map next to 10 000 small ones."""
    pr = problems("small")
    rng = np.random.default_rng(10)
    g = api.KdTree(0, 0.5); g.Build(pr.map_pts)
    n = 10000
    c = pr.map_pts[rng.integers(0, len(pr.map_pts), n), :3] + rng.normal(0, 0.5, (n, 3)).astype(np.float32)
    spheres = np.zeros((n + 1, 4), dtype=np.float32)
    spheres[1:, :3] = c
    spheres[1:, 3] = rng.uniform(0.2, 1.5, n).astype(np.float32)
    spheres[0] = [*pr.map_pts[:, :3].mean(0), 1e4]
    off, pts = g.Radius_Search(spheres[:, :3], spheres[:, 3])
    assert off[1] == len(pr.map_pts)
    assert_literal(off, pts, rr.radius_sets(spheres, pr.map_pts)[0])
    boxes = np.concatenate([np.array([[-1e4] * 3 + [1e4] * 3], np.float32),
                            np.concatenate([c - 0.7, c + 0.7], axis=1).astype(np.float32)])
    off, pts = g.Box_Search(boxes)
    assert off[1] == len(pr.map_pts)
    assert_literal(off, pts, rr.box_sets(boxes, pr.map_pts))


def test_cpp_facade_range_queries_run_on_the_gpu(problems, tmp_path):
    pr = problems("small")
    exe = tmp_path / "facade_range"
    cmd = ["/usr/bin/g++", "-O1", "-std=c++14", "-Wall", "-Wno-unused",
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "facade"), "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(ROOT, "tests", "facade", "facade_range.cpp"), "-o", str(exe), build.LIB, "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    boxes, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(14), 200)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("3i", len(pr.map_pts), len(boxes), len(spheres)))
        for a in (pr.map_pts, boxes, spheres):
            f.write(np.ascontiguousarray(a, np.float32).tobytes())
    run = subprocess.run([str(exe), str(fin), str(fout)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    raw, at = open(fout, "rb").read(), 0
    sets = []
    for n in (len(boxes), len(spheres), len(boxes), len(spheres)):
        cnt = np.frombuffer(raw, np.int32, n, at); at += 4 * n
        pts = np.frombuffer(raw, np.float32, 4 * int(cnt.sum()), at).reshape(-1, 4); at += 16 * int(cnt.sum())
        sets.append((np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32), pts))
    assert at == len(raw)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    want_box = t.Box_Search(boxes)
    want_rad = t.Radius_Search(spheres[:, :3], spheres[:, 3])
    for (o, p), (wo, wp) in zip(sets, [want_box, want_rad, want_box, want_rad]):
        assert np.array_equal(o, wo) and p.tobytes() == wp.tobytes()       # same points, same order
