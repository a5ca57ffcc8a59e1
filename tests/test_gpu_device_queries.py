"""Device-buffer forms of the map queries (fl_map_nearest_search_device, fl_map_box_search_device, fl_map_radius_search_device)
and of Build / Add_Points (fl_map_build_device, fl_map_add_points_device): the same bytes as the host forms, stream-ordered on
the caller's stream, no stray writes, no host synchronisation (so CUDA-graph capturable)."""
import os
import subprocess
import struct

import numpy as np
import pytest

import range_rules as rr
from fast_lio_b200 import api, build
from refknn import mutation_batch, world_queries
from semantics import sort_rows

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KS_ALL = (1, 3, 5, 6, 8, 16, 32)
MDS = (np.inf, 1.0, 0.0, -0.5, np.nan)
SENTINEL = -123456789


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def with_nonfinite(q):
    q = q.copy()
    q[3::17, 0] = np.nan
    q[5::23, 1] = np.inf
    q[7::29, 2] = -np.inf
    return q


def assert_nearest_equal(t, q, k, md):
    want = t.Nearest_Search_K(q, k, md)
    got = [host(x) for x in t.nearest_search_device(dev(q), k, md)]
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (k, md)


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k"])
def test_nearest_equals_host_form(problems, name):
    pr = problems(name)
    q = with_nonfinite(world_queries(pr)[:1500])
    q[:40] = pr.map_pts[np.random.default_rng(3).integers(0, len(pr.map_pts), 40)]        # max_dist = 0 finds these
    for cell_dir in (True, False):
        t = api.KdTree(0, 0.5, cell_directory=cell_dir); t.Build(pr.map_pts)
        for k in KS_ALL:
            for md in MDS:
                assert_nearest_equal(t, q, k, md)


def host_range(t, radius, q, cap):
    L = api.load()
    off = np.zeros(len(q) + 1, np.int32)
    out = np.zeros((max(cap, 1), 4), np.float32)
    fn = L.fl_map_radius_search if radius else L.fl_map_box_search
    total = fn(t.h, np.ascontiguousarray(q, np.float32), len(q), off, out, cap)
    assert total >= 0
    return off, out[:min(total, cap)], total


def raw_range(t, radius, qd, cap, ws_bytes, guard=64):
    """One call of the device form into buffers followed by sentinel-filled guard regions.  Returns (offsets, points, status,
    guards intact)."""
    L = api.load()
    nq = qd.shape[0]
    off = torch.full((nq + 1 + guard,), SENTINEL, dtype=torch.int32, device="cuda")
    pts = torch.full((cap + guard, 4), float(SENTINEL), dtype=torch.float32, device="cuda")
    ws = torch.full((ws_bytes + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
    st = torch.full((2 + guard,), SENTINEL, dtype=torch.int64, device="cuda")
    fn = L.fl_map_radius_search_device if radius else L.fl_map_box_search_device
    rc = fn(t.h, qd.data_ptr(), nq, off.data_ptr(), pts.data_ptr() if cap > 0 else None, cap, ws.data_ptr(), ws_bytes,
            st.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, api.load().fl_last_error()
    o, p, s, w = host(off), host(pts), host(st), host(ws)
    intact = (o[nq + 1:] == SENTINEL).all() and (p[cap:] == SENTINEL).all() and (s[2:] == SENTINEL).all() and (w[ws_bytes:] == 0xA5).all()
    return o[:nq + 1], p[:cap], s[:2], bool(intact)


def check_range_caps(t, radius, q):
    off_h, pts_h, total = host_range(t, radius, q, 1 << 22)
    qd = dev(q)
    npairs = None
    for cap in (0, total // 2, total, total + 7):
        ws_bytes = t.range_workspace_bytes(len(q), npairs if npairs is not None else 8 * len(q) + 4096)
        o, p, s, intact = raw_range(t, radius, qd, cap, ws_bytes)
        if s[0] == -1:                                         # a first guess too small: retry sized from status[1]
            npairs = int(s[1])
            o, p, s, intact = raw_range(t, radius, qd, cap, t.range_workspace_bytes(len(q), npairs))
        npairs = int(s[1])
        assert intact
        assert s[0] == total and np.array_equal(o, off_h)
        assert p[:min(cap, total)].tobytes() == pts_h[:min(cap, total)].tobytes()
        assert (p[min(cap, total):] == SENTINEL).all()         # nothing past the total
    return total


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_range_equals_host_form_at_every_cap(problems, name):
    pr = problems(name)
    boxes, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(5), 600)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    assert check_range_caps(t, False, boxes) > 0
    assert check_range_caps(t, True, spheres) > 0
    # the binding: default (reads the status, retries) and explicit (never synchronises)
    for radius, q in ((False, boxes), (True, spheres)):
        off_h, pts_h, total = host_range(t, radius, q, 1 << 22)
        call = t.radius_search_device if radius else t.box_search_device
        o, p, s = call(dev(q), cap=7)
        assert np.array_equal(host(o), off_h) and host(p).tobytes() == pts_h.tobytes() and host(s)[0] == total


def test_range_after_mutation_sequence(problems):
    pr = problems("small")
    rng = np.random.default_rng(12)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    for step in range(3):
        batch = mutation_batch(rng, pr.map_pts, 1500)
        t.Add_Points(batch[:1000], True)
        t.Add_Points(batch[1000:], False)
        c = pr.map_pts[rng.integers(0, len(pr.map_pts)), :3]
        t.Delete_Point_Boxes(np.array([[*(c - 6), *(c + 6)]], dtype=np.float32))
        boxes, spheres = rr.make_queries(sort_rows(t.flatten()), rng, 300)
        check_range_caps(t, False, boxes)
        check_range_caps(t, True, spheres)


def test_small_workspace_reports_pairs_and_writes_nothing(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    _, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(6), 500)
    off_h, pts_h, total = host_range(t, True, spheres, 1 << 22)
    qd = dev(spheres)
    small = t.range_workspace_bytes(len(spheres), 3)
    o, p, s, intact = raw_range(t, True, qd, total, small)
    assert intact and s[0] == -1 and s[1] > 3
    assert (o == 0).all() and (p == SENTINEL).all()
    o, p, s, intact = raw_range(t, True, qd, total, t.range_workspace_bytes(len(spheres), int(s[1])))
    assert intact and s[0] == total and np.array_equal(o, off_h) and p.tobytes() == pts_h.tobytes()
    # below the fixed part: refused before anything is enqueued
    L = api.load()
    z = torch.zeros(16, dtype=torch.int64, device="cuda")
    rc = L.fl_map_radius_search_device(t.h, qd.data_ptr(), len(spheres), z.data_ptr(), None, 0, z.data_ptr(),
                                       t.range_workspace_bytes(len(spheres), 0) - 1, z.data_ptr(), None)
    assert rc == -2
    # nq = 0: offsets[0] = 0 and the status, nothing else
    o, p, s, intact = raw_range(t, False, torch.zeros((0, 6), dtype=torch.float32, device="cuda"), 4, 0)
    assert intact and list(o) == [0] and list(s) == [0, 0] and (p == SENTINEL).all()


def test_query_on_a_busy_stream_sees_the_map_before_a_later_mutation(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    _, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(7), 400)
    q = world_queries(pr)[:800]
    want_r = host_range(t, True, spheres, 1 << 22)
    want_k = t.Nearest_Search_K(q, 8)
    ws = t.range_workspace(len(spheres), 1 << 16)
    qd, sd = dev(q), dev(spheres)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                         # ~0.1 s: the queries below are still queued when Add_Points runs
        k_out = t.nearest_search_device(qd, 8)
        r_out = t.radius_search_device(sd, cap=len(pr.map_pts), workspace=ws)
    batch = mutation_batch(np.random.default_rng(8), q, 2000)  # lands among the queries' neighbours
    t.Add_Points(batch, False)
    side.synchronize()
    assert all(host(g).tobytes() == w.tobytes() for g, w in zip(k_out, want_k))
    o, p, s = (host(x) for x in r_out)
    assert s[0] == want_r[2] and np.array_equal(o, want_r[0]) and p[:s[0]].tobytes() == want_r[1].tobytes()
    assert t.Nearest_Search_K(q, 8)[1].tobytes() != want_k[1].tobytes()       # the mutation did change the answer


def test_query_after_filter_run_and_map_incremental(problems):
    pr = problems("avia_2k_50k")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)
    q = world_queries(pr)
    qd = dev(q)
    f.upload_scan(pr.scan); f.upload_state(pr.x_prior, pr.P_prior, pr.R)
    f.run()                                                   # asynchronous on the handle's stream
    got = t.nearest_search_device(qd, 16, 1.0)
    assert all(host(g).tobytes() == w.tobytes() for g, w in zip(got, t.Nearest_Search_K(q, 16, 1.0)))
    f.download_state()
    f.map_incremental(0.5, True)
    for k in (5, 16):
        got = t.nearest_search_device(qd, k)
        assert all(host(g).tobytes() == w.tobytes() for g, w in zip(got, t.Nearest_Search_K(q, k)))


def test_graph_capture_and_replay(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    rng = np.random.default_rng(9)
    base = world_queries(pr)[:1000]
    q5, q16 = dev(base), dev(base[::-1].copy())
    _, spheres = rr.make_queries(pr.map_pts, rng, 300)
    spheres[:, 3] = 1.0
    sd = dev(spheres)
    ws = t.range_workspace(len(spheres), 1 << 16)
    cap = len(pr.map_pts) * 4
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                              # warm-up outside capture
        t.nearest_search_device(q5, 5); t.radius_search_device(sd, cap=cap, workspace=ws)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a = t.nearest_search_device(q5, 5)
        b = t.nearest_search_device(q16, 16, 2.0)
        c = t.radius_search_device(sd, cap=cap, workspace=ws)
    for rep in range(3):
        nq = with_nonfinite(base + rng.normal(0, 0.5, base.shape).astype(np.float32))
        ns = spheres.copy(); ns[:, :3] += rng.normal(0, 0.5, (len(ns), 3)).astype(np.float32)
        q5.copy_(dev(nq)); q16.copy_(dev(nq[::-1].copy())); sd.copy_(dev(ns))
        g.replay()
        torch.cuda.synchronize()
        assert all(host(x).tobytes() == w.tobytes() for x, w in zip(a, t.Nearest_Search_K(nq, 5)))
        assert all(host(x).tobytes() == w.tobytes() for x, w in zip(b, t.Nearest_Search_K(nq[::-1].copy(), 16, 2.0)))
        off_h, pts_h, total = host_range(t, True, ns, cap)
        o, p, s = (host(x) for x in c)
        assert s[0] == total and np.array_equal(o, off_h) and p[:total].tobytes() == pts_h.tobytes()


def test_dir_stats_and_determinism(problems):
    pr = problems("avia_2k_50k")
    q = with_nonfinite(world_queries(pr))
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    qd = dev(q)
    walked_any = 0
    for k, md in ((5, np.inf), (3, 1.0), (16, np.inf), (32, 0.5)):
        t.dir_stats()
        t.Nearest_Search_K(q, k, md)
        walked_host = t.dir_stats()["walked"]
        a = t.nearest_search_device(qd, k, md)
        torch.cuda.synchronize()
        walked_dev = t.dir_stats()["walked"]
        assert walked_dev == walked_host, (k, walked_host, walked_dev)
        walked_any += walked_host
        b = t.nearest_search_device(qd, k, md)
        assert all(host(x).tobytes() == host(y).tobytes() for x, y in zip(a, b))
    assert walked_any > 0                                      # the walk count is exercised
    _, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(4), 500)
    r1 = [host(x) for x in t.radius_search_device(dev(spheres))]
    r2 = [host(x) for x in t.radius_search_device(dev(spheres))]
    assert all(x.tobytes() == y.tobytes() for x, y in zip(r1, r2))


def test_arguments():
    L = api.load()
    pts = np.random.default_rng(1).uniform(-5, 5, (2000, 4)).astype(np.float32)
    t = api.KdTree(0, 0.5); t.Build(pts)
    qh = pts[:10].copy()
    qd = dev(qh)
    with pytest.raises(ValueError):
        t.nearest_search_device(torch.from_numpy(qh), 5)               # a CPU tensor
    with pytest.raises(TypeError):
        t.nearest_search_device(qd.double(), 5)
    with pytest.raises(ValueError):
        t.box_search_device(qd)                                        # (n, 4) is not a box
    with pytest.raises(ValueError):
        t.nearest_search_device(qd, 33)
    s = torch.cuda.current_stream().cuda_stream
    p, d, c = (torch.zeros(10 * 33 * 4, device="cuda"), torch.zeros(10 * 33, device="cuda"), torch.zeros(10, dtype=torch.int32, device="cuda"))
    for k in (0, 33):
        assert L.fl_map_nearest_search_device(t.h, qd.data_ptr(), 10, k, np.inf, p.data_ptr(), d.data_ptr(), c.data_ptr(), s) == -2
    hp, hd, hc = np.zeros((10, 5, 4), np.float32), np.zeros((10, 5), np.float32), np.zeros(10, np.int32)
    assert L.fl_map_nearest_search_device(t.h, qh.ctypes.data, 10, 5, np.inf, p.data_ptr(), d.data_ptr(), c.data_ptr(), s) == -2
    assert L.fl_map_nearest_search_device(t.h, qd.data_ptr(), 10, 5, np.inf, hp.ctypes.data, d.data_ptr(), c.data_ptr(), s) == -2
    assert L.fl_map_nearest_search_device(t.h, qd.data_ptr(), 10, 5, np.inf, p.data_ptr(), hd.ctypes.data, c.data_ptr(), s) == -2
    assert L.fl_map_nearest_search_device(t.h, qd.data_ptr(), 10, 5, np.inf, p.data_ptr(), d.data_ptr(), hc.ctypes.data, s) == -2
    assert L.fl_map_nearest_search_device(t.h, None, 10, 5, np.inf, p.data_ptr(), d.data_ptr(), c.data_ptr(), s) == -2
    assert L.fl_map_nearest_search_device(t.h, qd.data_ptr() + 4, 10, 5, np.inf, p.data_ptr(), d.data_ptr(), c.data_ptr(), s) == -2   # misaligned
    assert L.fl_map_nearest_search_device(t.h, None, 0, 5, np.inf, None, None, None, s) == 0
    off = torch.zeros(11, dtype=torch.int32, device="cuda")
    st = torch.zeros(2, dtype=torch.int64, device="cuda")
    ws = t.range_workspace(10, 100)
    nbytes = ws.numel()
    boxes_h = np.concatenate([pts[:10, :3] - 1, pts[:10, :3] + 1], axis=1).astype(np.float32)
    bd = dev(boxes_h)
    assert L.fl_map_box_search_device(t.h, boxes_h.ctypes.data, 10, off.data_ptr(), p.data_ptr(), 4, ws.data_ptr(), nbytes, st.data_ptr(), s) == -2
    assert L.fl_map_box_search_device(t.h, bd.data_ptr(), 10, off.data_ptr(), hp.ctypes.data, 4, ws.data_ptr(), nbytes, st.data_ptr(), s) == -2
    assert L.fl_map_box_search_device(t.h, bd.data_ptr(), 10, off.data_ptr(), p.data_ptr(), 4, None, nbytes, st.data_ptr(), s) == -2
    assert L.fl_map_box_search_device(t.h, bd.data_ptr(), 10, off.data_ptr(), p.data_ptr(), 4, ws.data_ptr(), nbytes, None, s) == -2
    assert L.fl_map_box_search_device(t.h, bd.data_ptr(), 10, off.data_ptr(), p.data_ptr(), -1, ws.data_ptr(), nbytes, st.data_ptr(), s) == -2
    assert L.fl_map_box_search_device(t.h, bd.data_ptr(), 10, off.data_ptr(), p.data_ptr(), 4, ws.data_ptr(), nbytes, st.data_ptr(), s) == 0
    assert L.fl_map_build_device(t.h, pts.ctypes.data, len(pts), s) == -2
    assert L.fl_map_add_points_device(t.h, pts.ctypes.data, len(pts), 1, s) == -2
    assert t.validnum() == len(pts)
    if torch.cuda.device_count() < 2:
        pytest.skip("the wrong-device case needs a second GPU")
    other = qd.to("cuda:1")
    assert L.fl_map_nearest_search_device(t.h, other.data_ptr(), 10, 5, np.inf, p.data_ptr(), d.data_ptr(), c.data_ptr(), s) == -2
    with pytest.raises(ValueError):
        t.nearest_search_device(other, 5)


def test_device_input_build_and_add_points(problems):
    pr = problems("small")
    rng = np.random.default_rng(21)
    a = api.KdTree(0, 0.5); a.Build(pr.map_pts)
    b = api.KdTree(0, 0.5); b.build_device(dev(pr.map_pts))
    q = world_queries(pr)[:1000]

    def same():
        assert a.validnum() == b.validnum() and a.size() == b.size()
        assert np.array_equal(sort_rows(a.flatten()), sort_rows(b.flatten()))
        for k in (5, 16):
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a.Nearest_Search_K(q, k), b.Nearest_Search_K(q, k)))

    same()
    for step in range(3):
        batch = mutation_batch(rng, pr.map_pts, 3000)
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):                          # the input is produced on the caller's stream, read in order
            bd = dev(batch[:2000]) * 1.0
            assert b.add_points_device(bd, True) == a.Add_Points(batch[:2000], True)
        assert b.add_points_device(dev(batch[2000:]), False) == a.Add_Points(batch[2000:], False)
        same()
    empty = torch.zeros((0, 4), dtype=torch.float32, device="cuda")
    assert b.add_points_device(empty, True) == 0
    b.build_device(empty)
    assert b.validnum() == 0


def test_config2_scale(problems):
    pr = problems("velodyne_30k_1m")
    q = world_queries(pr)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    assert len(q) == 30000
    assert_nearest_equal(t, q, 32, np.inf)
    rng = np.random.default_rng(2)
    c = (pr.map_pts[rng.integers(0, len(pr.map_pts), 30000), :3] + rng.normal(0, 0.5, (30000, 3))).astype(np.float32)
    spheres = np.concatenate([c, np.ones((30000, 1), np.float32)], axis=1)
    off_h, pts_h = t.Radius_Search(c, 1.0)
    o, p, s = (host(x) for x in t.radius_search_device(dev(spheres)))
    assert np.array_equal(o, off_h) and p.tobytes() == pts_h.tobytes() and s[0] == len(pts_h)


def test_plain_c_program_on_its_own_stream(problems, tmp_path):
    pr = problems("small")
    exe = tmp_path / "device_queries"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "facade", "device_queries.cu"),
           "-o", str(exe), build.LIB, "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    boxes, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(14), 300)
    q = with_nonfinite(world_queries(pr)[:500])
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", len(pr.map_pts), len(q), len(boxes), len(spheres)))
        for a in (pr.map_pts, q, boxes, spheres):
            f.write(np.ascontiguousarray(a, np.float32).tobytes())
    run = subprocess.run([str(exe), str(fin)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "all equal" in run.stdout, run.stdout
