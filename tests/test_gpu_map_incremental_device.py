"""Device forms of Add_Points and map_incremental (fl_map_add_points_async, fl_filter_map_incremental_device, fl_map_maintain):
the results of the host forms, on the caller's stream, without a host synchronisation, capturable with the update, and never
half applied."""
import numpy as np
import pytest

from fast_lio_b200 import api, synth
from refcalls import RefTree, rows_digest
from semantics import sort_rows

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = 0, -2, -4, -5


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def world_points(pr, scan):
    x = pr.x_prior
    qx, qy, qz, qw = x[3:7]
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw)],
                  [2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw)],
                  [2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)]])
    q = np.array(scan, dtype=np.float32).copy()
    q[:, :3] = (scan[:, :3].astype(np.float64) @ R.T + x[:3]).astype(np.float32)
    return q


def twins(pr, n=2, **kw):
    trees = [api.KdTree(0, 0.5) for _ in range(n)]
    for t in trees:
        t.Build(pr.map_pts)
    return trees


def same_map(a, b, queries):
    """validnum, size and the point set; where neither side re-packed or re-listed also the leaf geometry of fl_map_stats and
    fl_map_dir_stats (the overflow leaves and pool use are left out: two inserts racing for one chain link may leave a fresh leaf
    unused, on either form), and k-NN distances and counts in every case."""
    assert a.validnum() == b.validnum() and a.size() == b.size()
    assert sort_rows(a.flatten()).tobytes() == sort_rows(b.flatten()).tobytes()
    sa, sb = a.stats(), b.stats()
    da, db = a.dir_stats(), b.dir_stats()
    if sa["rebuilds"] == sb["rebuilds"] and da["relists"] == db["relists"]:
        assert {k: sa[k] for k in ("main_leaves", "levels", "rebuilds")} == {k: sb[k] for k in ("main_leaves", "levels", "rebuilds")}
        assert {k: da[k] for k in ("cells", "capacity", "relists")} == {k: db[k] for k in ("cells", "capacity", "relists")}
    pa, ea, ca = a.Nearest_Search(queries, 5)
    pb, eb, cb = b.Nearest_Search(queries, 5)
    assert ea.tobytes() == eb.tobytes() and ca.tobytes() == cb.tobytes()


@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
def test_equals_host_form(problems, name, extr):
    pr = problems(name)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr))
              for t in (th, td))
    xh, Ph, _ = fh.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    out3 = fh.map_incremental(0.5, True)
    x, P = dev(pr.x_prior), dev(pr.P_prior)
    st = fd.update_device(dev(pr.scan), x, P, pr.R)
    out4 = fd.map_incremental_device(0.5, True)
    o = host(out4)
    assert tuple(int(v) for v in o[:3]) == out3 and o[3] in (FL_OK, 1), o
    assert host(st)[0] == 0 and host(x).tobytes() == xh.tobytes() and host(P).tobytes() == Ph.tobytes()
    td.maintain()
    q = world_points(pr, pr.scan)
    same_map(th, td, q)
    # the next scan on both: state, Nearest_Points and point_selected_surf
    scan2 = pr.scan[::-1].copy()
    xh2, Ph2, _ = fh.update_iterated_dyn_share_modified(scan2, xh, Ph, pr.R)
    xd2, Pd2, _ = fd.update_iterated_dyn_share_modified(scan2, host(x), host(P), pr.R)
    assert xd2.tobytes() == xh2.tobytes() and Pd2.tobytes() == Ph2.tobytes()
    n = len(scan2)
    (ph, ch), (pd, cd) = fh.nearest(n), fd.nearest(n)
    assert pd.tobytes() == ph.tobytes() and cd.tobytes() == ch.tobytes()
    assert fd.selected(n).tobytes() == fh.selected(n).tobytes()


PARITY_N_MAX = 300


def parity_batches(pr):
    """(n, batch of PARITY_N_MAX rows): *n_device of 0, 1, n_max, above n_max (clamped) and in between."""
    q = world_points(pr, pr.scan)
    rng = np.random.default_rng(5)
    out = []
    for n in (0, 1, PARITY_N_MAX, PARITY_N_MAX + 40, 77):
        batch = q[rng.permutation(len(q))[:PARITY_N_MAX]].copy()
        batch[:, :3] += rng.normal(0, 0.05, (PARITY_N_MAX, 3)).astype(np.float32)
        out.append((n, batch))
    return out


@pytest.mark.parametrize("downsample_on", [True, False])
def test_add_points_async_matches_reference(problems, downsample_on):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    r = RefTree(f"add_points_async_{int(downsample_on)}", pr.map_pts)
    n_max = PARITY_N_MAX
    for step, (n, batch) in enumerate(parity_batches(pr)):
        st = t.add_points_async(dev(batch), dev(np.array([n], np.int32)), n_max, downsample_on)
        s = host(st)
        assert s[0] in (FL_OK, 1), (step, s)
        assert s[1] == r.add(batch[:min(n, n_max)], downsample_on), step
        t.maintain()
        assert t.validnum() == r.validnum(), step
    assert rows_digest(t.flatten()) == r.flatten_digest()


def stream_scans(pr, n_scans, n_pts=800):
    return [synth.make_scan(pr.scene, n_pts, synth.true_state(pr.cfg.lidar, step), seed=100 + step) for step in range(n_scans)]


@pytest.mark.parametrize("maintain", [False, True])
def test_stream_of_scans(problems, maintain):
    """20 scans as test_gpu_stream.py's loop (the window moves at scan 2): the device forms, with the host reading nothing until
    the end (or only the status, calling fl_map_maintain when it is due), track the host-form loop."""
    pr = problems("small")
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=2000, max_iter=3) for t in (th, td))
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd = dev(xh), dev(Ph)
    statuses = []
    for step, scan in enumerate(stream_scans(pr, 20)):
        if step == 2:
            box = np.array([[-1000, -1000, -1000, -60.0, 1000, 1000]], dtype=np.float32)
            assert th.Delete_Point_Boxes(box) == td.Delete_Point_Boxes(box)
        Ph = Ph + np.eye(23) * 1e-4
        Pd += torch.eye(23, dtype=torch.float64, device="cuda") * 1e-4
        xh, Ph, _ = fh.update_iterated_dyn_share_modified(scan, xh, Ph, pr.R)
        fh.map_incremental(0.5, True)
        fd.update_device(dev(scan), xd, Pd, pr.R)
        out4 = fd.map_incremental_device(0.5, True)
        statuses.append(out4)
        if maintain and int(host(out4)[3]) == 1:
            td.maintain()
    st = np.stack([host(s) for s in statuses])
    assert (st[:, 3] != FL_ERR_CAPACITY).all(), st
    assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes()
    td.maintain()
    same_map(th, td, world_points(pr, pr.scan))


def test_graph_of_update_and_map_incremental(problems):
    """update_device + map_incremental_device captured once, replayed over 12 scans of one size copied into the captured scan
    buffer: state and map equal the host-form loop's; a host-form validnum between two replays is right and keeps the graph."""
    pr = problems("small")
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=2000, max_iter=3) for t in (th, td))
    scans = stream_scans(pr, 13)
    n = min(len(s) for s in scans)
    scans = [s[:n].copy() for s in scans]
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd, sd = dev(xh), dev(Ph), dev(scans[0])
    out4 = torch.zeros(4, dtype=torch.int32, device="cuda")
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                      # warm-up (scan 0) outside capture, on both
        fd.update_device(sd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)
    torch.cuda.current_stream().wait_stream(side)
    xh, Ph, _ = fh.update_iterated_dyn_share_modified(scans[0], xh, Ph, pr.R)
    fh.map_incremental(0.5, True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fd.update_device(sd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)
    for step, scan in enumerate(scans[1:], 1):
        sd.copy_(dev(scan))
        g.replay()
        xh, Ph, _ = fh.update_iterated_dyn_share_modified(scan, xh, Ph, pr.R)
        o3 = fh.map_incremental(0.5, True)
        o = host(out4)
        assert tuple(int(v) for v in o[:3]) == o3 and o[3] in (FL_OK, 1), (step, o)
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), step
        assert td.validnum() == th.validnum(), step        # host-form read between replays: settles, layout unchanged
    same_map(th, td, world_points(pr, pr.scan))


def test_refusal_leaves_the_map_unchanged(problems):
    """A fine cell directory and fresh points every replay exhaust the headroom; the refusing replay changes nothing, maintain
    reports a layout change and a recaptured graph runs again.  A capturing call the host's bound refuses captures nothing."""
    rng = np.random.default_rng(3)
    pts = np.zeros((2000, 4), np.float32)
    pts[:, :3] = rng.uniform(-50, 50, (2000, 3))
    t = api.KdTree(0, 0.5, cell_size=0.05); t.Build(pts)
    t.maintain()                                       # reports the Build's layout; from here on it reports only later changes
    n_max = 256
    buf = dev(np.zeros((n_max, 4), np.float32))
    nd = dev(np.array([n_max], np.int32))
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    q = dev(pts[:64])

    def capture():
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            t.add_points_async(buf, nd, n_max, False, status)
        return g

    def fresh():
        b = np.zeros((n_max, 4), np.float32)
        b[:, :3] = rng.uniform(-50, 50, (n_max, 3))
        buf.copy_(dev(b))

    fresh(); t.add_points_async(buf, nd, n_max, False, status)                               # outside capture: scratch, bound
    s0 = int(host(status)[0])
    assert s0 in (FL_OK, 1)
    assert t.maintain() == (s0 == 1)                   # nothing moves unless maintenance was due
    g = capture()
    refused = None
    for rep in range(300):
        before = (t.validnum(), t.size(), sort_rows(t.flatten()).tobytes(), [host(a).tobytes() for a in t.nearest_search_device(q, 5)])
        fresh()
        g.replay()
        s = host(status)
        if s[0] == FL_ERR_CAPACITY:
            refused = rep
            assert s[1] == 0
            after = (t.validnum(), t.size(), sort_rows(t.flatten()).tobytes(), [host(a).tobytes() for a in t.nearest_search_device(q, 5)])
            assert after == before
            break
        assert s[0] in (FL_OK, 1), (rep, s)
    assert refused is not None, "the headroom was never exhausted"
    assert t.maintain()
    g = capture()
    fresh()
    g.replay()
    assert host(status)[0] in (FL_OK, 1)
    # a capturing call whose host bound cannot fit: FL_ERR_CAPACITY at once
    L = api.load()
    big = 1 << 26
    torch.cuda.synchronize()
    v0 = t.validnum()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g2 = torch.cuda.CUDAGraph()
        g2.capture_begin()
        rc = L.fl_map_add_points_async(t.h, buf.data_ptr(), nd.data_ptr(), big, 0, status.data_ptr(), s.cuda_stream)
        g2.capture_end()
    assert rc == FL_ERR_CAPACITY
    assert t.validnum() == v0


def test_ordering_against_streams(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    q = world_points(pr, pr.scan)[:256]
    q[:, :3] += 0.37                                   # off the map points: the inserted copies become the nearest
    want_before = t.Nearest_Search_K(q, 5)
    pts = dev(q)
    nd = dev(np.array([len(q)], np.int32))
    torch.cuda.synchronize()
    # an insert behind a sleep on the caller's stream: a host-form knn and a device query on another stream see it
    main = torch.cuda.Stream()
    with torch.cuda.stream(main):
        torch.cuda._sleep(200_000_000)
        p2 = pts * 1.0
        t.add_points_async(p2, nd, len(q), False)
    _, d2, cnt = t.Nearest_Search(q, 5)
    assert (d2[:, 0] == 0).all()
    other = torch.cuda.Stream()
    with torch.cuda.stream(other):
        _, dd, _ = t.nearest_search_device(pts, 5)
    assert (host(dd)[:, 0] == 0).all()
    # an insert issued after a device query still in flight on another stream does not overtake it
    t2 = api.KdTree(0, 0.5); t2.Build(pr.map_pts)
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(a):
        torch.cuda._sleep(200_000_000)
        qa = pts * 1.0
        res = t2.nearest_search_device(qa, 5)
    with torch.cuda.stream(b):
        t2.add_points_async(pts, nd, len(q), False)
    torch.cuda.synchronize()
    assert all(host(x).tobytes() == w.tobytes() for x, w in zip(res, want_before))
    assert t2.validnum() == t.validnum()


def test_arguments_and_scope(problems):
    pr = problems("small")
    L = api.load()
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    s = torch.cuda.current_stream().cuda_stream
    pts = dev(world_points(pr, pr.scan))
    nd = torch.full((2,), 50, dtype=torch.int32, device="cuda")
    st = torch.full((4,), -7, dtype=torch.int32, device="cuda")
    hn, hs = np.array([50], np.int32), np.zeros(4, np.int32)
    p_, n_, s_ = pts.data_ptr(), nd.data_ptr(), st.data_ptr()
    v0, flat0 = t.validnum(), sort_rows(t.flatten()).tobytes()
    refused = [
        (p_, hn.ctypes.data, 100, s_), (p_, n_, 100, hs.ctypes.data), (pr.scan.ctypes.data, n_, 100, s_),
        (None, n_, 100, s_), (p_, None, 100, s_), (p_, n_, 100, None),
        (p_ + 4, n_, 100, s_), (p_, n_ + 2, 100, s_), (p_, n_, 100, s_ + 2), (p_, n_, -1, s_),
    ]
    for i, (p, n, m, o) in enumerate(refused):
        assert L.fl_map_add_points_async(t.h, p, n, m, 1, o, s) == FL_ERR_ARG, i
    for o in (hs.ctypes.data, None, s_ + 2):
        assert L.fl_filter_map_incremental_device(f.h, 0.5, 1, o, s) == FL_ERR_ARG
    assert L.fl_filter_map_incremental_device(f.h, 0.0, 1, s_, s) == FL_ERR_ARG
    sharded = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    sharded.set_shard(0, len(pr.scan))
    assert L.fl_filter_map_incremental_device(sharded.h, 0.5, 1, s_, s) == FL_ERR_STATE
    torch.cuda.synchronize()
    assert (host(st) == -7).all()
    assert t.validnum() == v0 and sort_rows(t.flatten()).tobytes() == flat0
    with pytest.raises(ValueError):
        t.add_points_async(pts.cpu(), nd[:1], 10, True)
    with pytest.raises(TypeError):
        t.add_points_async(pts, nd[:1].long(), 10, True)
    with pytest.raises(ValueError):
        f.map_incremental_device(0.5, True, torch.zeros(3, dtype=torch.int32, device="cuda"))


def fresh_points(rng, n, half=50.0):
    p = np.zeros((n, 4), np.float32)
    p[:, :3] = rng.uniform(-half, half, (n, 3))
    return p


def test_owed_maintenance_survives_host_reads():
    """A status of 1 and a refusal are owed to fl_map_maintain even when read-only host calls (validnum, size, stats) settle
    the map in between: maintain then re-packs or grows, and the next call is accepted."""
    rng = np.random.default_rng(11)
    # maintenance due: more overflow leaves than the re-pack threshold
    t = api.KdTree(0, 0.5); t.Build(fresh_points(rng, 2000))
    t.maintain()
    n = 4096
    st = host(t.add_points_async(dev(fresh_points(rng, n)), dev(np.array([n], np.int32)), n, False))
    assert st[0] == 1, st
    rebuilds = t.stats()["rebuilds"]
    assert t.validnum() == 2000 + n and t.size() == 2000 + n
    assert t.maintain()
    assert t.stats()["rebuilds"] == rebuilds + 1
    st = host(t.add_points_async(dev(fresh_points(rng, 8)), dev(np.array([8], np.int32)), 8, False))
    assert st[0] == FL_OK, st
    # a refusal by the halo-list pool: a fine directory whose table has room to spare, fresh cells on every call
    t = api.KdTree(0, 0.5, cell_size=0.05); t.Build(fresh_points(rng, 50000))
    t.maintain()
    n = 1024
    nd = dev(np.array([n], np.int32))
    refused = False
    for _ in range(60):
        st = host(t.add_points_async(dev(fresh_points(rng, n)), nd, n, False))
        if st[0] == FL_ERR_CAPACITY:
            refused = True
            break
        assert st[0] in (FL_OK, 1), st
    assert refused, "the list pool was never exhausted"
    v, relists = t.validnum(), t.dir_stats()["relists"]
    assert t.size() >= v
    assert t.maintain()
    assert t.dir_stats()["relists"] == relists + 1
    st = host(t.add_points_async(dev(fresh_points(rng, n)), nd, n, False))
    assert st[0] in (FL_OK, 1), st
    assert t.validnum() == v + n


def test_plain_c_program_with_a_graph(problems, tmp_path):
    """tests/facade/map_incremental_device.cu: the C ABI alone (streams as void*, cudaStreamBeginCapture) -- update + map
    update captured into one graph, replayed over scans, equal to the host forms."""
    import os
    import struct
    import subprocess
    from fast_lio_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pr = problems("small")
    scans = stream_scans(pr, 8)
    nq = min(len(x) for x in scans)
    exe = tmp_path / "map_incremental_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(root, "include"),
           os.path.join(root, "tests", "facade", "map_incremental_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as fo:
        fo.write(struct.pack("4i", len(pr.map_pts), nq, len(scans), 3))
        fo.write(struct.pack("d", pr.R))
        fo.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes())
        for sc in scans:
            fo.write(np.ascontiguousarray(sc[:nq], np.float32).tobytes())
        for a in (pr.x_prior, pr.P_prior, np.broadcast_to(np.asarray(pr.limit, np.float64), (23,))):
            fo.write(np.ascontiguousarray(a, np.float64).tobytes())
    run = subprocess.run([str(exe), str(fin)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "all equal" in run.stdout, run.stdout
