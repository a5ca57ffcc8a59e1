"""Device-buffer form of the update (fl_filter_update_device, fl_filter_get_nearest_device, fl_filter_get_selected_device):
the bytes of fl_filter_update on the same inputs, stream-ordered on the caller's stream, no host synchronisation, so it can be
captured into a CUDA graph together with the map's device queries."""
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth
from semantics import sort_rows

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = -2, -4, -5


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def filters(t, pr, extr=0, n=2, max_points=None, **kw):
    return [api.Esekf(t, max_points=max_points or max(len(pr.scan), 1), max_iter=pr.cfg.max_iter, limit=pr.limit,
                      extrinsic_est_en=bool(extr), **kw) for _ in range(n)]


def host_update(f, scan, x0, P0, R):
    """fl_filter_update and its pass count."""
    x, P, _ = f.update_iterated_dyn_share_modified(scan, x0, P0, R)
    return x, P, f.download_state()[2]


def device_update(f, scan, x0, P0, R):
    x, P = dev(x0), dev(P0)
    st = f.update_device(dev(scan), x, P, R)
    return host(x), host(P), host(st)


def same_logs(a, b):
    assert len(a) == len(b)
    for la, lb in zip(a, b):
        for k in la:
            assert np.asarray(la[k]).tobytes() == np.asarray(lb[k]).tobytes(), k


def world_points(pr, scan):
    """The scan pushed through the prior pose, as (n, 4) float32 queries."""
    x = pr.x_prior
    qx, qy, qz, qw = x[3:7]
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw)],
                  [2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw)],
                  [2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)]])
    q = np.array(scan, dtype=np.float32).copy()
    q[:, :3] = (scan[:, :3].astype(np.float64) @ R.T + x[:3]).astype(np.float32)
    return q


@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
def test_equals_host_form(problems, name, extr):
    """avia_2k_50k runs the two-threads-per-point k_update<_, 2>, velodyne_30k_1m the one-thread k_update<_, 1>."""
    pr = problems(name)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    fh, fd = filters(t, pr, extr)
    n = len(pr.scan)
    xh, Ph, nh = host_update(fh, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    xd, Pd, st = device_update(fd, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert xd.tobytes() == xh.tobytes() and Pd.tobytes() == Ph.tobytes()
    assert list(st) == [0, nh] and nh >= 2
    same_logs(fd.pass_logs(), fh.pass_logs())
    (ph, ch), (pd, cd) = fh.nearest(n), fd.nearest(n)
    assert pd.tobytes() == ph.tobytes() and cd.tobytes() == ch.tobytes()
    assert fd.selected(n).tobytes() == fh.selected(n).tobytes()
    pt, ct = fd.nearest_device(n)
    assert host(pt).tobytes() == ph.tobytes() and host(ct).tobytes() == ch.tobytes()
    assert host(fd.selected_device(n)).tobytes() == fh.selected(n).tobytes()
    assert fd.download_state()[2] == nh


@pytest.mark.parametrize("case", ["0", "1", "5", "no_effective_points"])
def test_small_and_empty_scans(problems, case):
    pr = problems("tiny")
    if case == "no_effective_points":
        scan = pr.scan[:50].copy()
        scan[:, :3] += 5000.0                      # nothing within sqrt(5) m of any 5 map points
    else:
        scan = pr.scan[:int(case)].copy()
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    fh, fd = filters(t, pr, max_points=64)
    xh, Ph, nh = host_update(fh, scan, pr.x_prior, pr.P_prior, pr.R)
    xd, Pd, st = device_update(fd, scan, pr.x_prior, pr.P_prior, pr.R)
    assert xd.tobytes() == xh.tobytes() and Pd.tobytes() == Ph.tobytes()
    assert list(st) == [0, nh]
    same_logs(fd.pass_logs(), fh.pass_logs())
    if case == "no_effective_points":
        assert np.array_equal(xd, pr.x_prior)


def host_pipeline(pr, scan, x0, P0):
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f, = filters(t, pr, n=1)
    x, P, _ = host_update(f, scan, x0, P0, pr.R)
    return x, P, f.map_incremental(0.5, True), t.validnum(), sort_rows(t.flatten()), f.nearest(len(scan))


def test_busy_caller_stream(problems):
    """x, P and the scan are produced on a stream that is still busy when the call is made; the update and the host-form
    map_incremental that follows still see them."""
    pr = problems("small")
    want = host_pipeline(pr, pr.scan, pr.x_prior, pr.P_prior)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f, = filters(t, pr, n=1)
    xb, Pb, sb = dev(pr.x_prior), dev(pr.P_prior), dev(pr.scan)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)             # ~0.1 s: the call below is enqueued long before its inputs exist
        x, P, s = xb * 1.0, Pb * 1.0, sb * 1.0
        st = f.update_device(s, x, P, pr.R)
    counts = f.map_incremental(0.5, True)          # host form: waits for the update on `side`
    side.synchronize()
    assert host(x).tobytes() == want[0].tobytes() and host(P).tobytes() == want[1].tobytes() and host(st)[0] == 0
    assert counts == want[2] and t.validnum() == want[3]
    assert sort_rows(t.flatten()).tobytes() == want[4].tobytes()


def test_scan_buffer_reused_after_the_call(problems):
    pr = problems("small")
    want = host_pipeline(pr, pr.scan, pr.x_prior, pr.P_prior)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f, = filters(t, pr, n=1)
    x, P, s = dev(pr.x_prior), dev(pr.P_prior), dev(pr.scan)
    f.update_device(s, x, P, pr.R)
    s.fill_(1.0e6)                                 # overwritten, then freed: the caching allocator hands the block out again
    del s
    junk = torch.full((len(pr.scan), 4), -3.0e5, dtype=torch.float32, device="cuda")
    assert f.map_incremental(0.5, True) == want[2]
    assert t.validnum() == want[3] and sort_rows(t.flatten()).tobytes() == want[4].tobytes()
    assert host(x).tobytes() == want[0].tobytes()
    assert f.nearest(len(pr.scan))[0].tobytes() == want[5][0].tobytes()
    del junk


def test_graph_capture_and_replay(problems):
    """Update plus a k = 5 nearest search in one graph, replayed with a different prior each time.  Every replay must equal the
    host form for its prior: that fails when k_update's publication block keeps the previous replay's words (same nonce).  A
    host-form update between two replays leaves a mirrored result behind; download_state and get_pass_logs after the next
    replay must return the replay's."""
    pr = problems("avia_2k_50k")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    fh, fd = filters(t, pr)
    rng = np.random.default_rng(31)
    q = world_points(pr, pr.scan)
    qd, sd = dev(q), dev(pr.scan)
    xs, Ps = dev(pr.x_prior), dev(pr.P_prior)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                  # warm-up outside capture
        fd.update_device(sd, xs, Ps, pr.R, status)
        t.nearest_search_device(qd, 5)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fd.update_device(sd, xs, Ps, pr.R, status)
        nn = t.nearest_search_device(qd, 5)
    want_nn = t.Nearest_Search_K(q, 5)
    for rep in range(4):
        x0 = pr.x_prior.copy()
        x0[:3] += rng.normal(0, 0.05, 3)
        P0 = pr.P_prior * (1.0 + 0.25 * rep)
        xs.copy_(dev(x0)); Ps.copy_(dev(P0))
        g.replay()
        torch.cuda.synchronize()
        xh, Ph, nh = host_update(fh, pr.scan, x0, P0, pr.R)
        assert host(xs).tobytes() == xh.tobytes() and host(Ps).tobytes() == Ph.tobytes(), rep
        assert list(host(status)) == [0, nh], rep
        assert all(host(a).tobytes() == w.tobytes() for a, w in zip(nn, want_nn))
        if rep >= 2:                               # the replay after a host-form update on the same filter
            xr, Pr, nr = fd.download_state()
            assert xr.tobytes() == xh.tobytes() and Pr.tobytes() == Ph.tobytes() and nr == nh
            same_logs(fd.pass_logs(), fh.pass_logs())
        if rep == 1:
            other = pr.x_prior.copy(); other[:3] -= 0.1
            fd.update_iterated_dyn_share_modified(pr.scan, other, pr.P_prior, pr.R)


def test_stream_of_scans(problems):
    """Five scans, as test_gpu_stream.py::test_stream_of_scans: a device update then the host map_incremental each scan; state
    and map equal the all-host pipeline's bit for bit."""
    pr = problems("small")
    trees = [api.KdTree(0, 0.5) for _ in range(2)]
    for t in trees:
        t.Build(pr.map_pts)
    fh, fd = (api.Esekf(t, max_points=2000, max_iter=3) for t in trees)
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd = dev(xh), dev(Ph)
    for step in range(5):
        scan = synth.make_scan(pr.scene, 800, synth.true_state(pr.cfg.lidar, step), seed=100 + step)
        if step == 2:
            box = np.array([[-1000, -1000, -1000, -60.0, 1000, 1000]], dtype=np.float32)
            assert trees[0].Delete_Point_Boxes(box) == trees[1].Delete_Point_Boxes(box)
        Ph = Ph + np.eye(23) * 1e-4
        Pd += torch.eye(23, dtype=torch.float64, device="cuda") * 1e-4
        xh, Ph, _ = fh.update_iterated_dyn_share_modified(scan, xh, Ph, pr.R)
        st = fd.update_device(dev(scan), xd, Pd, pr.R)
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes() and host(st)[0] == 0, step
        assert fd.map_incremental(0.5, True) == fh.map_incremental(0.5, True), step
        assert trees[0].validnum() == trees[1].validnum()
    assert sort_rows(trees[0].flatten()).tobytes() == sort_rows(trees[1].flatten()).tobytes()


def test_arguments_and_scope(problems):
    pr = problems("small")
    L = api.load()
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f, = filters(t, pr, n=1, max_points=len(pr.scan))
    n = len(pr.scan)
    sd = dev(pr.scan)
    xs = torch.full((26 + 2,), -7.0, dtype=torch.float64, device="cuda")
    Ps = torch.full((23 * 23 + 2,), -7.0, dtype=torch.float64, device="cuda")
    ss = torch.full((4,), -7, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    xh, Ph, sh = np.zeros(26), np.zeros((23, 23)), np.zeros(2, np.int32)

    def call(ff, body, nq, x, P, st):
        return L.fl_filter_update_device(ff.h, body, nq, x, P, pr.R, st, s)

    x_, P_, s_ = xs.data_ptr(), Ps.data_ptr(), ss.data_ptr()
    refused = [
        (f, pr.scan.ctypes.data, n, x_, P_, s_, FL_ERR_ARG),          # host scan
        (f, sd.data_ptr(), n, xh.ctypes.data, P_, s_, FL_ERR_ARG),    # host x
        (f, sd.data_ptr(), n, x_, Ph.ctypes.data, s_, FL_ERR_ARG),    # host P
        (f, sd.data_ptr(), n, x_, P_, sh.ctypes.data, FL_ERR_ARG),    # host status
        (f, None, n, x_, P_, s_, FL_ERR_ARG),
        (f, sd.data_ptr(), n, None, P_, s_, FL_ERR_ARG),
        (f, sd.data_ptr(), n, x_, None, s_, FL_ERR_ARG),
        (f, sd.data_ptr(), n, x_, P_, None, FL_ERR_ARG),
        (f, sd.data_ptr(), -1, x_, P_, s_, FL_ERR_ARG),
        (f, sd.data_ptr() + 4, n - 1, x_, P_, s_, FL_ERR_ARG),        # misaligned scan
        (f, sd.data_ptr(), n, x_ + 4, P_, s_, FL_ERR_ARG),            # misaligned x
        (f, sd.data_ptr(), n, x_, P_ + 4, s_, FL_ERR_ARG),            # misaligned P
        (f, sd.data_ptr(), n, x_, P_, s_ + 2, FL_ERR_ARG),            # misaligned status
    ]
    big = torch.zeros((n * 2 + 4096, 4), dtype=torch.float32, device="cuda")
    refused.append((f, big.data_ptr(), len(big), x_, P_, s_, FL_ERR_CAPACITY))
    sharded, = filters(t, pr, n=1); sharded.set_shard(0, n)
    solver0, = filters(t, pr, n=1, solver=0)
    split, = filters(t, pr, n=1, fused=0)
    for ff in (sharded, solver0, split):
        refused.append((ff, sd.data_ptr(), n, x_, P_, s_, FL_ERR_STATE))
    for i, (ff, body, nq, x, P, st, rc) in enumerate(refused):
        assert call(ff, body, nq, x, P, st) == rc, i
    torch.cuda.synchronize()
    assert (host(xs) == -7.0).all() and (host(Ps) == -7.0).all() and (host(ss) == -7).all()
    # the getters
    out = torch.zeros((n, 5, 4), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    assert L.fl_filter_get_nearest_device(f.h, out.data_ptr(), cnt.data_ptr(), n, s) == FL_ERR_ARG      # no scan bound yet
    assert call(f, sd.data_ptr(), n, x_, P_, s_) == 0
    assert L.fl_filter_get_nearest_device(f.h, out.data_ptr(), cnt.data_ptr(), n + 1, s) == FL_ERR_ARG
    assert L.fl_filter_get_nearest_device(f.h, out.data_ptr() + 4, cnt.data_ptr(), n, s) == FL_ERR_ARG
    assert L.fl_filter_get_selected_device(f.h, sh.ctypes.data, 2, s) == FL_ERR_ARG
    assert L.fl_filter_get_nearest_device(sharded.h, out.data_ptr(), cnt.data_ptr(), 0, s) == FL_ERR_STATE
    # the binding's checks
    xg, Pg = dev(pr.x_prior), dev(pr.P_prior)
    with pytest.raises(ValueError):
        f.update_device(torch.from_numpy(pr.scan), xg, Pg)                  # a CPU tensor
    with pytest.raises(TypeError):
        f.update_device(sd, xg.float(), Pg)
    with pytest.raises(ValueError):
        f.update_device(sd, xg[:25], Pg)
    with pytest.raises(ValueError):
        f.update_device(sd, xg, Pg.t())                                     # not contiguous
    with pytest.raises(ValueError):
        f.update_device(sd[:, :3].contiguous(), xg, Pg)
    if torch.cuda.device_count() < 2:
        pytest.skip("the wrong-device case needs a second GPU")
    other = dev(pr.x_prior).to("cuda:1")
    assert call(f, sd.data_ptr(), n, other.data_ptr(), P_, s_) == FL_ERR_ARG
    with pytest.raises(ValueError):
        f.update_device(sd, other, Pg)


def test_plain_c_program_on_its_own_stream(problems, tmp_path):
    pr = problems("small")
    exe = tmp_path / "filter_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "facade", "filter_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as fo:
        fo.write(struct.pack("3i", len(pr.map_pts), len(pr.scan), pr.cfg.max_iter))
        fo.write(struct.pack("d", pr.R))
        for a in (pr.map_pts, pr.scan):
            fo.write(np.ascontiguousarray(a, np.float32).tobytes())
        for a in (pr.x_prior, pr.P_prior, np.broadcast_to(np.asarray(pr.limit, np.float64), (23,))):
            fo.write(np.ascontiguousarray(a, np.float64).tobytes())
    run = subprocess.run([str(exe), str(fin)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "all equal" in run.stdout, run.stdout
