"""Device forms of the scan front end and of the update on it (fl_scan_upload_device, fl_scan_undistort_device,
fl_scan_voxel_downsample_device, fl_filter_update_scan_device): byte for byte the host forms at the device count, on the
caller's stream, and one CUDA graph for a stream of scans of different sizes."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth
from semantics import sort_rows

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = 0, -2, -4, -5


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def tree(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return t


@pytest.fixture(scope="module")
def raw(problems):
    pr = problems("small")
    return synth.make_raw_scan(pr.scene, 20_000, pr.x_true, seed=31)


def padded(a, rows, fill=np.nan):
    """a with rows appended up to `rows`, filled with NaN garbage (the device forms must not read them)."""
    out = np.full((rows,) + a.shape[1:], fill, dtype=a.dtype)
    out[:len(a)] = a
    return out


def host_chain(tree, xyzi, t, poses, x_end, leaf):
    s = api.Scan(tree)
    s.upload(xyzi, t)
    s.undistort(poses, x_end)
    deskewed = s.download(0)
    n = s.voxel_downsample(leaf)
    return s, deskewed, n, s.download(1)


def device_chain(tree, xyzi, t, poses, x_end, leaf, n_max, n_pose_max):
    s = api.Scan(tree)
    s.reserve(n_max, n_pose_max)
    s.upload_device(dev(padded(xyzi, n_max)), dev(padded(t, n_max)), dev(np.array([len(xyzi)], np.int32)), n_max)
    s.undistort_device(dev(padded(poses, n_pose_max)), dev(np.array([len(poses)], np.int32)), dev(x_end))
    n_out = s.voxel_downsample_device(leaf)
    return s, int(host(n_out)[0])


CASES = [  # (leaf, count, n_max): leaf 1e-4 over a scene tens of metres wide overflows the grid -- PCL's passthrough exit
    (0.5, 20_000, 20_000), (0.5, 12_345, 20_000), (0.25, 20_000, 24_000), (0.25, 777, 20_000),
    (1e-4, 5_000, 8_000), (0.5, 0, 1_000), (0.5, 1, 1_000), (0.25, 0, 0),
]


@pytest.mark.parametrize("leaf, n, n_max", CASES)
def test_stages_equal_host_forms(tree, raw, leaf, n, n_max):
    """The de-skewed cloud (and its order) and the down-sampled cloud and count, read through the host forms (which take the
    device forms' cloud over) and as n_out."""
    xyzi, t = raw.xyzi[:n], raw.offset_ms[:n]
    _, want_deskew, want_n, want_down = host_chain(tree, xyzi, t, raw.imu_pose, raw.x_end, leaf)
    s, n_out = device_chain(tree, xyzi, t, raw.imu_pose, raw.x_end, leaf, n_max, len(raw.imu_pose) + 7)
    assert n_out == want_n
    assert s.download(1).tobytes() == want_down.tobytes()
    assert s.download(0).tobytes() == want_deskew.tobytes()
    assert s.voxel_downsample(leaf) == want_n                    # a host form after the device forms continues from their cloud
    assert s.download(1).tobytes() == want_down.tobytes()


def test_undistort_quirks_and_few_poses(tree, raw):
    """The inputs of test_undistort_quirks_match_oracle (negative IMU offsets, no point at offset 0), NaN and tied times, and
    fewer than two poses (only the sort)."""
    poses = np.vstack([raw.imu_pose[:1], raw.imu_pose[:1], raw.imu_pose[1:]])
    poses[1, 0] = -0.004
    t = raw.offset_ms.copy()
    t[np.argmin(t)] = 7.0
    t[::97] = np.nan
    t[1::89] = t[5]
    t[2::101] = -0.0
    t[3::103] = np.inf
    for ps in (poses, raw.imu_pose[:1], raw.imu_pose[:0]):
        _, want, want_n, want_down = host_chain(tree, raw.xyzi, t, ps, raw.x_end, 0.5)
        s, n_out = device_chain(tree, raw.xyzi, t, ps, raw.x_end, 0.5, len(t) + 100, len(poses))
        assert s.download(0).tobytes() == want.tobytes()
        assert n_out == want_n and s.download(1).tobytes() == want_down.tobytes()


def same_map(a, b, queries):
    assert a.validnum() == b.validnum() and a.size() == b.size()
    assert sort_rows(a.flatten()).tobytes() == sort_rows(b.flatten()).tobytes()
    pa, ea, ca = a.Nearest_Search(queries, 5)
    pb, eb, cb = b.Nearest_Search(queries, 5)
    assert ea.tobytes() == eb.tobytes() and ca.tobytes() == cb.tobytes()


def twins(pr):
    trees = [api.KdTree(0, 0.5) for _ in range(2)]
    for t in trees:
        t.Build(pr.map_pts)
    return trees


# (extrinsic_est_en, raw points, n_max, leaf).  40k rows take one thread per point (k_update's pair form needs the tiles to fit
# the 512-thread grid) while the ~10k down-sampled points take two; 150k raw points at 5 cm leave more tiles than co-resident
# worker blocks.
UPDATE_CASES = [(0, 8_000, 8_000, 0.5), (1, 8_000, 12_000, 0.5), (0, 20_000, 40_000, 0.25), (1, 20_000, 40_000, 0.25),
                (0, 150_000, 160_000, 0.05), (1, 150_000, 150_000, 0.05)]


@pytest.mark.parametrize("extr, n_raw, n_max, leaf", UPDATE_CASES)
def test_update_equals_host_form(problems, extr, n_raw, n_max, leaf):
    """x, P, Nearest_Points, selected, the pass logs, map_incremental's out4 and the map after fl_map_maintain; the host forms
    after the device forms read the device count."""
    pr = problems("small")
    rs = synth.make_raw_scan(pr.scene, n_raw, pr.x_true, seed=41 + n_raw)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr)) for t in (th, td))
    sh, _, n, _ = host_chain(th, rs.xyzi, rs.offset_ms, rs.imu_pose, rs.x_end, leaf)
    xh, Ph, _ = sh.update(fh, pr.x_prior, pr.P_prior, pr.R)
    sd, n_out = device_chain(td, rs.xyzi, rs.offset_ms, rs.imu_pose, rs.x_end, leaf, n_max, len(rs.imu_pose))
    assert n_out == n
    x, P = dev(pr.x_prior), dev(pr.P_prior)
    st = sd.update_device(fd, x, P, pr.R)
    assert host(st)[0] == FL_OK
    assert host(x).tobytes() == xh.tobytes() and host(P).tobytes() == Ph.tobytes()
    (ph, ch), (pd, cd) = fh.nearest(n), fd.nearest(n)
    assert pd.tobytes() == ph.tobytes() and cd.tobytes() == ch.tobytes()
    assert fd.selected(n).tobytes() == fh.selected(n).tobytes()
    with pytest.raises(api.FastLioError):
        fd.nearest(n + 1)                                         # the count read back bounds the host forms, not n_max
    lh, ld = fh.pass_logs(), fd.pass_logs()
    assert len(lh) == len(ld) and all(a["HtH"].tobytes() == b["HtH"].tobytes() and a["x_after"].tobytes() == b["x_after"].tobytes()
                                      for a, b in zip(lh, ld))
    out3 = fh.map_incremental(0.5, True)
    o = host(fd.map_incremental_device(0.5, True))
    assert tuple(int(v) for v in o[:3]) == out3 and o[3] in (FL_OK, 1), o
    td.maintain()
    q = rs.xyzi[::7].copy()
    same_map(th, td, q)


def test_host_form_map_incremental_after_device_update(problems):
    pr = problems("small")
    rs = synth.make_raw_scan(pr.scene, 6_000, pr.x_true, seed=7)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=9_000, max_iter=3) for t in (th, td))
    sh, _, n, _ = host_chain(th, rs.xyzi, rs.offset_ms, rs.imu_pose, rs.x_end, 0.5)
    sh.update(fh, pr.x_prior, pr.P_prior, pr.R)
    sd, _ = device_chain(td, rs.xyzi, rs.offset_ms, rs.imu_pose, rs.x_end, 0.5, 9_000, len(rs.imu_pose))
    sd.update_device(fd, dev(pr.x_prior), dev(pr.P_prior), pr.R)
    assert fd.map_incremental(0.5, True) == fh.map_incremental(0.5, True)
    same_map(th, td, rs.xyzi[::5].copy())


def stream_of_raw_scans(pr, n_scans, n_max):
    rng = np.random.default_rng(11)
    out = []
    for step in range(n_scans):
        n = int(rng.integers(n_max // 3, n_max + 1))
        hz = float(rng.choice([100.0, 200.0, 250.0, 400.0]))
        out.append(synth.make_raw_scan(pr.scene, n, synth.true_state(pr.cfg.lidar, step), seed=200 + step, imu_hz=hz))
    return out


def test_one_graph_for_a_stream_of_scans(problems):
    """upload -> undistort -> down-sample -> update -> map_incremental captured with n_max (again only after a maintenance that
    moved the map), replayed over 24 raw scans of different sizes and IMU pose counts: x, P and out4 equal the host-form chain's after every scan, the maps after maintenance."""
    pr = problems("small")
    n_max, leaf = 9_000, 0.5
    scans = stream_of_raw_scans(pr, 24, n_max)
    n_pose_max = max(len(r.imu_pose) for r in scans)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=n_max, max_iter=3) for t in (th, td))
    sh, sd = api.Scan(th), api.Scan(td)
    sd.reserve(n_max, n_pose_max)
    xyzi = torch.zeros((n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros(n_max, dtype=torch.float32, device="cuda")
    n_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    poses = torch.zeros((n_pose_max, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    xend = torch.zeros(26, dtype=torch.float64, device="cuda")
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd = dev(xh), dev(Ph)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    out4 = torch.zeros(4, dtype=torch.int32, device="cuda")

    def fill(r):
        xyzi[:len(r.xyzi)] = dev(r.xyzi); tms[:len(r.xyzi)] = dev(r.offset_ms); n_d.fill_(len(r.xyzi))
        poses[:len(r.imu_pose)] = dev(r.imu_pose); np_d.fill_(len(r.imu_pose)); xend.copy_(dev(r.x_end))

    def chain():
        sd.upload_device(xyzi, tms, n_d, n_max)
        sd.undistort_device(poses, np_d, xend)
        sd.voxel_downsample_device(leaf)
        sd.update_device(fd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)

    side = torch.cuda.Stream()
    g, replayed = None, []                                   # the raw sizes each captured graph was replayed for
    for step, r in enumerate(scans):
        sh.upload(r.xyzi, r.offset_ms); sh.undistort(r.imu_pose, r.x_end); sh.voxel_downsample(leaf)
        xh, Ph, _ = sh.update(fh, xh, Ph, pr.R)
        o3 = fh.map_incremental(0.5, True)
        fill(r)
        torch.cuda.synchronize()
        if step == 0:                                        # outside capture once: the map's scratch for n_max
            with torch.cuda.stream(side):
                chain()
            torch.cuda.synchronize()
        else:
            if g is None:
                td.maintain()                                # settles the host's bound of the map's headroom
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):                    # capturing runs nothing
                    chain()
                replayed.append(set())
            g.replay()
            replayed[-1].add(len(r.xyzi))
        o = host(out4)
        assert host(status)[0] == FL_OK, step
        assert tuple(int(v) for v in o[:3]) == o3 and o[3] in (FL_OK, 1), (step, o)
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), step
        if o[3] == 1 and td.maintain():                      # maintenance moved the map: capture again
            g = None
    assert max(len(sizes) for sizes in replayed) >= 2        # one graph served scans of different sizes
    td.maintain()
    same_map(th, td, scans[-1].xyzi[::5].copy())
    # host forms after the replays see the last replay's scan
    assert sd.download(1).tobytes() == sh.download(1).tobytes()


def test_refusals_enqueue_nothing(problems, tree, raw):
    pr = problems("small")
    L = api.load()
    s = api.Scan(tree)
    s.reserve(1_000, 10)
    xyzi, t = dev(raw.xyzi[:1_000]), dev(raw.offset_ms[:1_000])
    n = dev(np.array([1_000], np.int32))
    stream = tree._stream()
    # above the reserve
    assert L.fl_scan_upload_device(s.h, xyzi.data_ptr(), t.data_ptr(), n.data_ptr(), 1_001, stream) == FL_ERR_CAPACITY
    # no device-form upload yet
    assert L.fl_scan_voxel_downsample_device(s.h, 0.5, None, stream) == FL_ERR_STATE
    # a host pointer, a misaligned one
    h_n = np.array([5], np.int32)
    assert L.fl_scan_upload_device(s.h, xyzi.data_ptr(), t.data_ptr(), h_n.ctypes.data, 1_000, stream) == FL_ERR_ARG
    assert L.fl_scan_upload_device(s.h, xyzi.data_ptr() + 4, t.data_ptr(), n.data_ptr(), 1_000, stream) == FL_ERR_ARG
    s.upload_device(xyzi, t, n, 1_000)
    poses = dev(raw.imu_pose[:11])
    assert L.fl_scan_undistort_device(s.h, poses.data_ptr(), n.data_ptr(), 11, dev(raw.x_end).data_ptr(), stream) == FL_ERR_CAPACITY
    f = api.Esekf(tree, max_points=2_000)
    x, P = dev(pr.x_prior), dev(pr.P_prior)
    status = dev(np.array([77, 77], np.int32))
    # no device-form down-sample since the upload
    assert L.fl_filter_update_scan_device(f.h, s.h, x.data_ptr(), P.data_ptr(), 0.001, status.data_ptr(), stream) == FL_ERR_STATE
    out = dev(np.array([-9], np.int32))
    s.voxel_downsample_device(0.5, out)
    # a scan from another map
    other = api.KdTree(0, 0.5); other.Build(pr.map_pts)
    fo = api.Esekf(other, max_points=2_000)
    assert L.fl_filter_update_scan_device(fo.h, s.h, x.data_ptr(), P.data_ptr(), 0.001, status.data_ptr(), stream) == FL_ERR_ARG
    # a filter below the scan's n_max, a sharded filter
    small = api.Esekf(tree, max_points=500)
    assert L.fl_filter_update_scan_device(small.h, s.h, x.data_ptr(), P.data_ptr(), 0.001, status.data_ptr(), stream) == FL_ERR_CAPACITY
    sharded = api.Esekf(tree, max_points=2_000)
    sharded.set_shard(0, 10)
    assert L.fl_filter_update_scan_device(sharded.h, s.h, x.data_ptr(), P.data_ptr(), 0.001, status.data_ptr(), stream) == FL_ERR_STATE
    assert host(status).tolist() == [77, 77]
    assert host(x).tobytes() == pr.x_prior.tobytes()
    # and the scan still works
    st = s.update_device(f, x, P, 0.001)
    assert host(st)[0] == FL_OK


def test_ordering_against_a_busy_caller_stream(tree, raw):
    """The inputs are written on the caller's stream behind a long kernel; the device forms read them after it."""
    n = 5_000
    _, want_deskew, want_n, want_down = host_chain(tree, raw.xyzi[:n], raw.offset_ms[:n], raw.imu_pose, raw.x_end, 0.5)
    s = api.Scan(tree)
    s.reserve(n, len(raw.imu_pose))
    xyzi = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    t = torch.zeros(n, dtype=torch.float32, device="cuda")
    src_x, src_t = dev(raw.xyzi[:n]), dev(raw.offset_ms[:n])
    poses, xe = dev(raw.imu_pose), dev(raw.x_end)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        xyzi.copy_(src_x); t.copy_(src_t)
        s.upload_device(xyzi, t)
        s.undistort_device(poses, None, xe)
        out = s.voxel_downsample_device(0.5)
    torch.cuda.synchronize()
    assert int(host(out)[0]) == want_n
    assert s.download(0).tobytes() == want_deskew.tobytes() and s.download(1).tobytes() == want_down.tobytes()


def test_plain_c_program_with_one_graph(problems, tmp_path):
    """tests/facade/frontend_device.cu: the C ABI alone captures the whole chain once and replays it over raw scans of
    different sizes, equal to the host forms."""
    pr = problems("small")
    n_max, leaf = 6_000, 0.5
    scans = stream_of_raw_scans(pr, 8, n_max)
    n_pose_max = max(len(r.imu_pose) for r in scans)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as fo:
        fo.write(struct.pack("5i", len(pr.map_pts), len(scans), n_max, n_pose_max, 3))
        fo.write(struct.pack("d", pr.R)); fo.write(struct.pack("f", leaf))
        fo.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes())
        fo.write(pr.x_prior.astype(np.float64).tobytes()); fo.write(pr.P_prior.astype(np.float64).tobytes())
        for r in scans:
            fo.write(struct.pack("2i", len(r.xyzi), len(r.imu_pose)))
            fo.write(r.xyzi.tobytes()); fo.write(r.offset_ms.tobytes())
            fo.write(r.imu_pose.astype(np.float64).tobytes()); fo.write(r.x_end.astype(np.float64).tobytes())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "frontend_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(root, "include"),
           os.path.join(root, "tests", "facade", "frontend_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    res = subprocess.run([str(exe), str(inp)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "all equal" in res.stdout, res.stdout + res.stderr


def test_host_reads_between_device_stages(problems, tree, raw):
    """Every device-form stage makes its result the scan's current one: host-form reads between the stages, a second
    down-sample at another leaf and a host-form update all see the host-form chain's clouds."""
    pr = problems("small")
    n = 9_000
    xyzi, t = raw.xyzi[:n], raw.offset_ms[:n]
    sh, want_deskew, want_n, want_down = host_chain(tree, xyzi, t, raw.imu_pose, raw.x_end, 0.5)
    s = api.Scan(tree)
    s.reserve(n + 50, len(raw.imu_pose))
    s.upload_device(dev(padded(xyzi, n + 50)), dev(padded(t, n + 50)), dev(np.array([n], np.int32)), n + 50)
    assert s.download(0).tobytes() == xyzi.tobytes()                       # as uploaded
    s.undistort_device(dev(raw.imu_pose), None, dev(raw.x_end))
    assert s.download(0).tobytes() == want_deskew.tobytes()
    assert len(s.download(1)) == 0
    out = s.voxel_downsample_device(0.5)
    assert int(host(out)[0]) == want_n and s.download(1).tobytes() == want_down.tobytes()
    f1, f2 = (api.Esekf(tree, max_points=n + 50) for _ in range(2))
    xh, Ph, _ = sh.update(f1, pr.x_prior, pr.P_prior, pr.R)
    xs, Ps, _ = s.update(f2, pr.x_prior, pr.P_prior, pr.R)                # the host form binds the device forms' cloud
    assert xs.tobytes() == xh.tobytes() and Ps.tobytes() == Ph.tobytes()
    want_n2 = sh.voxel_downsample(0.25)
    out = s.voxel_downsample_device(0.25)                                   # again, at another leaf
    assert int(host(out)[0]) == want_n2 and s.download(1).tobytes() == sh.download(1).tobytes()
    s.undistort_device(dev(raw.imu_pose), None, dev(raw.x_end))             # the device forms de-skew their upload again
    assert s.download(0).tobytes() == want_deskew.tobytes()


def test_host_stage_after_device_upload_needs_a_new_upload(tree, raw):
    """A host-form undistort or down-sample replaces the device forms' cloud: their later stages and the update refuse."""
    L = api.load()
    for host_stage in ("undistort", "voxel"):
        s = api.Scan(tree)
        s.reserve(2_000, len(raw.imu_pose))
        s.upload_device(dev(raw.xyzi[:2_000]), dev(raw.offset_ms[:2_000]))
        s.voxel_downsample_device(0.5)
        if host_stage == "undistort":
            s.undistort(raw.imu_pose, raw.x_end)
        else:
            s.voxel_downsample(0.5)
        stream = tree._stream()
        assert L.fl_scan_voxel_downsample_device(s.h, 0.5, None, stream) == FL_ERR_STATE
        f = api.Esekf(tree, max_points=2_000)
        x, P = dev(np.zeros(26)), dev(np.eye(23))
        status = dev(np.zeros(2, np.int32))
        assert L.fl_filter_update_scan_device(f.h, s.h, x.data_ptr(), P.data_ptr(), 0.001, status.data_ptr(), stream) == FL_ERR_STATE
        n_pose = dev(np.array([len(raw.imu_pose)], np.int32))
        assert L.fl_scan_undistort_device(s.h, dev(raw.imu_pose).data_ptr(), n_pose.data_ptr(), len(raw.imu_pose),
                                          dev(raw.x_end).data_ptr(), stream) == FL_ERR_STATE


def test_filter_host_forms_follow_a_replay_after_a_host_update(problems):
    """A graph of the chain is captured; a host-form update on the same filter binds another scan; then the graph replays. The
    filter's host forms (get_nearest, get_selected, pass logs) answer for the replayed scan and its device count."""
    pr = problems("small")
    n_max, leaf = 7_000, 0.5
    scans = stream_of_raw_scans(pr, 3, n_max)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=n_max, max_iter=3) for t in (th, td))
    sh, sd = api.Scan(th), api.Scan(td)
    sd.reserve(n_max, max(len(r.imu_pose) for r in scans))
    n_pose_max = max(len(r.imu_pose) for r in scans)
    xyzi = torch.zeros((n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros(n_max, dtype=torch.float32, device="cuda")
    n_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    poses = torch.zeros((n_pose_max, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    xend = torch.zeros(26, dtype=torch.float64, device="cuda")
    xd, Pd = dev(pr.x_prior), dev(pr.P_prior)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    out4 = torch.zeros(4, dtype=torch.int32, device="cuda")

    def fill(r):
        xyzi[:len(r.xyzi)] = dev(r.xyzi); tms[:len(r.xyzi)] = dev(r.offset_ms); n_d.fill_(len(r.xyzi))
        poses[:len(r.imu_pose)] = dev(r.imu_pose); np_d.fill_(len(r.imu_pose)); xend.copy_(dev(r.x_end))
        torch.cuda.synchronize()

    def chain():
        sd.upload_device(xyzi, tms, n_d, n_max)
        sd.undistort_device(poses, np_d, xend)
        sd.voxel_downsample_device(leaf)
        sd.update_device(fd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)

    def host_step(r, x, P):
        sh.upload(r.xyzi, r.offset_ms); sh.undistort(r.imu_pose, r.x_end); n = sh.voxel_downsample(leaf)
        x, P, _ = sh.update(fh, x, P, pr.R)
        fh.map_incremental(0.5, True)
        return x, P, n

    xh, Ph, _ = host_step(scans[0], pr.x_prior, pr.P_prior)
    fill(scans[0])
    chain()
    torch.cuda.synchronize()
    td.maintain()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        chain()
    fd.update_iterated_dyn_share_modified(scans[1].xyzi[:500], pr.x_prior, pr.P_prior, pr.R)   # a host form binds another scan
    xh, Ph, n = host_step(scans[2], xh, Ph)
    fill(scans[2])
    assert not td.maintain()                                # the map's layout is the graph's
    g.replay()
    torch.cuda.synchronize()
    assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes()
    (ph, ch), (pd, cd) = fh.nearest(n), fd.nearest(n)
    assert pd.tobytes() == ph.tobytes() and cd.tobytes() == ch.tobytes()
    assert fd.selected(n).tobytes() == fh.selected(n).tobytes()
    with pytest.raises(api.FastLioError):
        fd.nearest(n + 1)
    lh, ld = fh.pass_logs(), fd.pass_logs()
    assert len(lh) == len(ld) and all(a["x_after"].tobytes() == b["x_after"].tobytes() for a, b in zip(lh, ld))
