"""The scan's clouds in a frame (fl_scan_frame, fl_scan_frame_device): the loops of publish_frame_world, publish_frame_body,
pcl_wait_save and the map's first Build (laserMapping.cpp:177-220, :478-549, :909-921) on the device, bit for bit a numpy FP64
restatement in the order of Eigen's _transformVector; host and device forms byte for byte; device counts, guard rows, the
append contract, refusals, stream ordering, the first scan's map, and one CUDA graph over a stream of raw scans."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth
from test_gpu_frontend_device import stream_of_raw_scans
from test_gpu_localmap_device import cross, same_map, twins

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = 0, -2, -4, -5
LIDAR, IMU, WORLD = api.FRAME_LIDAR, api.FRAME_IMU, api.FRAME_WORLD
GUARD = 77.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def qrot(q, v):
    """QuaternionBase::_transformVector of rows v (n, 3) by q = (x, y, z, w), in its order of operations."""
    qv = np.broadcast_to(q[:3], v.shape).T
    uv = cross(qv, v.T)
    uv = uv + uv
    return ((v.T + uv * q[3]) + cross(qv, uv)).T


def restated(xyzi, frame, x):
    """RGBpointBodyLidarToIMU / RGBpointBodyToWorld in FP64, rounded to float32, the intensity passed through."""
    out = np.array(xyzi, np.float32, copy=True).reshape(-1, 4)
    if frame == LIDAR:
        return out
    p_this = qrot(x[7:11], out[:, :3].astype(np.float64)) + x[11:14]
    out[:, :3] = (p_this if frame == IMU else qrot(x[3:7], p_this) + x[0:3]).astype(np.float32)
    return out


def turned_state(pr, seed):
    """A state 1 500 m from the origin, with a turned attitude and a non-identity extrinsic."""
    rng = np.random.default_rng(seed)
    x = pr.x_prior.copy()
    x[0:3] = [1500.0 * np.cos(seed), 1500.0 * np.sin(seed), 12.5]
    x[3:7] = synth.quat_mul(x[3:7], synth.quat_exp(rng.normal(0, 0.8, 3)))
    x[7:11] = synth.quat_exp(rng.normal(0, 0.3, 3))
    x[11:14] = [0.31, -0.22, 0.153]
    return x


def chains(tree, r, n_max, deskew, leaf=0.5):
    """The host-form chain on one scan handle and the device-form chain on another (over n_max rows) for the raw scan r."""
    sh, sd = api.Scan(tree), api.Scan(tree)
    sh.upload(r.xyzi, r.offset_ms)
    if deskew:
        sh.undistort(r.imu_pose, r.x_end)
    sh.voxel_downsample(leaf)
    sd.reserve(n_max, len(r.imu_pose))
    n = len(r.xyzi)
    xyzi = torch.full((n_max, 4), float("nan"), device="cuda")
    tms = torch.full((n_max,), float("nan"), device="cuda")
    xyzi[:n] = dev(r.xyzi)
    tms[:n] = dev(r.offset_ms)
    sd.upload_device(xyzi, tms, dev(np.array([n], np.int32)), n_max)
    if deskew:
        sd.undistort_device(dev(r.imu_pose), None, dev(r.x_end))
    sd.voxel_downsample_device(leaf)
    return sh, sd


@pytest.fixture(scope="module")
def small(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return pr, t


@pytest.fixture(scope="module")
def config4(problems):
    pr = problems("avia_stream_24k")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts[:1000])
    return pr, t


def check_forms(sh, sd, n_max, x, seed):
    """For every (which, frame): the host form is the restatement, the device form (appended at an offset, guard rows around)
    is the host form, FL_FRAME_LIDAR is fl_scan_download, and the host forms after the device forms read the same clouds."""
    xd = dev(x)
    for which in (0, 1):
        cloud = sh.download(which)
        n = len(cloud)
        for frame in (LIDAR, IMU, WORLD):
            want = restated(cloud, frame, x)
            got = sh.frame(which, frame, x)
            assert got.tobytes() == want.tobytes(), (which, frame)
            if frame == LIDAR:
                assert got.tobytes() == cloud.tobytes() and sh.frame(which, frame, None).tobytes() == cloud.tobytes()
            at = 3 + seed % 5
            out = torch.full((n_max + 16, 4), GUARD, device="cuda")
            n_io = dev(np.array([at], np.int32))
            st = sd.frame_device(which, frame, None if frame == LIDAR else xd, out, n_io)
            o = host(out)
            assert tuple(host(st)) == (FL_OK, n) and int(host(n_io)[0]) == at + n, (which, frame)
            assert o[at:at + n].tobytes() == want.tobytes(), (which, frame)
            assert (o[:at] == GUARD).all() and (o[at + n:] == GUARD).all()
            assert sd.frame(which, frame, x).tobytes() == want.tobytes()


@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("n", [1, 37, 400])
def test_tiny_scans(small, deskew, n):
    pr, tree = small
    r = synth.make_raw_scan(pr.scene, n, pr.x_true, seed=60 + n)
    sh, sd = chains(tree, r, n + 13, deskew)
    check_forms(sh, sd, n + 13, turned_state(pr, n), n)


@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("n", [20_000, 40_000, 65_000])
def test_config4_raw_scans(config4, deskew, n):
    pr, tree = config4
    r = synth.make_raw_scan(pr.scene, n, synth.true_state(pr.cfg.lidar, 3), seed=n + deskew)
    sh, sd = chains(tree, r, n, deskew)
    check_forms(sh, sd, n, turned_state(pr, 7 + n), 7)


def test_device_counts_and_guard_rows(small):
    """*n of 0, 1 and below n_max: rows [at, at + n) written, every other row and the position's neighbours untouched."""
    pr, tree = small
    n_max = 500
    r = synth.make_raw_scan(pr.scene, n_max, pr.x_true, seed=71)
    x = turned_state(pr, 3)
    for n in (0, 1, 321):
        sh, sd = chains(tree, synth.RawScan(r.xyzi[:n], r.offset_ms[:n], r.imu_pose, r.x_end, r.truth_end[:n]), n_max, True)
        for which in (0, 1):
            want = sh.frame(which, WORLD, x)
            k = len(want)
            assert k <= n and (which == 1 or k == n)
            out = torch.full((n_max + 8, 4), GUARD, device="cuda")
            pos = torch.full((3,), 555, dtype=torch.int32, device="cuda")
            pos[1] = 8
            st = sd.frame_device(which, WORLD, dev(x), out, pos[1:2])
            o = host(out)
            assert tuple(host(st)) == (FL_OK, k) and host(pos).tolist() == [555, 8 + k, 555]
            assert o[8:8 + k].tobytes() == want.tobytes() and (o[:8] == GUARD).all() and (o[8 + k:] == GUARD).all()


def test_appends_like_pcl_wait_save(small):
    """Three scans into a buffer whose cap is exactly their total: the concatenation of the host forms.  A fourth is refused
    with (FL_ERR_CAPACITY, n) and changes nothing; a position outside [0, cap] is FL_ERR_ARG."""
    pr, tree = small
    sizes = [900, 1_300, 700]
    scans = [synth.make_raw_scan(pr.scene, n, synth.true_state(pr.cfg.lidar, k), seed=80 + k) for k, n in enumerate(sizes)]
    cap = sum(sizes)
    out = torch.full((cap + 4, 4), GUARD, device="cuda")
    n_io = torch.zeros(1, dtype=torch.int32, device="cuda")
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    want = []
    for k, r in enumerate(scans):
        sh, sd = chains(tree, r, 1_500, True)
        x = turned_state(pr, 20 + k)
        want.append(sh.frame(0, WORLD, x))
        sd.frame_device(0, WORLD, dev(x), out[:cap], n_io, status)
        assert host(status).tolist() == [FL_OK, sizes[k]]
    assert int(host(n_io)[0]) == cap
    before = host(out).copy()
    assert before[:cap].tobytes() == np.concatenate(want).tobytes() and (before[cap:] == GUARD).all()
    sh, sd = chains(tree, scans[0], 1_500, True)
    sd.frame_device(0, WORLD, dev(turned_state(pr, 30)), out[:cap], n_io, status)
    assert host(status).tolist() == [FL_ERR_CAPACITY, sizes[0]] and int(host(n_io)[0]) == cap
    assert host(out).tobytes() == before.tobytes()
    for bad in (-1, cap + 1):
        n_io.fill_(bad)
        sd.frame_device(0, LIDAR, None, out[:cap], n_io, status)
        assert host(status).tolist() == [FL_ERR_ARG, sizes[0]] and int(host(n_io)[0]) == bad
        assert host(out).tobytes() == before.tobytes()
    n_io.fill_(cap - sizes[0])                                   # exactly fits at the end
    sd.frame_device(0, LIDAR, None, out[:cap], n_io, status)
    assert host(status).tolist() == [FL_OK, sizes[0]] and int(host(n_io)[0]) == cap
    assert host(out)[cap - sizes[0]:cap].tobytes() == sh.download(0).tobytes()


def test_refusals_enqueue_nothing(small):
    pr, tree = small
    L = api.load()
    r = synth.make_raw_scan(pr.scene, 600, pr.x_true, seed=90)
    s = api.Scan(tree)
    s.reserve(600, len(r.imu_pose))
    out = torch.full((700, 4), GUARD, device="cuda")
    x = dev(turned_state(pr, 5))
    n_io = dev(np.array([0], np.int32))
    st2 = dev(np.array([9, 9], np.int32))
    hbuf = np.zeros(700 * 4, np.float32)
    hint = np.zeros(4, np.int32)
    stream = torch.cuda.Stream()
    sp = C.c_void_p(stream.cuda_stream)

    def call(which=1, frame=WORLD, x_p=x.data_ptr(), o_p=out.data_ptr(), n_p=n_io.data_ptr(), cap=700, s_p=st2.data_ptr()):
        return L.fl_scan_frame_device(s.h, which, frame, x_p, o_p, n_p, cap, s_p, sp)

    arg = [dict(which=2), dict(which=-1), dict(frame=3), dict(frame=-1), dict(cap=-1), dict(o_p=hbuf.ctypes.data), dict(o_p=out.data_ptr() + 8),
           dict(o_p=None), dict(x_p=x.data_ptr() + 4), dict(x_p=hbuf.ctypes.data), dict(x_p=None), dict(x_p=None, frame=IMU),
           dict(n_p=n_io.data_ptr() + 2), dict(n_p=hint.ctypes.data), dict(n_p=None), dict(s_p=st2.data_ptr() + 1), dict(s_p=hint.ctypes.data),
           dict(s_p=None)]

    def check_all(state):
        for kw in arg:
            assert call(**kw) == FL_ERR_ARG, kw
        for kw in state:
            assert call(**kw) == FL_ERR_STATE, kw

    # no device-form upload yet
    check_all([dict(which=0), dict(which=1), dict(which=0, frame=LIDAR, x_p=None)])
    s.upload_device(dev(r.xyzi), dev(r.offset_ms))
    check_all([dict(which=1)])                                   # no device-form down-sample since the upload
    s.voxel_downsample_device(0.5)
    s.upload(r.xyzi, r.offset_ms)                                # a host-form upload: the device forms need a new one
    check_all([dict(which=0), dict(which=1)])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        check_all([dict(which=0), dict(which=1)])
    g.replay()
    stream.synchronize()
    assert (host(out) == GUARD).all() and host(n_io).tolist() == [0] and host(st2).tolist() == [9, 9]
    # host form
    for which, frame, xh in ((2, WORLD, pr.x_prior), (0, 3, pr.x_prior), (0, WORLD, None), (1, IMU, None)):
        with pytest.raises(api.FastLioError):
            s.frame(which, frame, xh)
    # and the scan still works
    s.upload_device(dev(r.xyzi), dev(r.offset_ms))
    s.voxel_downsample_device(0.5)
    assert tuple(host(s.frame_device(1, WORLD, x, out)))[0] == FL_OK


def test_ordering_behind_a_busy_caller_stream(small):
    """The state is written on the caller's stream behind a long kernel; the call reads it after that."""
    pr, tree = small
    r = synth.make_raw_scan(pr.scene, 5_000, pr.x_true, seed=91)
    sh, sd = chains(tree, r, 5_000, True)
    xs = turned_state(pr, 11)
    want = sh.frame(0, WORLD, xs)
    x = torch.zeros(26, dtype=torch.float64, device="cuda")
    src = dev(xs)
    out = torch.full((5_000, 4), GUARD, device="cuda")
    n_io = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        x.copy_(src)
        st = sd.frame_device(0, WORLD, x, out, n_io)
    torch.cuda.synchronize()
    assert tuple(host(st)) == (FL_OK, 5_000) and host(out).tobytes() == want.tobytes()


def test_first_scan_builds_the_map(small):
    """Map initialisation (:909-921): the down-sampled cloud in the world frame with the predicted state, built through
    fl_map_build_device, equals KdTree.Build of the restated cloud."""
    pr, tree = small
    r = synth.make_raw_scan(pr.scene, 8_000, pr.x_true, seed=92)
    sh, sd = chains(tree, r, 8_000, True)
    x = turned_state(pr, 13)
    down = sh.download(1)
    want = restated(down, WORLD, x)
    out = torch.zeros((8_000, 4), device="cuda")
    st = sd.frame_device(1, WORLD, dev(x), out)
    n = int(host(st)[1])
    assert n == len(down) > 5
    built, ref = api.KdTree(0, 0.5), api.KdTree(0, 0.5)
    built.build_device(out[:n])
    ref.Build(want)
    same_map(ref, built, want[::3].copy())


def test_one_graph_with_the_published_clouds(problems):
    """upload -> undistort -> down-sample -> update -> map_incremental -> a memset of the publish positions -> the dense world
    cloud, the dense IMU-frame cloud and the dense world cloud appended, captured once and replayed over 20 raw scans: every
    scan's clouds, the accumulated cloud and the final x, P and map equal the host-form chain followed by fl_scan_frame."""
    pr = problems("small")
    n_max, leaf, n_scans = 9_000, 0.5, 20
    scans = stream_of_raw_scans(pr, n_scans, n_max)
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
    world = torch.full((n_max, 4), GUARD, device="cuda")
    imu = torch.full((n_max, 4), GUARD, device="cuda")
    cap = sum(len(r.xyzi) for r in scans)
    save = torch.full((cap + 8, 4), GUARD, device="cuda")
    pub = torch.full((2,), 99, dtype=torch.int32, device="cuda")
    n_save = torch.zeros(1, dtype=torch.int32, device="cuda")
    fst = torch.zeros((3, 2), dtype=torch.int32, device="cuda")

    def fill(r):
        xyzi[:len(r.xyzi)] = dev(r.xyzi); tms[:len(r.xyzi)] = dev(r.offset_ms); n_d.fill_(len(r.xyzi))
        poses[:len(r.imu_pose)] = dev(r.imu_pose); np_d.fill_(len(r.imu_pose)); xend.copy_(dev(r.x_end))

    def chain():
        sd.upload_device(xyzi, tms, n_d, n_max)
        sd.undistort_device(poses, np_d, xend)
        sd.voxel_downsample_device(leaf)
        sd.update_device(fd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)
        pub.zero_()
        sd.frame_device(0, WORLD, xd, world, pub[0:1], fst[0])
        sd.frame_device(0, IMU, xd, imu, pub[1:2], fst[1])
        sd.frame_device(0, WORLD, xd, save[:cap], n_save, fst[2])

    side = torch.cuda.Stream()
    g, saved, replays = None, [], 0
    for step, r in enumerate(scans):
        sh.upload(r.xyzi, r.offset_ms); sh.undistort(r.imu_pose, r.x_end); sh.voxel_downsample(leaf)
        xh, Ph, _ = sh.update(fh, xh, Ph, pr.R)
        o3 = fh.map_incremental(0.5, True)
        want_w, want_i = sh.frame(0, WORLD, xh), sh.frame(0, IMU, xh)
        saved.append(want_w)
        fill(r)
        torch.cuda.synchronize()
        if step == 0:
            with torch.cuda.stream(side):
                chain()
            torch.cuda.synchronize()
        else:
            if g is None:
                td.maintain()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    chain()
            g.replay()
            replays += 1
        n = len(r.xyzi)
        o = host(out4)
        assert host(status)[0] == FL_OK and tuple(int(v) for v in o[:3]) == o3, step
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), step
        assert host(fst).tolist() == [[FL_OK, n]] * 3 and host(pub).tolist() == [n, n], step
        assert host(world)[:n].tobytes() == want_w.tobytes() and host(imu)[:n].tobytes() == want_i.tobytes(), step
        if o[3] == 1 and td.maintain():
            g = None
    assert replays == n_scans - 1
    assert int(host(n_save)[0]) == cap
    s = host(save)
    assert s[:cap].tobytes() == np.concatenate(saved).tobytes() and (s[cap:] == GUARD).all()
    td.maintain()
    same_map(th, td, scans[-1].xyzi[::5].copy(), size=False)


def test_plain_c_program(problems, tmp_path):
    """tests/facade/scan_frame_device.cu: the C ABI alone captures the chain with the three frame calls and replays it."""
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
    exe = tmp_path / "scan_frame_device"
    cmd = [build._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "facade", "scan_frame_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    res = subprocess.run([str(exe), str(inp)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "all equal" in res.stdout, res.stdout + res.stderr
