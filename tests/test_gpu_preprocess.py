"""Preprocess::process on the device (fl_preprocess, fl_preprocess_device) against the reference's own preprocess.cpp, live
or replayed (tests/golden/ref/preprocess_gpu.npz), on full-size raw frames of the four LiDAR types; device counts, guard
bytes, an unaligned layout, the dropped-ring count, refusals, stream ordering, and one CUDA graph from raw points to
map_incremental."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import preprocess_rules as R
from fast_lio_b200 import api, build, synth
from refcalls import digest
from refpreprocess import RefPreprocess
from test_gpu_frontend_device import same_map, stream_of_raw_scans, twins

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_CAPACITY = 0, -2, -5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = {R.AVIA: dict(n_scans=6, scan_rate=10, time_unit=R.NS), R.VELO16: dict(n_scans=32, scan_rate=10, time_unit=R.US),
       R.OUST64: dict(n_scans=64, scan_rate=10, time_unit=R.NS), R.MARSIM: dict(n_scans=1, scan_rate=10, time_unit=R.US)}
GUARD = 77


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def ref():
    return RefPreprocess("preprocess_gpu")


# (name, lidar type, frame, point_filter_num, blind)
def _frames():
    return [("avia_24k", R.AVIA, lambda: synth.raw_frame("avia", seed=1, blind=0.5), 1, 0.5),
            ("avia_24k_pfn3", R.AVIA, lambda: synth.raw_frame("avia", seed=1, blind=2.0), 3, 2.0),
            ("velo32x1800_times", R.VELO16, lambda: synth.raw_frame("velodyne", seed=2, blind=0.5), 2, 0.5),
            ("velo32x1800_yaw", R.VELO16, lambda: synth.raw_frame("velodyne", seed=3, blind=0.5, yaw0_deg=-123.0, times=False), 1, 0.5),
            ("velo32x1800_yaw_pfn4", R.VELO16, lambda: synth.raw_frame("velodyne", seed=3, blind=2.0, yaw0_deg=-123.0, times=False), 4, 2.0),
            ("ouster64x1024", R.OUST64, lambda: synth.raw_frame("ouster", seed=4, blind=0.5), 1, 0.5),
            ("ouster64x1024_pfn4", R.OUST64, lambda: synth.raw_frame("ouster", seed=4, blind=2.0), 4, 2.0),
            ("marsim", R.MARSIM, lambda: synth.raw_frame("marsim", seed=5, blind=0.5), 3, 0.5)]


def yaw_bound(raw, omega_l):
    """Per raw row: 1 ulp of the float yaw (radians) of the row and of its ring's first row, through 57.2957 / omega_l.  The
    device rounds atan2 in double to float where the reference calls atan2f, which is not correctly rounded (DESIGN §4c)."""
    yaw = np.arctan2(raw["y"].astype(np.float64), raw["x"].astype(np.float64)).astype(np.float32)
    first = {}
    for i, r in enumerate(raw["ring"]):
        first.setdefault(int(r), i)
    yfp = yaw[[first[int(r)] for r in raw["ring"]]]
    return (np.spacing(np.abs(yaw)) + np.spacing(np.abs(yfp))).astype(np.float64) * 57.2957 / omega_l


def check_against_ref(want, xyzi, ms, last, yaw_path, raw=None, omega_l=None):
    assert len(ms) == want["count"]
    assert digest(np.ascontiguousarray(xyzi)) == want["xyzi_digest"]      # the count, the order and the x/y/z/intensity bytes
    if not yaw_path:
        assert digest(np.ascontiguousarray(ms)) == want["ms_digest"]
        assert np.float32(last).tobytes() == want["last_ms"].tobytes()
        return
    # the yaw-derived times: within the bound, row by row (output rows are matched to raw rows by their exact x/y/z bytes)
    xyz = np.ascontiguousarray(np.stack([raw["x"], raw["y"], raw["z"]], 1))
    row = {r.tobytes(): i for i, r in enumerate(xyz)}
    idx = np.array([row[p.tobytes()] for p in np.ascontiguousarray(xyzi[:, :3])], np.int64)
    ref_ms = want["ms"].astype(np.float64)
    tol = yaw_bound(raw, omega_l)[idx] + np.spacing(np.abs(want["ms"])).astype(np.float64)
    d = np.abs(ms.astype(np.float64) - ref_ms)
    assert (d <= tol).all(), float((d - tol).max())
    assert d.max() < 0.25 * 360.0 / omega_l          # so each row took the same wrap decision (lo or hi) as the reference
    assert abs(float(last) - float(want["last_ms"])) <= tol[-1]


@pytest.mark.parametrize("case", range(len(_frames())), ids=[f[0] for f in _frames()])
def test_forms_against_reference(ref, case):
    name, t, make, pfn, blind = _frames()[case]
    raw = make()
    cfg = CFG[t]
    yaw_path = name.startswith("velo") and "yaw" in name
    want = ref.process(raw, api.layout_offsets(raw.dtype, t), t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, blind,
                       keep_ms=yaw_path)
    n = len(raw)
    pp = api.Preprocess(0, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, blind, n_raw_max=n + 300)
    xyzi, ms, last = pp.process(raw)
    check_against_ref(want, xyzi, ms, last, yaw_path, raw, 0.361 * cfg["scan_rate"])
    # device form: n held in device memory below n_max, guard bytes past the output rows
    n_max = n + 300
    buf = np.zeros((n_max, raw.dtype.itemsize), np.uint8)
    buf[:n] = raw.view(np.uint8).reshape(n, -1)
    buf[n:] = 0xA5
    xo = torch.full((n_max, 4), float(GUARD), device="cuda")
    mo = torch.full((n_max,), float(GUARD), device="cuda")
    out2 = torch.zeros(2, dtype=torch.int32, device="cuda")
    lo = torch.zeros(1, device="cuda")
    pp.process_device(dev(buf), dev(np.array([n], np.int32)), n_max, xo, mo, out2, lo)
    o2 = host(out2)
    k = int(o2[0])
    assert k == want["count"] and o2[1] == 0
    xd, md = host(xo), host(mo)
    assert xd[:k].tobytes() == xyzi.tobytes() and md[:k].tobytes() == ms.tobytes() and host(lo)[0] == np.float32(last)
    assert (xd[k:] == GUARD).all() and (md[k:] == GUARD).all()


@pytest.mark.parametrize("t", [R.AVIA, R.VELO16, R.OUST64, R.MARSIM])
def test_small_device_counts(t):
    """n in {0, 1, 2, 40} with n_max 64: the rules' pl_surf, guard rows untouched; last_ms 0 when nothing is kept."""
    cfg = CFG[t]
    kind = {R.AVIA: "avia", R.VELO16: "velodyne", R.OUST64: "ouster", R.MARSIM: "marsim"}[t]
    raw = synth.raw_frame(kind, seed=9, **({"n": 64} if t in (R.AVIA, R.MARSIM) else {"rings": 8, "cols": 8}))
    pp = api.Preprocess(0, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5, n_raw_max=64)
    draw = dev(raw.view(np.uint8).reshape(len(raw), -1))
    for n in (0, 1, 2, 40):
        wx, wm = R.process(raw[:n], api.layout_offsets(raw.dtype, t), t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5)
        xo = torch.full((64, 4), float(GUARD), device="cuda")
        mo = torch.full((64,), float(GUARD), device="cuda")
        xyzi, ms, out2, last = pp.process_device(draw, dev(np.array([n], np.int32)), 64, xo, mo)
        k = int(host(out2)[0])
        assert k == len(wm), (n, k, len(wm))
        assert host(xo)[:k].tobytes() == wx.tobytes() and host(mo)[:k].tobytes() == wm.tobytes()
        assert (host(xo)[k:] == GUARD).all() and (host(mo)[k:] == GUARD).all()
        assert host(last)[0] == (wm[-1] if k else 0.0)
        hx, hm, hl = pp.process(raw[:n])
        assert hx.tobytes() == wx.tobytes() and hm.tobytes() == wm.tobytes()


def test_unaligned_layout(ref):
    """A 22-byte point_step with every field at an odd offset (an Ouster cloud repacked by a driver)."""
    src = synth.raw_frame("ouster", seed=6, blind=0.5)
    dt = np.dtype({"names": ["x", "y", "z", "intensity", "t"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u4"],
                   "offsets": [1, 5, 9, 13, 17], "itemsize": 22})
    raw = np.zeros(len(src), dt)
    for f in dt.names:
        raw[f] = src[f]
    cfg = CFG[R.OUST64]
    off = api.layout_offsets(dt, R.OUST64)
    want = ref.process(raw, off, R.OUST64, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 2, 0.5)
    pp = api.Preprocess(0, R.OUST64, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 2, 0.5, layout=dt, n_raw_max=len(raw))
    xyzi, ms, last = pp.process(raw)
    check_against_ref(want, xyzi, ms, last, False)
    xo, mo, out2, lo = pp.process_device(dev(raw.view(np.uint8)))
    k = int(host(out2)[0])
    assert host(xo)[:k].tobytes() == xyzi.tobytes() and host(mo)[:k].tobytes() == ms.tobytes()


def test_dropped_rings():
    """Rows with ring >= N_SCANS on the Velodyne yaw path are dropped and counted; the rest is the rules' pl_surf of the frame
    without them (the reference is never given such rows).  With point times the ring is not read, and nothing is dropped."""
    raw = synth.raw_frame("velodyne", seed=7, rings=16, cols=100, times=False)
    raw["ring"][raw["ring"] >= 14] += 20                       # rings 34, 35 with N_SCANS 16
    bad = raw["ring"] >= 16
    cfg = dict(CFG[R.VELO16], n_scans=16)
    pp = api.Preprocess(0, R.VELO16, 16, 10, R.US, 1, 0.5, n_raw_max=len(raw))
    xo, mo, out2, lo = pp.process_device(dev(raw.view(np.uint8)))
    o2 = host(out2)
    assert o2[1] == bad.sum() > 0
    wx, wm = R.process(raw[~bad], api.layout_offsets(raw.dtype, R.VELO16), R.VELO16, 16, 10, R.US, 1, 0.5)
    assert o2[0] == len(wm) and host(xo)[:o2[0]].tobytes() == wx.tobytes()
    timed = raw.copy()
    timed["time"] = np.linspace(0, 1e5, len(raw), dtype=np.float32)
    _, _, out2, _ = pp.process_device(dev(timed.view(np.uint8)))
    wx, wm = R.process(timed, api.layout_offsets(raw.dtype, R.VELO16), R.VELO16, 16, 10, R.US, 1, 0.5)
    assert tuple(host(out2)) == (len(wm), 0)


def test_refusals_enqueue_nothing():
    L = api.load()
    raw = synth.raw_frame("marsim", seed=8, n=500)
    pp = api.Preprocess(0, R.MARSIM, 1, 10, R.US, 1, 0.5, n_raw_max=500)
    d = dev(raw.view(np.uint8))
    n = dev(np.array([500], np.int32))
    xo = torch.full((600, 4), float(GUARD), device="cuda")
    mo = torch.full((600,), float(GUARD), device="cuda")
    out2 = torch.full((2,), 9, dtype=torch.int32, device="cuda")
    lo = torch.full((1,), float(GUARD), device="cuda")
    s = torch.cuda.Stream()
    st = C.c_void_p(s.cuda_stream)
    hbuf = np.zeros(600 * 4, np.float32)

    def call(raw_p=d.data_ptr(), n_p=n.data_ptr(), n_max=500, x_p=xo.data_ptr(), m_p=mo.data_ptr(), o_p=out2.data_ptr(), l_p=lo.data_ptr()):
        return L.fl_preprocess_device(pp.h, raw_p, n_p, n_max, x_p, m_p, o_p, l_p, st)

    cases = [(dict(n_max=501), FL_ERR_CAPACITY), (dict(raw_p=None), FL_ERR_ARG), (dict(n_p=None), FL_ERR_ARG),
             (dict(x_p=xo.data_ptr() + 4), FL_ERR_ARG), (dict(m_p=hbuf.ctypes.data), FL_ERR_ARG), (dict(o_p=None), FL_ERR_ARG),
             (dict(l_p=lo.data_ptr() + 1), FL_ERR_ARG), (dict(n_max=-1), FL_ERR_ARG)]
    for kw, rc in cases:
        assert call(**kw) == rc, kw
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for kw, rc in cases:
            assert call(**kw) == rc, kw
    g.replay()
    s.synchronize()
    assert (host(xo) == GUARD).all() and (host(mo) == GUARD).all() and (host(out2) == 9).all() and host(lo)[0] == GUARD
    # bad parameters at creation
    for kw in (dict(lidar_type=5), dict(time_unit=4), dict(point_filter_num=0), dict(n_scans=0), dict(n_scans=129)):
        args = dict(device=0, lidar_type=R.MARSIM, n_scans=1, scan_rate=10, time_unit=R.US, point_filter_num=1, blind=0.5,
                    layout=api.POINT_XYZI)
        args.update(kw)
        with pytest.raises(api.FastLioError):
            api.Preprocess(**args)
    # a field past point_step: t (u32) at bytes 8-11 of a 10-byte point
    bad = api.PreprocessParams(R.OUST64, 64, 10, R.NS, 1, 0.5, 10, 0, 4, -1, -1, 8, -1, -1, -1)
    h = C.c_void_p()
    assert L.fl_preprocess_create(C.byref(h), 0, C.byref(bad), 100) == FL_ERR_ARG and not h.value
    with pytest.raises(api.FastLioError):
        big = np.zeros(501, raw.dtype)                             # 501 rows above n_raw_max
        big[:500] = raw
        pp.process(big)


def test_ordering_behind_a_busy_caller_stream():
    """The raw bytes are written on the caller's stream behind a long kernel; the call sees them."""
    raw = synth.raw_frame("avia", seed=10, n=20000)
    pp = api.Preprocess(0, R.AVIA, 6, 10, R.NS, 2, 0.5, n_raw_max=len(raw))
    want = pp.process(raw)
    s = torch.cuda.Stream()
    src = dev(raw.view(np.uint8))
    with torch.cuda.stream(s):
        d = torch.zeros_like(src)
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(20):
            big = big @ big / 64.0                                # keeps the stream busy
        d.copy_(src)
        xo, mo, out2, lo = pp.process_device(d)
    k = int(host(out2)[0])
    assert k == len(want[1]) and host(xo)[:k].tobytes() == want[0].tobytes() and host(mo)[:k].tobytes() == want[1].tobytes()


def _avia_from_scan(r, seed):
    rng = np.random.default_rng(seed)
    n = len(r.xyzi)
    a = np.zeros(n + 1, api.CUSTOM_POINT)                         # row 0 is never output: a dummy first row
    a["x"][1:], a["y"][1:], a["z"][1:] = r.xyzi[:, 0], r.xyzi[:, 1], r.xyzi[:, 2]
    a["offset_time"][1:] = (np.clip(r.offset_ms, 0, None) * 1e6).astype(np.uint32)
    a["reflectivity"][1:] = rng.integers(0, 256, n)
    a["tag"] = 0x10
    a["line"] = np.arange(n + 1) % 6
    return a


def test_one_graph_from_raw_points(ref, problems):
    """preprocess -> upload -> undistort -> down-sample -> update -> map_incremental captured once and replayed over 20 raw
    Avia frames of different sizes: x, P and the map equal the host-form chain fed with the reference's pl_surf."""
    pr = problems("small")
    n_max, leaf = 9_000, 0.5
    scans = stream_of_raw_scans(pr, 20, n_max - 1)
    frames = [_avia_from_scan(r, 100 + i) for i, r in enumerate(scans)]
    cfg = CFG[R.AVIA]
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=n_max, max_iter=3) for t in (th, td))
    sh, sd = api.Scan(th), api.Scan(td)
    sd.reserve(n_max, 2)
    pp = api.Preprocess(0, R.AVIA, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5, n_raw_max=n_max)
    raw_d = torch.zeros((n_max, 20), dtype=torch.uint8, device="cuda")
    n_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    xyzi = torch.zeros((n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros(n_max, dtype=torch.float32, device="cuda")
    out2 = torch.zeros(2, dtype=torch.int32, device="cuda")
    last = torch.zeros(1, dtype=torch.float32, device="cuda")
    poses = torch.zeros((2, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    xend = dev(pr.x_prior)
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd = dev(xh), dev(Ph)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    out4 = torch.zeros(4, dtype=torch.int32, device="cuda")

    def chain():
        pp.process_device(raw_d, n_d, n_max, xyzi, tms, out2, last)
        sd.upload_device(xyzi, tms, out2[:1], n_max)
        sd.undistort_device(poses, np_d, xend)
        sd.voxel_downsample_device(leaf)
        sd.update_device(fd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)

    side = torch.cuda.Stream()
    g = None
    for step, a in enumerate(frames):
        want = ref.process(a, api.layout_offsets(a.dtype, R.AVIA), R.AVIA, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5)
        px, pm, _ = pp.process(a)
        assert digest(px) == want["xyzi_digest"] and digest(pm) == want["ms_digest"], step   # the host chain's input is pl_surf
        sh.upload(px, pm); sh.undistort(np.zeros((0, 22)), pr.x_prior); sh.voxel_downsample(leaf)
        xh, Ph, _ = sh.update(fh, xh, Ph, pr.R)
        fh.map_incremental(0.5, True)
        raw_d[:len(a)] = dev(a.view(np.uint8).reshape(len(a), -1))
        n_d.fill_(len(a))
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
        o = host(out4)
        assert host(out2)[0] == want["count"] and host(status)[0] == FL_OK, step
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), step
        if o[3] == 1 and td.maintain():
            g = None
    td.maintain()
    same_map(th, td, scans[-1].xyzi[::5].copy())


def test_plain_c_program(tmp_path):
    """tests/facade/preprocess_device.cu: the C ABI from a plain CUDA program, one captured graph replayed."""
    exe = tmp_path / "preprocess_device"
    nvcc = build._nvcc()
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-ccbin", "/usr/bin/g++", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "facade", "preprocess_device.cu"), "-o", str(exe), "-L", os.path.dirname(build.LIB),
                    "-lfastlio_b200", "-Xlinker", f"-rpath={os.path.dirname(build.LIB)}"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "preprocess_device ok" in out.stdout
