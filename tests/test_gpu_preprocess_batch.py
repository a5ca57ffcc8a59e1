"""Preprocess::process of many raw frames in one call (fl_preprocess_batch_run_device): every slot's pl_surf rows, offset times,
out2 and last_ms equal, byte for byte, a twin fl_preprocess_device call on the same frame and count; refused slots write no row,
change no other slot and are refused again by the scan batch and the batched update; the call follows the device forms'
ordering and graph rules, and a fleet graph from raw Avia frames equals per-robot chains."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import preprocess_rules as R
from fast_lio_b200 import api, build, synth
from refpreprocess import RefPreprocess
from test_gpu_preprocess import CFG, _avia_from_scan, check_against_ref

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_CAPACITY = 0, -2, -5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 77.0
KIND = {R.AVIA: "avia", R.VELO16: "velodyne", R.OUST64: "ouster", R.MARSIM: "marsim"}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def frame(t, seed, size, times=True, dt=None):
    """A raw frame of about `size` points of type t (Velodyne on the yaw path when not `times`), in layout dt when given."""
    if t in (R.AVIA, R.MARSIM):
        a = synth.raw_frame(KIND[t], seed=seed, n=size)
    else:
        rings = 16 if t == R.VELO16 else 32
        a = synth.raw_frame(KIND[t], seed=seed, rings=rings, cols=max(size // rings, 2), times=times,
                            **({"yaw0_deg": float(seed % 360 - 180)} if t == R.VELO16 else {}))
    if dt is None:
        return a
    b = np.zeros(len(a), dt)
    for f in dt.names:
        b[f] = a[f]
    return b


def handles(t, pfn, S_max, n_raw_max, n_scans=None, layout=None):
    cfg = dict(CFG[t])
    if n_scans is not None:
        cfg["n_scans"] = n_scans
    args = (0, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, 0.5)
    return (api.PreprocessBatch(*args, layout=layout, n_slots_max=S_max, n_raw_max=n_raw_max),
            api.Preprocess(*args, layout=layout, n_raw_max=n_raw_max))


class Slots:
    """Per slot a raw buffer of n_max rows (0xA5 past the frame) and a device count; the same tensors feed the batch and the twin."""

    def __init__(self, frames, counts, n_max, step):
        self.bufs, self.ns = [], []
        for a, c in zip(frames, counts):
            buf = np.full((n_max, step), 0xA5, np.uint8)
            k = min(len(a), n_max)
            buf[:k] = a[:k].view(np.uint8).reshape(k, -1)
            self.bufs.append(dev(buf))
            self.ns.append(dev(np.array([c], np.int32)))

    def table(self):
        return api.preprocess_raws(list(zip(self.bufs, self.ns)))


def guard_outputs(pb):
    xyzi, ms, out2, last = pb.outputs()
    xyzi.fill_(GUARD); ms.fill_(GUARD); out2.fill_(-7); last.fill_(GUARD)
    return xyzi, ms, out2, last


def twin_out(pp, buf, n, n_max):
    xo = torch.full((max(n_max, 1), 4), GUARD, device="cuda")
    mo = torch.full((max(n_max, 1),), GUARD, device="cuda")
    out2 = torch.zeros(2, dtype=torch.int32, device="cuda")
    lo = torch.zeros(1, device="cuda")
    pp.process_device(buf, n, n_max, xo, mo, out2, lo)
    o2 = host(out2)
    return host(xo)[:o2[0]], host(mo)[:o2[0]], o2, host(lo)[0]


def check_slots(pb, pp, sl, n_max, status, slots, refused=()):
    """Every accepted slot equals its twin, rows past its count keep the guard; refused slots (index -> status) wrote nothing."""
    xyzi, ms, out2, last = (host(t) for t in pb.outputs())
    st = host(status)
    for s in slots:
        if s in refused:
            assert tuple(st[s]) == (refused[s], 0), (s, st[s])
            assert tuple(out2[s]) == (-1, 0) and last[s] == 0.0, s
            assert (xyzi[s] == GUARD).all() and (ms[s] == GUARD).all(), s
            continue
        wx, wm, wo2, wl = twin_out(pp, sl.bufs[s], sl.ns[s], n_max)
        k = int(wo2[0])
        assert tuple(st[s]) == (FL_OK, k), (s, st[s], k)
        assert tuple(out2[s]) == tuple(wo2), (s, out2[s], wo2)
        assert xyzi[s, :k].tobytes() == wx.tobytes() and ms[s, :k].tobytes() == wm.tobytes(), s
        assert last[s].tobytes() == np.float32(wl).tobytes(), s
        assert (xyzi[s, k:] == GUARD).all() and (ms[s, k:] == GUARD).all(), s


CASES = [("avia", R.AVIA, True), ("velo_times", R.VELO16, True), ("velo_yaw", R.VELO16, False), ("ouster", R.OUST64, True),
         ("marsim", R.MARSIM, True)]


@pytest.mark.parametrize("pfn", [1, 3])
@pytest.mark.parametrize("S", [1, 3, 64])
@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_each_slot_equals_its_twin(case, S, pfn):
    """Counts 0, 1, 2, random and n_max among the slots, S_max above S so some slots stay uncovered (out2 = (-1, 0))."""
    _, t, times = CASES[case]
    rng = np.random.default_rng(100 * case + S + pfn)
    n_max = 4_000 if S == 64 else 12_000
    pb, pp = handles(t, pfn, S + 2, n_max)
    frames = [frame(t, 1000 * case + s, n_max if s == S - 1 else int(rng.integers(n_max // 2, n_max + 1)), times) for s in range(S)]
    counts = [int(rng.integers(0, min(len(a), n_max) + 1)) for a in frames]
    for s, c in zip(range(S), (0, 1, 2, min(len(frames[-1]), n_max))):
        counts[(s * 7) % S] = min(c, len(frames[(s * 7) % S]))
    sl = Slots(frames, counts, n_max, pb.layout.itemsize)
    guard_outputs(pb)
    status = pb.run_device(sl.table(), S, n_max)
    check_slots(pb, pp, sl, n_max, status, range(S))
    o2 = host(pb.outputs()[2])
    assert (o2[S:] == np.array([-1, 0])).all()


def test_dropped_rings_unaligned_layout_and_shared_buffers():
    """Velodyne yaw-path frames with rings >= N_SCANS (dropped and counted per slot), a 22-byte Ouster layout with every field at
    an odd offset, and slots that share one raw buffer with different counts."""
    n_max = 3_200
    pb, pp = handles(R.VELO16, 1, 5, n_max, n_scans=16)
    frames = []
    for s in range(5):
        a = synth.raw_frame("velodyne", seed=40 + s, rings=16, cols=200, times=False)
        if s % 2 == 0:
            a["ring"][a["ring"] >= 14] += 20
        frames.append(a)
    sl = Slots(frames, [len(a) for a in frames], n_max, pb.layout.itemsize)
    sl.bufs[4] = sl.bufs[0]                                        # slot 4 reads slot 0's buffer, 1 000 rows of it
    sl.ns[4] = dev(np.array([1000], np.int32))
    guard_outputs(pb)
    status = pb.run_device(sl.table(), 5, n_max)
    check_slots(pb, pp, sl, n_max, status, range(5))
    o2 = host(pb.outputs()[2])
    assert o2[0, 1] > 0 and o2[1, 1] == 0 and o2[2, 1] > 0

    dt = np.dtype({"names": ["x", "y", "z", "intensity", "t"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u4"],
                   "offsets": [1, 5, 9, 13, 17], "itemsize": 22})
    pb, pp = handles(R.OUST64, 2, 3, 8_192, layout=dt)
    frames = [frame(R.OUST64, 50 + s, 8_192, dt=dt) for s in range(3)]
    sl = Slots(frames, [8_192, 5_000, 8_192], 8_192, 22)
    sl.bufs[2] = sl.bufs[0]
    guard_outputs(pb)
    status = pb.run_device(sl.table(), 3, 8_192)
    check_slots(pb, pp, sl, 8_192, status, range(3))


@pytest.fixture(scope="module")
def ref():
    return RefPreprocess("preprocess_gpu")


def test_full_size_frames_against_the_reference(ref):
    """One full-size frame per type (the frames of test_gpu_preprocess) in one slot among others, against the recorded answers."""
    cases = [("avia_24k", R.AVIA, synth.raw_frame("avia", seed=1, blind=0.5), 1, False),
             ("velo32x1800_yaw", R.VELO16, synth.raw_frame("velodyne", seed=3, blind=0.5, yaw0_deg=-123.0, times=False), 1, True),
             ("ouster64x1024", R.OUST64, synth.raw_frame("ouster", seed=4, blind=0.5), 1, False),
             ("marsim", R.MARSIM, synth.raw_frame("marsim", seed=5, blind=0.5), 3, False)]
    for name, t, raw, pfn, yaw_path in cases:
        cfg = CFG[t]
        want = ref.process(raw, api.layout_offsets(raw.dtype, t), t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, 0.5,
                           keep_ms=yaw_path)
        n_max = len(raw) + 64
        pb = api.PreprocessBatch(0, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, 0.5, n_slots_max=3, n_raw_max=n_max)
        sl = Slots([raw[:100], raw, raw[::-1].copy()], [100, len(raw), len(raw)], n_max, raw.dtype.itemsize)
        st = host(pb.run_device(sl.table(), 3, n_max))
        assert (st[:, 0] == FL_OK).all(), name
        xyzi, ms, last = pb.download(1)
        check_against_ref(want, xyzi, ms, last, yaw_path, raw, 0.361 * cfg["scan_rate"])


def test_refused_slots_and_the_later_stages_refuse_them(problems):
    """Null and misaligned counts, c < 0, a null raw with c > 0 and c > n_max: each slot's status, out2 = (-1, 0), no row; the
    other slots equal their twins; fed on through the scan batch and the batched update, the refused slots are refused there."""
    n_max = 2_000
    pb, pp = handles(R.AVIA, 1, 8, n_max)
    frames = [frame(R.AVIA, 70 + s, n_max) for s in range(8)]
    sl = Slots(frames, [n_max] * 8, n_max, pb.layout.itemsize)
    bad_n = torch.tensor([5, 5], dtype=torch.int32, device="cuda")
    entries = list(zip(sl.bufs, sl.ns))
    entries[1] = (sl.bufs[1], None)                                               # null count
    entries[2] = (sl.bufs[2], bad_n.data_ptr() + 2)                               # misaligned count
    entries[3] = (sl.bufs[3], dev(np.array([-1], np.int32)))                       # c < 0
    entries[4] = (None, sl.ns[4])                                                 # null raw with c > 0
    entries[5] = (sl.bufs[5], dev(np.array([n_max + 1], np.int32)))                # c > n_max
    entries[6] = (None, dev(np.array([0], np.int32)))                              # null raw with c = 0: accepted, empty
    keep = [e[1] for e in entries]
    guard_outputs(pb)
    status = pb.run_device(api.preprocess_raws(entries), 8, n_max)
    refused = {1: FL_ERR_ARG, 2: FL_ERR_ARG, 3: FL_ERR_ARG, 4: FL_ERR_ARG, 5: FL_ERR_CAPACITY}
    check_slots(pb, pp, sl, n_max, status, [0, 1, 2, 3, 4, 5, 7], refused)
    st, o2 = host(status), host(pb.outputs()[2])
    assert tuple(st[6]) == (FL_OK, 0) and tuple(o2[6]) == (0, 0)
    del keep
    # the scan batch reads out2[s, 0] = -1 as c < 0; the update refuses the slot the scan batch refused
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    sb = api.ScanBatch(t)
    sb.reserve(8, n_max, 2)
    sstatus = sb.run_device(pb.scan_raws(), n_max, 2, 0.5, undistort=False)
    f = api.Esekf(t, max_points=n_max, max_iter=3)
    f.reserve_batch(n_max)
    refs, m = sb.refs(1)
    x = dev(np.stack([pr.x_prior] * 8))
    P = dev(np.stack([pr.P_prior] * 8))
    ustatus = torch.zeros((8, 2), dtype=torch.int32, device="cuda")
    f.update_scans_device(refs[:8], x, P, m, pr.R, ustatus)
    ss, us = host(sstatus), host(ustatus)
    for s in refused:
        assert ss[s][0] == FL_ERR_ARG and us[s][0] == FL_ERR_ARG, (s, ss[s], us[s])
    for s in (0, 7):
        assert ss[s][0] == FL_OK and us[s][0] == FL_OK, (s, ss[s], us[s])


def test_host_refusals_enqueue_nothing():
    L = api.load()
    n_max = 500
    pb, _ = handles(R.MARSIM, 1, 2, n_max)
    sl = Slots([frame(R.MARSIM, 3, n_max)] * 2, [n_max] * 2, n_max, pb.layout.itemsize)
    table = sl.table()
    status = torch.full((2, 2), 9, dtype=torch.int32, device="cuda")
    hstat = np.zeros(4, np.int32)
    htab = np.zeros(4, np.int64)
    s = torch.cuda.Stream()
    st = C.c_void_p(s.cuda_stream)

    def call(t=table.data_ptr(), n=2, m=n_max, o=status.data_ptr()):
        return L.fl_preprocess_batch_run_device(pb.h, t, n, m, o, st)

    cases = [(dict(n=-1), FL_ERR_ARG), (dict(m=-1), FL_ERR_ARG), (dict(t=None), FL_ERR_ARG), (dict(t=table.data_ptr() + 4), FL_ERR_ARG),
             (dict(t=htab.ctypes.data), FL_ERR_ARG), (dict(o=None), FL_ERR_ARG), (dict(o=status.data_ptr() + 2), FL_ERR_ARG),
             (dict(o=hstat.ctypes.data), FL_ERR_ARG), (dict(n=3), FL_ERR_CAPACITY), (dict(m=n_max + 1), FL_ERR_CAPACITY)]
    guard_outputs(pb)
    torch.cuda.synchronize()
    for kw, rc in cases:
        assert call(**kw) == rc, kw
    assert call(n=0, t=None, o=None) == FL_OK
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for kw, rc in cases:
            assert call(**kw) == rc, kw
    g.replay()
    s.synchronize()
    xyzi, ms, out2, last = (host(t) for t in pb.outputs())
    assert (host(status) == 9).all() and (xyzi == GUARD).all() and (out2 == -7).all() and (last == GUARD).all()
    # creation: bad parameters as fl_preprocess_create, and the slot bounds
    p = api.PreprocessParams(R.MARSIM, 1, 10, R.US, 1, 0.5, 32, 0, 4, 8, 16, -1, -1, -1, -1)
    h = C.c_void_p()
    assert L.fl_preprocess_batch_create(C.byref(h), 0, C.byref(p), 65536, 1) == FL_ERR_CAPACITY and not h.value
    assert L.fl_preprocess_batch_create(C.byref(h), 0, C.byref(p), 65536 // 2, 1 << 16) == FL_ERR_CAPACITY and not h.value
    assert L.fl_preprocess_batch_create(C.byref(h), 0, C.byref(p), -1, 10) == FL_ERR_ARG and not h.value
    bad = api.PreprocessParams(R.OUST64, 64, 10, R.NS, 1, 0.5, 10, 0, 4, -1, -1, 8, -1, -1, -1)
    assert L.fl_preprocess_batch_create(C.byref(h), 0, C.byref(bad), 2, 100) == FL_ERR_ARG and not h.value
    for kw in (dict(lidar_type=5), dict(time_unit=4), dict(point_filter_num=0), dict(n_scans=129)):
        args = dict(device=0, lidar_type=R.MARSIM, n_scans=1, scan_rate=10, time_unit=R.US, point_filter_num=1, blind=0.5,
                    layout=api.POINT_XYZI, n_slots_max=2, n_raw_max=10)
        args.update(kw)
        with pytest.raises(api.FastLioError):
            api.PreprocessBatch(**args)


def test_busy_stream_reused_inputs_and_replays():
    """The frames and counts are written on the caller's stream behind a long kernel, then overwritten once the stream has passed
    the call; a captured graph replayed with new counts gives the new answers."""
    n_max, S = 6_000, 4
    pb, pp = handles(R.AVIA, 2, S, n_max)
    frames = [frame(R.AVIA, 90 + s, n_max) for s in range(S)]
    sl = Slots(frames, [n_max] * S, n_max, pb.layout.itemsize)
    src = [b.clone() for b in sl.bufs]
    table = sl.table()
    status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
    guard_outputs(pb)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for b in sl.bufs:
            b.zero_()
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(20):
            big = big @ big / 64.0                                 # keeps the stream busy
        for b, c in zip(sl.bufs, src):
            b.copy_(c)
        pb.run_device(table, S, n_max, status)
        for b in sl.bufs:
            b.fill_(0x5A)                                          # reused once the stream has passed the call
    s.synchronize()
    for b, c in zip(sl.bufs, src):
        b.copy_(c)
    check_slots(pb, pp, sl, n_max, status, range(S))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pb.run_device(table, S, n_max, status)
    rng = np.random.default_rng(5)
    for _ in range(3):
        for n in sl.ns:
            n.fill_(int(rng.integers(0, n_max + 1)))
        guard_outputs(pb)
        g.replay()
        torch.cuda.synchronize()
        check_slots(pb, pp, sl, n_max, status, range(S))


def test_fleet_graph_from_raw_avia_frames(problems):
    """16 robots' raw Avia frames: the preprocess batch, the scan batch and update_scans captured once and replayed over 6 steps
    with changing counts.  Per robot, x and P equal a chain of fl_preprocess_device -> fl_scan_t device forms ->
    fl_filter_update_device, byte for byte."""
    pr = problems("small")
    R_, n_max, leaf, steps = 16, 9_000, 0.5, 6
    rng = np.random.default_rng(41)
    frames = [[_avia_from_scan(synth.make_raw_scan(pr.scene, int(rng.integers(n_max // 3, n_max)), synth.true_state(pr.cfg.lidar, 2 * k + 25 * r),
                                                   seed=900 + 50 * r + k), 10 * r + k) for k in range(steps)] for r in range(R_)]
    cfg = CFG[R.AVIA]
    pb = api.PreprocessBatch(0, R.AVIA, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5, n_slots_max=R_, n_raw_max=n_max)
    pp = api.Preprocess(0, R.AVIA, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], 1, 0.5, n_raw_max=n_max)
    tg, tt = api.KdTree(0, 0.5), api.KdTree(0, 0.5)
    tg.Build(pr.map_pts); tt.Build(pr.map_pts)
    fg = api.Esekf(tg, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    fg.reserve_batch(n_max)
    ft = api.Esekf(tt, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    sb = api.ScanBatch(tg)
    sb.reserve(R_, n_max, 2)
    twin = api.Scan(tt)
    twin.reserve(n_max, 2)
    raw_d = torch.zeros((R_, n_max, 20), dtype=torch.uint8, device="cuda")
    n_d = torch.zeros((R_, 1), dtype=torch.int32, device="cuda")
    praws = api.preprocess_raws([(raw_d[r], n_d[r]) for r in range(R_)])
    xend = torch.stack([dev(synth.make_prior(synth.true_state(pr.cfg.lidar, 25 * r), seed=60 + r)[0]) for r in range(R_)])
    n_pose = torch.zeros(R_, dtype=torch.int32, device="cuda")          # the table points at it: kept alive with the graph
    sraws = pb.scan_raws(None, n_pose, xend)
    refs, m = sb.refs(1)
    refs = refs[:R_]
    x0 = host(xend)
    xg, Pg = dev(x0), dev(np.stack([pr.P_prior] * R_))
    xt, Pt = [dev(x0[r]) for r in range(R_)], [dev(pr.P_prior) for _ in range(R_)]
    pstatus, fstatus, ustatus = (torch.zeros((R_, 2), dtype=torch.int32, device="cuda") for _ in range(3))

    def fleet(x, P):
        pb.run_device(praws, R_, n_max, pstatus)
        sb.run_device(sraws, n_max, 2, leaf, status=fstatus)
        fg.update_scans_device(refs, x, P, m, pr.R, ustatus)

    def fill(k):
        for r in range(R_):
            a = frames[r][k]
            raw_d[r, :len(a)] = dev(a.view(np.uint8).reshape(len(a), -1))
            n_d[r].fill_(len(a))

    fill(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fleet(xg.clone(), Pg.clone())
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fleet(xg, Pg)
    xo = torch.zeros((n_max, 4), device="cuda")
    mo = torch.zeros(n_max, device="cuda")
    o2 = torch.zeros(2, dtype=torch.int32, device="cuda")
    for k in range(steps):
        fill(k)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        for r in range(R_):
            pp.process_device(raw_d[r], n_d[r], n_max, xo, mo, o2)
            twin.upload_device(xo, mo, o2[:1], n_max)
            twin.undistort_device(torch.zeros((2, 22), dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
                                  xend[r])
            twin.voxel_downsample_device(leaf)
            assert host(twin.update_device(ft, xt[r], Pt[r], pr.R))[0] == FL_OK
        x, P, ps, us = host(xg), host(Pg), host(pstatus), host(ustatus)
        for r in range(R_):
            assert ps[r][0] == FL_OK and us[r][0] == FL_OK, (k, r, ps[r], us[r])
            assert x[r].tobytes() == host(xt[r]).tobytes() and P[r].tobytes() == host(Pt[r]).tobytes(), (k, r)


def test_plain_c_program_node_count(tmp_path):
    """tests/facade/preprocess_batch_device.cu: the preprocess batch, the scan batch and update_scans captured into one graph by
    a plain CUDA program, with the same number of nodes at 1 and 64 slots."""
    exe = tmp_path / "preprocess_batch_device"
    nvcc = build._nvcc()
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-ccbin", "/usr/bin/g++", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "facade", "preprocess_batch_device.cu"), "-o", str(exe), "-L", os.path.dirname(build.LIB),
                    "-lfastlio_b200", "-Xlinker", f"-rpath={os.path.dirname(build.LIB)}"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "preprocess_batch_device ok" in out.stdout
