"""The scan front end of many scans in one call (fl_scan_batch_run_device): every slot's feats_undistort, feats_down_body,
feats_down_size and status equal, byte for byte, a single fl_scan_t's device forms on the same inputs; refused slots change no
other slot and are refused again by fl_filter_update_scans_device; the call follows the device forms' ordering and graph rules."""
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = -2, -4, -5
PAD_BITS = 0x7FFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def tree(pr):
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return t


class Slot:
    """One slot's device inputs, padded to n_max rows and n_pose_max poses: the same tensors feed the batch and the twin."""

    def __init__(self, xyzi, tms, poses, x_end, n_max, n_pose_max, n=None, n_pose=None):
        c = len(xyzi)
        self.xyzi = torch.zeros((max(n_max, 1), 4), dtype=torch.float32, device="cuda")
        self.tms = torch.zeros(max(n_max, 1), dtype=torch.float32, device="cuda")
        if c:
            self.xyzi[:c] = dev(xyzi); self.tms[:c] = dev(tms)
        self.poses = torch.zeros((max(n_pose_max, 1), 22), dtype=torch.float64, device="cuda")
        k = min(len(poses), n_pose_max)
        if k:
            self.poses[:k] = dev(poses[:k])
        self.x_end = dev(np.asarray(x_end, np.float64))
        self.n = torch.tensor([c if n is None else n], dtype=torch.int32, device="cuda")
        self.n_pose = torch.tensor([len(poses) if n_pose is None else n_pose], dtype=torch.int32, device="cuda")

    def entry(self):
        return (self.xyzi, self.tms, self.n, self.poses, self.n_pose, self.x_end)


def twin_chain(sc, slot, n_max, n_pose_max, leaf, undistort):
    """fl_scan_upload_device -> [undistort_device ->] voxel_downsample_device on a single front end: (cloud 0, cloud 1, status)."""
    sc.upload_device(slot.xyzi, slot.tms, slot.n, n_max)
    if undistort:
        sc.undistort_device(slot.poses[:n_pose_max], slot.n_pose, slot.x_end)
    cnt = sc.voxel_downsample_device(leaf)
    c = int(host(cnt)[0])
    return sc.download(0), sc.download(1), [0, c]


def check_batch(b, st, twins, slots=None):
    st = host(st) if isinstance(st, torch.Tensor) else st
    for s in (range(len(twins)) if slots is None else slots):
        u, d, sw = twins[s]
        assert list(st[s]) == sw, (s, st[s], sw)
        assert b.download(0, s).tobytes() == u.tobytes(), s
        assert b.download(1, s).tobytes() == d.tobytes(), s


class _Ints:
    """One int32 in device memory at `ptr`, for torch.as_tensor."""

    def __init__(self, ptr):
        self.__cuda_array_interface__ = {"shape": (1,), "typestr": "<i4", "data": (ptr, False), "version": 2}


def table_counts(refs):
    """The count each fl_scan_ref_t entry of a device table points at."""
    return [int(host(torch.as_tensor(_Ints(int(n)), device="cuda"))[0]) for _, n in host(refs)]


def awkward(tms, rng):
    """NaN payloads, +-0, +-inf and the padding pattern among a slot's offset times."""
    t = tms.copy()
    n = len(t)
    bits = np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, PAD_BITS, 0x7FFFFFFE, 0x80000000, 0x00000000, 0x7F800000,
                     0xFF800000], np.uint32)
    pick = rng.random(n) < 0.15
    t[pick] = rng.choice(bits, n)[pick].view(np.float32)
    return t


def raw_slots(pr, counts, n_max, rng, seed, undistort_variety=True, awkward_slots=()):
    """Raw scans of the given counts at distinct poses, 100 or 200 Hz IMUs, n_pose 0, 1, 2, all or clamped among them."""
    raws = []
    for s, c in enumerate(counts):
        x_end = synth.true_state(pr.cfg.lidar, 3 * s)
        hz = 100.0 if s % 2 else 200.0
        r = synth.make_raw_scan(pr.scene, max(int(c), 1), x_end, seed=seed + s, imu_hz=hz)
        xyzi, tms = r.xyzi[:c], r.offset_ms[:c]
        if s in awkward_slots:
            tms = awkward(tms, rng)
        k = [len(r.imu_pose), 0, 1, 2, len(r.imu_pose), 10 ** 6][s % 6] if undistort_variety else len(r.imu_pose)
        raws.append((xyzi, tms, r.imu_pose, r.x_end, k))
    return raws


@pytest.mark.parametrize("leaf", [0.5, 0.02])
@pytest.mark.parametrize("undistort", [1, 0])
@pytest.mark.parametrize("S", [1, 3, 64])
def test_each_slot_equals_its_single_chain(problems, S, undistort, leaf):
    """Counts 0, 1, 2, n_max and random ones in one call; n_pose 0, 1, 2, all and clamped; awkward offset times in chosen slots;
    at leaf 0.02 the large slots overflow PCL's grid into pass-through while the small ones do not."""
    pr = problems("small")
    t = tree(pr)
    rng = np.random.default_rng(S * 10 + undistort)
    n_max = 3_000
    counts = [int(v) for v in rng.integers(0, n_max + 1, S)]
    for i, c in enumerate((n_max, 0, 1, 2)):
        if i < S:
            counts[(5 * i) % S] = c
    raws = raw_slots(pr, counts, n_max, rng, seed=100 * S, awkward_slots={s for s in range(S) if s % 4 == 3} | ({0} if S == 1 else set()))
    n_pose_max = max(len(r[2]) for r in raws)
    slots = [Slot(x, tm, p, xe, n_max, n_pose_max, n_pose=k) for x, tm, p, xe, k in raws]
    b, sc = api.ScanBatch(t), api.Scan(t)
    b.reserve(S, n_max, n_pose_max)
    sc.reserve(n_max, n_pose_max)
    st = b.run_device(api.scan_raws([s.entry() for s in slots]), n_max, n_pose_max, leaf, undistort=bool(undistort))
    torch.cuda.synchronize()
    twins = [twin_chain(sc, s, n_max, n_pose_max, leaf, undistort) for s in slots]
    check_batch(b, st, twins)
    if leaf == 0.02 and S == 64:
        big = [s for s in range(S) if counts[s] > 1_000]
        assert any(twins[s][2][1] == counts[s] for s in big)            # pass-through: every point is its own cell
        assert twins[counts.index(2)][2][1] in (1, 2)


def test_aliased_inputs(problems):
    """Slots share one buffer, overlap rows of one packed buffer, or repeat a scan with other poses."""
    pr = problems("small")
    t = tree(pr)
    n_max, leaf = 4_000, 0.5
    rs = [synth.make_raw_scan(pr.scene, n_max, synth.true_state(pr.cfg.lidar, 3 * i), seed=40 + i) for i in range(3)]
    pk_x = dev(np.concatenate([r.xyzi for r in rs]))
    pk_t = dev(np.concatenate([r.offset_ms for r in rs]))
    n_pose_max = max(len(r.imu_pose) for r in rs)
    poses = [dev(np.pad(r.imu_pose, ((0, n_pose_max - len(r.imu_pose)), (0, 0)))) for r in rs]
    np_d = torch.tensor([len(r.imu_pose) for r in rs], dtype=torch.int32, device="cuda")
    xe = [dev(r.x_end) for r in rs]
    cnt = torch.tensor([n_max, 1_500, n_max, 700, n_max], dtype=torch.int32, device="cuda")
    offs = [0, 600, n_max, n_max - 300, 0]
    pose_of = [0, 0, 1, 1, 2]                                   # slot 4: scan 0 again with scan 2's poses and end state
    c = cnt.data_ptr()
    ents = [(pk_x.data_ptr() + 16 * o, pk_t.data_ptr() + 4 * o, c + 4 * s, poses[pose_of[s]], np_d.data_ptr() + 4 * pose_of[s], xe[pose_of[s]])
            for s, o in enumerate(offs)]
    b, sc = api.ScanBatch(t), api.Scan(t)
    b.reserve(5, n_max, n_pose_max)
    sc.reserve(n_max, n_pose_max)
    before = host(pk_x).copy()
    st = b.run_device(api.scan_raws(ents), n_max, n_pose_max, leaf)
    torch.cuda.synchronize()
    twins = []
    for s, o in enumerate(offs):
        k = int(host(cnt)[s])
        sl = Slot(host(pk_x)[o:o + k], host(pk_t)[o:o + k], host(poses[pose_of[s]]), host(xe[pose_of[s]]), n_max, n_pose_max,
                  n_pose=int(host(np_d)[pose_of[s]]))
        twins.append(twin_chain(sc, sl, n_max, n_pose_max, leaf, 1))
    check_batch(b, st, twins)
    assert host(pk_x).tobytes() == before.tobytes()


def test_refused_slots_and_the_update_refuses_them(problems):
    """Each refusal among valid slots: (status, 0), count -1 in both tables, every other slot unchanged; the same table then goes
    through fl_filter_update_scans_device, which refuses exactly those slots and updates the others as the single update does."""
    pr = problems("small")
    t = tree(pr)
    n_max, leaf = 3_000, 0.5
    rng = np.random.default_rng(7)
    raws = raw_slots(pr, [2_500] * 12, n_max, rng, seed=300, undistort_variety=False)
    n_pose_max = max(len(r[2]) for r in raws)
    slots = [Slot(x, tm, p, xe, n_max, n_pose_max) for x, tm, p, xe, _ in raws]
    ents = [list(s.entry()) for s in slots]
    neg = torch.tensor([-1, n_max + 1], dtype=torch.int32, device="cuda")
    ents[1][2] = neg.data_ptr()                                 # c < 0
    ents[2][2] = neg.data_ptr() + 4                             # c > n_max
    ents[3][0] = 0                                              # null xyzi
    ents[4][1] = slots[4].tms.data_ptr() + 2                    # misaligned offset times
    ents[5][2] = 0                                              # null n
    ents[6][2] = slots[6].n.data_ptr() + 2                      # misaligned n
    ents[7][5] = 0                                              # null x26_end
    ents[8][3] = 0                                              # null poses with n_pose >= 2
    ents[9][0] = slots[9].xyzi.data_ptr() + 8                   # misaligned xyzi
    refused = {1: FL_ERR_ARG, 2: FL_ERR_CAPACITY, 3: FL_ERR_ARG, 4: FL_ERR_ARG, 5: FL_ERR_ARG, 6: FL_ERR_ARG, 7: FL_ERR_ARG,
               8: FL_ERR_ARG, 9: FL_ERR_ARG}
    b, sc = api.ScanBatch(t), api.Scan(t)
    S = len(slots)
    b.reserve(S + 4, n_max, n_pose_max)
    sc.reserve(n_max, n_pose_max)
    st = host(b.run_device(api.scan_raws(ents), n_max, n_pose_max, leaf))
    for which in (0, 1):
        refs, m = b.refs(which)
        assert refs.shape == (S + 4, 2) and m == n_max
        cnt = table_counts(refs)
        assert [cnt[s] for s in refused] == [-1] * len(refused) and cnt[S:] == [-1] * 4
        assert all(cnt[s] == (2_500 if which == 0 else st[s][1]) for s in range(S) if s not in refused)
    for s, code in refused.items():
        assert list(st[s]) == [code, 0], (s, st[s])
        assert len(b.download(0, s)) == 0 and len(b.download(1, s)) == 0
    # null poses with fewer than two of them, and a null n_pose, are valid
    ok = [s for s in range(S) if s not in refused]
    twins = {s: twin_chain(sc, slots[s], n_max, n_pose_max, leaf, 1) for s in ok}
    check_batch(b, st, twins, ok)
    # the update over the same table: refused slots (FL_ERR_ARG, 0), the others as the single update on their rows
    refs, m = b.refs(1)
    f = api.Esekf(t, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    f.reserve_batch(m)
    X = np.stack([synth.make_prior(synth.true_state(pr.cfg.lidar, 3 * s), seed=10 + s)[0] for s in range(S)])
    P = np.stack([pr.P_prior] * S)
    x, p = dev(X), dev(P)
    ust = host(f.update_scans_device(refs[:S], x, p, m, pr.R))
    fs = api.Esekf(t, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    for s in range(S):
        if s in refused:
            assert list(ust[s]) == [FL_ERR_ARG, 0], s
            assert host(x)[s].tobytes() == X[s].tobytes()
        else:
            xs, Ps = dev(X[s]), dev(P[s])
            sst = host(fs.update_device(dev(twins[s][1]), xs, Ps, pr.R))
            assert list(ust[s]) == list(sst), s
            assert host(x)[s].tobytes() == host(xs).tobytes() and host(p)[s].tobytes() == host(Ps).tobytes(), s
    # slots the call did not cover have the count -1 in both tables: the update refuses them too
    xx, pp = dev(X[:1].repeat(4, 0)), dev(P[:1].repeat(4, 0))
    assert (host(f.update_scans_device(refs[S:S + 4], xx, pp, m, pr.R))[:, 0] == FL_ERR_ARG).all()


def test_fleet_graph(problems):
    """16 robots, each with its own IMU poses: one fl_scan_batch_run_device and one fl_filter_update_scans_device captured once and
    replayed over 10 raw scans per robot.  Each robot's chained x and P equal a chain of fl_filter_update_scan_device calls on a
    twin front end per robot."""
    pr = problems("small")
    R_, n_max, leaf, steps = 16, 9_000, 0.5, 10
    rng = np.random.default_rng(31)
    raw = [[synth.make_raw_scan(pr.scene, int(rng.integers(n_max // 3, n_max + 1)), synth.true_state(pr.cfg.lidar, 2 * k + 25 * r),
                                seed=700 + 50 * r + k, imu_hz=float(rng.choice([100.0, 200.0])))
            for k in range(steps)] for r in range(R_)]
    n_pose_max = max(len(s.imu_pose) for rs in raw for s in rs)
    tg, tt = tree(pr), tree(pr)
    fg = api.Esekf(tg, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    fg.reserve_batch(n_max)
    ft = api.Esekf(tt, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
    b = api.ScanBatch(tg)
    b.reserve(R_, n_max, n_pose_max)
    twins = [api.Scan(tt) for _ in range(R_)]
    for s in twins:
        s.reserve(n_max, n_pose_max)
    xyzi = torch.zeros((R_, n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros((R_, n_max), dtype=torch.float32, device="cuda")
    n_d = torch.zeros((R_, 1), dtype=torch.int32, device="cuda")
    poses = torch.zeros((R_, n_pose_max, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros((R_, 1), dtype=torch.int32, device="cuda")
    xend = torch.zeros((R_, 26), dtype=torch.float64, device="cuda")
    raws = api.scan_raws([(xyzi[r], tms[r], n_d[r], poses[r], np_d[r], xend[r]) for r in range(R_)])
    refs, m = b.refs(1)
    refs = refs[:R_]
    x0 = np.stack([synth.make_prior(synth.true_state(pr.cfg.lidar, 25 * r), seed=60 + r)[0] for r in range(R_)])
    P0 = np.stack([pr.P_prior] * R_)
    xg, Pg = dev(x0), dev(P0)
    fstatus = torch.zeros((R_, 2), dtype=torch.int32, device="cuda")
    ustatus = torch.zeros((R_, 2), dtype=torch.int32, device="cuda")
    xt, Pt = [dev(x0[r]) for r in range(R_)], [dev(P0[r]) for r in range(R_)]

    def fill(k):
        for r in range(R_):
            s = raw[r][k]
            n = len(s.xyzi)
            xyzi[r, :n] = dev(s.xyzi); tms[r, :n] = dev(s.offset_ms); n_d[r].fill_(n)
            poses[r, :len(s.imu_pose)] = dev(s.imu_pose); np_d[r].fill_(len(s.imu_pose)); xend[r].copy_(dev(s.x_end))

    def fleet(x, P):
        b.run_device(raws, n_max, n_pose_max, leaf, status=fstatus)
        fg.update_scans_device(refs, x, P, m, pr.R, ustatus)

    fill(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm-up outside capture, on throw-away states
        fleet(xg.clone(), Pg.clone())
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fleet(xg, Pg)
    for k in range(steps):
        fill(k)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        for r, s in enumerate(twins):
            sr = raw[r][k]
            s.upload_device(dev(sr.xyzi), dev(sr.offset_ms))
            s.undistort_device(dev(sr.imu_pose), None, dev(sr.x_end))
            s.voxel_downsample_device(leaf)
            assert host(s.update_device(ft, xt[r], Pt[r], pr.R))[0] == 0
        x, p, fs, us = host(xg), host(Pg), host(fstatus), host(ustatus)
        for r in range(R_):
            assert fs[r][0] == 0 and us[r][0] == 0, (k, r, fs[r], us[r])
            assert fs[r][1] == len(twins[r].download(1)), (k, r)
            assert x[r].tobytes() == host(xt[r]).tobytes() and p[r].tobytes() == host(Pt[r]).tobytes(), (k, r)


def test_config4_sized_scans(problems):
    """64 slots of 30k-60k raw points on config 4's scene, equal to the single chains."""
    pr = problems("avia_stream_24k")
    t = tree(pr)
    S, n_max, leaf = 64, 60_000, 0.5
    rng = np.random.default_rng(4)
    counts = [int(v) for v in rng.integers(30_000, n_max + 1, S)]
    counts[0] = n_max
    raws = raw_slots(pr, counts, n_max, rng, seed=2_000, undistort_variety=False, awkward_slots={5})
    n_pose_max = max(len(r[2]) for r in raws)
    slots = [Slot(x, tm, p, xe, n_max, n_pose_max) for x, tm, p, xe, _ in raws]
    b, sc = api.ScanBatch(t), api.Scan(t)
    b.reserve(S, n_max, n_pose_max)
    sc.reserve(n_max, n_pose_max)
    st = b.run_device(api.scan_raws([s.entry() for s in slots]), n_max, n_pose_max, leaf)
    torch.cuda.synchronize()
    twins = [twin_chain(sc, s, n_max, n_pose_max, leaf, 1) for s in slots]
    check_batch(b, st, twins)


def test_inputs_reusable_busy_stream_and_replays(problems):
    """The inputs are produced on a stream that is still busy when the call is enqueued and overwritten once the stream has passed
    the call; a captured call replays with new counts and pose counts written into device memory."""
    pr = problems("small")
    t = tree(pr)
    S, n_max, leaf = 6, 3_000, 0.5
    rng = np.random.default_rng(11)
    raws = raw_slots(pr, [3_000, 2_000, 1, 0, 2_999, 1_234], n_max, rng, seed=900)
    n_pose_max = max(len(r[2]) for r in raws)
    slots = [Slot(x, tm, p, xe, n_max, n_pose_max, n_pose=k) for x, tm, p, xe, k in raws]
    b, sc = api.ScanBatch(t), api.Scan(t)
    b.reserve(S, n_max, n_pose_max)
    sc.reserve(n_max, n_pose_max)
    twins = [twin_chain(sc, s, n_max, n_pose_max, leaf, 1) for s in slots]
    saved = [(s.xyzi.clone(), s.tms.clone(), s.n.clone()) for s in slots]
    table = api.scan_raws([s.entry() for s in slots])
    for s in slots:
        s.xyzi.zero_(); s.tms.zero_(); s.n.zero_()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                     # the call is enqueued long before its inputs exist
        for s, (a, tm, n) in zip(slots, saved):
            s.xyzi.copy_(a); s.tms.copy_(tm); s.n.copy_(n)
        st = b.run_device(table, n_max, n_pose_max, leaf)
        for s in slots:                                    # reusable once the stream has passed the call
            s.xyzi.fill_(7.0); s.tms.fill_(3.0); s.n.fill_(5)
    side.synchronize()
    check_batch(b, st, twins)
    for s, (a, tm, n) in zip(slots, saved):
        s.xyzi.copy_(a); s.tms.copy_(tm); s.n.copy_(n)
    status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        b.run_device(table, n_max, n_pose_max, leaf, status=status)
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.run_device(table, n_max, n_pose_max, leaf, status=status)
    for rep in range(3):
        counts = rng.integers(0, n_max + 1, S).astype(np.int32)
        for s, c in zip(slots, counts):
            s.n.fill_(int(c)); s.n_pose.fill_(int(rng.integers(0, n_pose_max + 2)))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        check_batch(b, status, [twin_chain(sc, s, n_max, n_pose_max, leaf, 1) for s in slots])


def test_host_refusals_enqueue_nothing(problems):
    pr = problems("small")
    L = api.load()
    t = tree(pr)
    b = api.ScanBatch(t)
    S, n_max, n_pose_max = 3, 1_000, 8
    r = synth.make_raw_scan(pr.scene, n_max, synth.true_state(pr.cfg.lidar, 0), seed=5)
    slots = [Slot(r.xyzi, r.offset_ms, r.imu_pose, r.x_end, n_max, n_pose_max) for _ in range(S)]
    table = api.scan_raws([s.entry() for s in slots])
    ss = torch.full((2 * S + 2,), -7, dtype=torch.int32, device="cuda")
    th = host(table).copy()
    sh = np.zeros(2 * S, np.int32)
    cs = torch.cuda.current_stream().cuda_stream
    t_, s_ = table.data_ptr(), ss.data_ptr()

    def call(tb, ns, nm, npm, und, leaf, st, stream=cs):
        return L.fl_scan_batch_run_device(b.h, tb, ns, nm, npm, und, leaf, st, stream)

    def untouched():
        return (host(ss) == -7).all()

    assert call(t_, S, n_max, n_pose_max, 1, 0.5, s_) == FL_ERR_STATE            # before reserve, also while capturing
    g = torch.cuda.CUDAGraph()
    rc = []
    marker = torch.zeros(1, device="cuda")
    with torch.cuda.graph(g):
        marker.add_(1.0)
        rc.append(call(t_, S, n_max, n_pose_max, 1, 0.5, s_, torch.cuda.current_stream().cuda_stream))
    g.replay()
    assert rc == [FL_ERR_STATE] and untouched() and host(marker)[0] == 1.0
    b.reserve(S, n_max, n_pose_max)
    assert L.fl_scan_batch_reserve(b.h, 1, 1, 3_000) == FL_ERR_CAPACITY           # poses beyond k_undistort's shared memory
    assert L.fl_scan_batch_reserve(b.h, 70_000, 1, 1) == FL_ERR_CAPACITY
    assert L.fl_scan_batch_reserve(b.h, 40_000, 60_000, 1) == FL_ERR_CAPACITY       # above INT_MAX rows
    refused = [
        (t_, -1, n_max, n_pose_max, 1, 0.5, s_, FL_ERR_ARG),
        (t_, S, -1, n_pose_max, 1, 0.5, s_, FL_ERR_ARG),
        (t_, S, n_max, -1, 1, 0.5, s_, FL_ERR_ARG),
        (t_, S, n_max, n_pose_max, 2, 0.5, s_, FL_ERR_ARG),
        (t_, S, n_max, n_pose_max, 1, 0.0, s_, FL_ERR_ARG),
        (t_, S, n_max, n_pose_max, 1, float("nan"), s_, FL_ERR_ARG),
        (th.ctypes.data, S, n_max, n_pose_max, 1, 0.5, s_, FL_ERR_ARG),       # host table
        (None, S, n_max, n_pose_max, 1, 0.5, s_, FL_ERR_ARG),
        (t_ + 4, S, n_max, n_pose_max, 1, 0.5, s_, FL_ERR_ARG),               # misaligned table
        (t_, S, n_max, n_pose_max, 1, 0.5, sh.ctypes.data, FL_ERR_ARG),       # host status
        (t_, S, n_max, n_pose_max, 1, 0.5, None, FL_ERR_ARG),
        (t_, S, n_max, n_pose_max, 1, 0.5, s_ + 2, FL_ERR_ARG),               # misaligned status
        (t_, S + 1, n_max, n_pose_max, 1, 0.5, s_, FL_ERR_CAPACITY),
        (t_, S, n_max + 1, n_pose_max, 1, 0.5, s_, FL_ERR_CAPACITY),
        (t_, S, n_max, n_pose_max + 1, 1, 0.5, s_, FL_ERR_CAPACITY),
    ]
    for i, (tb, ns, nm, npm, und, leaf, st, want) in enumerate(refused):
        assert call(tb, ns, nm, npm, und, leaf, st) == want, i
    rc = []
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        marker.add_(1.0)
        for tb, ns, nm, npm, und, leaf, st, want in refused[:4] + refused[-3:]:
            rc.append(call(tb, ns, nm, npm, und, leaf, st, torch.cuda.current_stream().cuda_stream) == want)
    g2.replay()
    assert all(rc) and untouched() and host(marker)[0] == 2.0
    # n_scans = 0: FL_OK, nothing written (null table and status allowed)
    assert call(None, 0, n_max, n_pose_max, 1, 0.5, None) == 0 and call(t_, 0, n_max, n_pose_max, 1, 0.5, s_) == 0
    assert untouched()
    # get_refs and download
    p = api.C.c_void_p()
    assert L.fl_scan_batch_get_refs(b.h, 2, api.C.byref(p), None) == FL_ERR_ARG
    assert L.fl_scan_batch_get_refs(b.h, 1, None, None) == FL_ERR_ARG
    assert L.fl_scan_batch_download(b.h, 1, S, np.zeros((1, 4), np.float32), 0) == FL_ERR_ARG
    b2 = api.ScanBatch(t)
    assert L.fl_scan_batch_get_refs(b2.h, 1, api.C.byref(p), None) == FL_ERR_STATE
    # the binding's checks
    with pytest.raises(TypeError):
        b.run_device(table.int(), n_max, n_pose_max, 0.5)
    with pytest.raises(ValueError):
        api.scan_raws([(slots[0].xyzi.double(), slots[0].tms, slots[0].n)])
    assert untouched()
    st = host(b.run_device(table, n_max, n_pose_max, 0.5))
    assert (st[:, 0] == 0).all() and (st[:, 1] > 0).all()


def test_plain_c_program_captures_the_batch_and_the_update(problems, tmp_path):
    """tests/facade/scan_batch_device.cu: one fl_scan_batch_run_device and one fl_filter_update_scans_device captured with
    cudaStreamBeginCapture and replayed per step, against per-robot single chains (the input file of update_scans_device.cu)."""
    pr = problems("small")
    exe = tmp_path / "scan_batch_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "facade", "scan_batch_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    robots, steps, n_raw = 6, 4, 6_000
    raw = [[synth.make_raw_scan(pr.scene, n_raw, synth.true_state(pr.cfg.lidar, 2 * k + 25 * r), seed=900 + 50 * r + k)
            for k in range(steps)] for r in range(robots)]
    n_pose = len(raw[0][0].imu_pose)
    assert all(len(s.imu_pose) == n_pose for rs in raw for s in rs)
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as fo:
        fo.write(struct.pack("6i", len(pr.map_pts), robots, steps, n_raw, n_pose, pr.cfg.max_iter))
        fo.write(struct.pack("d", pr.R))
        fo.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes())
        for r in range(robots):
            fo.write(np.ascontiguousarray(synth.make_prior(synth.true_state(pr.cfg.lidar, 25 * r), seed=60 + r)[0], np.float64).tobytes())
        fo.write(np.ascontiguousarray(pr.P_prior, np.float64).tobytes())
        for rs in raw:
            for s in rs:
                fo.write(np.ascontiguousarray(s.xyzi, np.float32).tobytes())
                fo.write(np.ascontiguousarray(s.offset_ms, np.float32).tobytes())
                fo.write(np.ascontiguousarray(s.imu_pose, np.float64).tobytes())
                fo.write(np.ascontiguousarray(s.x_end, np.float64).tobytes())
    run = subprocess.run([str(exe), str(fin)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "all equal" in run.stdout, run.stdout
