"""Batched form of the update over many scans (fl_filter_update_scans_device): a scan and a prior per slot on one shared map, in
waves of k_update_scans launches planned at nq_max.  Every slot must equal, byte for byte, fl_filter_update_device on rows [0, c)
of its scan from its prior on a twin filter; refused slots leave their x, P and logs alone and change no other slot; the call
leaves the filter's own results (getters, map_incremental, later single updates) as they were."""
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


# ---- helpers (those of test_gpu_update_batch.py, restated here)
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def tree(pr):
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return t


def esekf(t, pr, extr=0, max_points=None, reserve=None, **kw):
    f = api.Esekf(t, max_points=max_points or max(len(pr.scan), 1), max_iter=pr.cfg.max_iter, limit=pr.limit,
                  extrinsic_est_en=bool(extr), **kw)
    if reserve:
        f.reserve_batch(reserve)
    return f


def same_logs(a, b):
    """Byte equality of pass logs; an entry of a pass without effective points (valid 0) has no HtH / Hth."""
    assert len(a) == len(b)
    for la, lb in zip(a, b):
        for k in la:
            if k in ("HtH", "Hth") and la["valid"] == 0:
                continue
            assert np.asarray(la[k]).tobytes() == np.asarray(lb[k]).tobytes(), k


def single(f, rows, x0, P0, R):
    """fl_filter_update_device from one prior on `rows`: (x, P, status, pass logs)."""
    x, P = dev(x0), dev(P0)
    st = f.update_device(dev(rows), x, P, R)
    return host(x), host(P), host(st), f.pass_logs()


def check_slots(want, got, slots=None):
    """want: {slot: single() result}; got: (x, P, status, raw logs) of one scans call."""
    x, P, st, lg = got
    for s in (want if slots is None else slots):
        xw, Pw, sw, lw = want[s]
        assert x[s].tobytes() == xw.tobytes() and P[s].tobytes() == Pw.tobytes(), s
        assert list(st[s]) == list(sw), s
        same_logs(api.decode_pass_logs(lg[s], int(st[s][1])), lw)
        assert not lg[s][int(st[s][1]):].any(), s            # entries from `passes` on are not written


def trajectory(pr, n, k, seed=0, n_rows=None):
    """k scans of n rows from distinct poses along the trajectory (0.1 m apart, every third step) with a prior each."""
    scans, xs, Ps = [], [], []
    for i in range(k):
        xt = synth.true_state(pr.cfg.lidar, 3 * i)
        scans.append(synth.make_scan(pr.scene, n_rows or n, xt, seed=500 + 37 * seed + i))
        x, P = synth.make_prior(xt, seed=900 + 37 * seed + i, pos_sigma=0.05 + 0.05 * (i % 3), rot_sigma_deg=0.5 + 0.5 * (i % 2))
        xs.append(x); Ps.append(P)
    return scans, np.stack(xs), np.stack(Ps)


class Slots:
    """Device rows and counts of a list of (scan rows, count) slots, and the table that references them."""

    def __init__(self, scans, which, counts):
        self.scans = scans
        self.bodies = [dev(s) for s in scans]
        self.which = list(which)
        self.cnt = torch.tensor(np.asarray(counts, np.int32), device="cuda")
        base = self.cnt.data_ptr()
        self.refs = api.scan_refs([(self.bodies[w], base + 4 * s) for s, w in enumerate(self.which)])

    def rows(self, s, counts=None):
        c = int((self.cnt.cpu().numpy() if counts is None else counts)[s])
        return self.scans[self.which[s]][:c]


def run(f, refs, X, P, nq_max, R):
    x, p = dev(X), dev(P)
    st, lg = f.update_scans_device(refs, x, p, nq_max, R, logs=True)
    return host(x), host(p), host(st), host(lg)


def mixed_counts(nq_max, S, rng):
    """0, 1, 255, 256, 257 and nq_max (those within nq_max) among random counts, so every wave mixes sizes."""
    fixed = [c for c in (0, 1, 255, 256, 257, nq_max) if c <= nq_max]
    out = [int(v) for v in rng.integers(0, nq_max + 1, S)]
    for i, c in enumerate(fixed):
        out[(7 * i + 3) % S] = c
    return out


# ---- equality with the single form
@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
def test_each_slot_equals_its_single_update(problems, name, extr):
    pr = problems(name)
    t = tree(pr)
    nq_max = len(pr.scan)
    fb, fs = esekf(t, pr, extr, reserve=nq_max), esekf(t, pr, extr)
    workers, slots, _ = fb.batch_plan(nq_max, 1)
    cap = 2 * torch.cuda.get_device_properties(0).multi_processor_count       # two k_update_scans blocks per SM
    assert workers == min(cap - 1, (nq_max + 255) // 256) and slots == cap // (workers + 1)
    S = 2 * slots + 1                                      # three waves, the last one short
    assert fb.batch_plan(nq_max, S)[2] == 3
    k = min(S, 12)
    scans, X0, P0 = trajectory(pr, nq_max, k, seed=extr)
    which = [s % k for s in range(S)]
    X, P = X0[which], P0[which]
    sl = Slots(scans, which, mixed_counts(nq_max, S, np.random.default_rng(extr)))
    want = {s: single(fs, sl.rows(s), X[s], P[s], pr.R) for s in range(S)}
    assert all(w[2][0] == 0 for w in want.values())
    check_slots(want, run(fb, sl.refs, X, P, nq_max, pr.R))


def test_more_tiles_than_co_resident_workers(problems):
    """nq_max = 70 000 rows on the 1 M map: more tiles than the co-resident workers, so a slot has cap - 1 workers (one slot per
    wave) and a 2 000-row slot shares that grid with a full one."""
    pr = problems("velodyne_30k_1m")
    t = tree(pr)
    nq_max = 70_000
    fb, fs = esekf(t, pr, max_points=nq_max, reserve=nq_max), esekf(t, pr, max_points=nq_max)
    cap = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    assert (nq_max + 255) // 256 > cap - 1
    assert fb.batch_plan(nq_max, 2) == (cap - 1, 1, 2)
    scans, X, P = trajectory(pr, nq_max, 2, seed=5)
    sl = Slots(scans, [0, 1], [2_000, nq_max])
    want = {s: single(fs, sl.rows(s), X[s], P[s], pr.R) for s in range(2)}
    check_slots(want, run(fb, sl.refs, X, P, nq_max, pr.R))


def test_aliased_scans(problems):
    """Slots that share one buffer, overlap rows of one packed buffer, and repeat a scan with another prior."""
    pr = problems("avia_2k_50k")
    t = tree(pr)
    nq_max = len(pr.scan)
    fb, fs = esekf(t, pr, reserve=nq_max), esekf(t, pr)
    scans, X0, P0 = trajectory(pr, nq_max, 3, seed=9)
    packed = np.concatenate(scans)                          # three scans back to back
    pk = dev(packed)
    cnt = torch.tensor([nq_max, 1_500, nq_max, 700, nq_max, nq_max], dtype=torch.int32, device="cuda")
    c = cnt.data_ptr()
    # (row offset into the packed buffer, count pointer): slot 1 starts inside scan 0, slot 3 straddles scans 0 and 1, slot 4 is
    # slot 0's scan again from another prior, slot 5 shares slot 0's count
    offs = [0, 600, nq_max, nq_max - 300, 0, 2 * nq_max]
    counts = [nq_max, 1_500, nq_max, 700, nq_max, nq_max]
    refs = api.scan_refs([(pk.data_ptr() + 16 * o, c + 4 * (s if s != 5 else 0)) for s, o in enumerate(offs)])
    X, P = X0[[0, 0, 1, 1, 2, 2]].copy(), P0[[0, 0, 1, 1, 2, 2]].copy()
    x4, P4 = synth.make_prior(synth.true_state(pr.cfg.lidar, 0), seed=4321, pos_sigma=0.2)
    X[4], P[4] = x4, P4
    want = {s: single(fs, packed[offs[s]:offs[s] + counts[s]], X[s], P[s], pr.R) for s in range(6)}
    check_slots(want, run(fb, refs, X, P, nq_max, pr.R))
    assert (host(pk) == packed).all()                       # read in place, never written


def test_refused_slots(problems):
    """Counts of -1 and nq_max + 1, a null body, a misaligned body and a null count pointer among valid slots: their statuses,
    their x, P and logs untouched, and every valid neighbour equal to its single update."""
    pr = problems("small")
    t = tree(pr)
    nq_max = len(pr.scan)
    fb, fs = esekf(t, pr, reserve=nq_max), esekf(t, pr)
    scans, X, P = trajectory(pr, nq_max, 8, seed=13)
    bodies = [dev(s) for s in scans]
    cnt = torch.tensor([nq_max, -1, 500, nq_max + 1, 300, 200, 100, 800], dtype=torch.int32, device="cuda")
    c = cnt.data_ptr()
    ents = [(bodies[0].data_ptr(), c), (bodies[1].data_ptr(), c + 4), (bodies[2].data_ptr(), c + 8), (bodies[3].data_ptr(), c + 12),
            (0, c + 16), (bodies[5].data_ptr() + 4, c + 20), (bodies[6].data_ptr(), 0), (bodies[7].data_ptr(), c + 28)]
    refs = api.scan_refs(ents)
    got = run(fb, refs, X, P, nq_max, pr.R)
    refused = {1: FL_ERR_ARG, 3: FL_ERR_CAPACITY, 4: FL_ERR_ARG, 5: FL_ERR_ARG, 6: FL_ERR_ARG}
    for s, code in refused.items():
        assert list(got[2][s]) == [code, 0], s
        assert got[0][s].tobytes() == X[s].tobytes() and got[1][s].tobytes() == P[s].tobytes(), s
        assert not got[3][s].any(), s
    counts = [nq_max, 0, 500, 0, 0, 0, 0, 800]
    want = {s: single(fs, scans[s][:counts[s]], X[s], P[s], pr.R) for s in (0, 2, 7)}
    check_slots(want, got)
    # a null body with a zero count is a valid empty scan
    cnt[4] = 0
    got = run(fb, refs, X, P, nq_max, pr.R)
    check_slots({4: single(fs, scans[4][:0], X[4], P[4], pr.R)}, got)


def getters(f, n):
    pts, cnt = f.nearest(n)
    pd, cd = f.nearest_device(n)
    return [pts, cnt, f.selected(n), host(pd), host(cd), host(f.selected_device(n)), *f.download_state()]


def test_filter_results_are_untouched(problems):
    """single update -> scans call -> every getter and map_incremental equals a twin filter with no call; a single update after a
    call equals one on a fresh filter."""
    pr = problems("small")
    n = len(pr.scan)
    scans, X, P = trajectory(pr, n, 5, seed=17)
    sl = Slots(scans, range(5), [n, 17, 600, 256, n])
    ta, tb = tree(pr), tree(pr)
    fa, fb = esekf(ta, pr, reserve=n), esekf(tb, pr)
    ra, rb = single(fa, pr.scan, pr.x_prior, pr.P_prior, pr.R), single(fb, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    run(fa, sl.refs, X, P, n, pr.R)
    for a, b in zip(getters(fa, n), getters(fb, n)):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    same_logs(fa.pass_logs(), fb.pass_logs())
    assert fa.map_incremental(0.5, True) == fb.map_incremental(0.5, True)
    assert ta.validnum() == tb.validnum() and sort_rows(ta.flatten()).tobytes() == sort_rows(tb.flatten()).tobytes()
    tc, td = tree(pr), tree(pr)
    fc, fd = esekf(tc, pr, reserve=n), esekf(td, pr)
    single(fc, pr.scan, pr.x_prior, pr.P_prior, pr.R); single(fd, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    run(fc, sl.refs, X, P, n, pr.R)
    assert host(fc.map_incremental_device(0.5, True)).tobytes() == host(fd.map_incremental_device(0.5, True)).tobytes()
    assert sort_rows(tc.flatten()).tobytes() == sort_rows(td.flatten()).tobytes()
    te, tf = tree(pr), tree(pr)
    fe, ff = esekf(te, pr, reserve=n), esekf(tf, pr)
    run(fe, sl.refs, X, P, n, pr.R)
    re_, rf = single(fe, pr.scan, X[2], P[2], pr.R), single(ff, pr.scan, X[2], P[2], pr.R)
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(re_[:3], rf[:3]))
    same_logs(re_[3], rf[3])
    assert fe.nearest(n)[0].tobytes() == ff.nearest(n)[0].tobytes() and fe.selected(n).tobytes() == ff.selected(n).tobytes()
    assert ra[0].tobytes() == rb[0].tobytes()


def test_deterministic_mode(problems):
    """With the map's deterministic mode on, every slot equals the single form in the mode."""
    pr = problems("avia_2k_50k")
    t = tree(pr)
    t.set_deterministic(True)
    nq_max = len(pr.scan)
    fb, fs = esekf(t, pr, reserve=nq_max), esekf(t, pr)
    _, slots, _ = fb.batch_plan(nq_max, 1)
    S = slots + 3
    scans, X0, P0 = trajectory(pr, nq_max, 6, seed=21)
    which = [s % 6 for s in range(S)]
    X, P = X0[which], P0[which]
    sl = Slots(scans, which, mixed_counts(nq_max, S, np.random.default_rng(21)))
    want = {s: single(fs, sl.rows(s), X[s], P[s], pr.R) for s in range(S)}
    check_slots(want, run(fb, sl.refs, X, P, nq_max, pr.R))


def test_graph_replays_with_new_counts_and_priors(problems):
    """One call captured over two waves, replayed three times with new counts and priors written into device memory in between:
    each replay equals the single updates."""
    pr = problems("avia_2k_50k")
    t = tree(pr)
    nq_max = len(pr.scan)
    fg, fs = esekf(t, pr, reserve=nq_max), esekf(t, pr)
    _, slots, _ = fg.batch_plan(nq_max, 1)
    S = slots + 5
    scans, X0, P0 = trajectory(pr, nq_max, 8, seed=23)
    which = [s % 8 for s in range(S)]
    rng = np.random.default_rng(23)
    sl = Slots(scans, which, mixed_counts(nq_max, S, rng))
    xs, Ps = dev(X0[which]), dev(P0[which])
    status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm-up outside capture
        fg.update_scans_device(sl.refs, xs, Ps, nq_max, pr.R, status)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fg.update_scans_device(sl.refs, xs, Ps, nq_max, pr.R, status)
    for rep in range(3):
        counts = np.asarray(mixed_counts(nq_max, S, rng), np.int32)
        X = np.stack([synth.make_prior(synth.true_state(pr.cfg.lidar, 3 * w), seed=1000 * rep + s)[0] for s, w in enumerate(which)])
        P = P0[which] * (1.0 + 0.25 * rep)
        sl.cnt.copy_(dev(counts)); xs.copy_(dev(X)); Ps.copy_(dev(P))
        g.replay()
        torch.cuda.synchronize()
        want = {s: single(fs, sl.rows(s, counts), X[s], P[s], pr.R) for s in range(S)}
        x, p, st = host(xs), host(Ps), host(status)
        for s in range(S):
            assert x[s].tobytes() == want[s][0].tobytes() and p[s].tobytes() == want[s][1].tobytes(), (rep, s)
            assert list(st[s]) == list(want[s][2]), (rep, s)


def test_fleet_graph(problems):
    """Four robots on one map: per robot fl_scan_upload_device -> undistort_device -> voxel_downsample_device on its own front end,
    then one fl_filter_update_scans_device over the four, captured once and replayed over 10 raw scans per robot.  Each robot's
    chained x and P equal a chain of fl_filter_update_scan_device calls on a twin filter."""
    pr = problems("small")
    R_, n_max, leaf, steps = 4, 9_000, 0.5, 10
    rng = np.random.default_rng(31)
    raw = [[synth.make_raw_scan(pr.scene, int(rng.integers(n_max // 3, n_max + 1)), synth.true_state(pr.cfg.lidar, 2 * k + 25 * r),
                                seed=700 + 50 * r + k, imu_hz=float(rng.choice([100.0, 200.0])))
            for k in range(steps)] for r in range(R_)]
    n_pose_max = max(len(s.imu_pose) for rs in raw for s in rs)
    tg, tt = tree(pr), tree(pr)
    fg, ft = esekf(tg, pr, max_points=n_max, reserve=n_max), esekf(tt, pr, max_points=n_max)
    fronts, twins = [api.Scan(tg) for _ in range(R_)], [api.Scan(tt) for _ in range(R_)]
    for s in fronts + twins:
        s.reserve(n_max, n_pose_max)
    refs_l = []
    for s in fronts:
        b, n, m = s.ref()
        assert m == n_max and b % 16 == 0
        refs_l.append((b, n))
    refs = api.scan_refs(refs_l)
    xyzi = torch.zeros((R_, n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros((R_, n_max), dtype=torch.float32, device="cuda")
    n_d = torch.zeros((R_, 1), dtype=torch.int32, device="cuda")
    poses = torch.zeros((R_, n_pose_max, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros((R_, 1), dtype=torch.int32, device="cuda")
    xend = torch.zeros((R_, 26), dtype=torch.float64, device="cuda")
    x0 = np.stack([synth.make_prior(synth.true_state(pr.cfg.lidar, 25 * r), seed=60 + r)[0] for r in range(R_)])
    P0 = np.stack([pr.P_prior] * R_)
    xg, Pg = dev(x0), dev(P0)
    status = torch.zeros((R_, 2), dtype=torch.int32, device="cuda")
    xt, Pt = [dev(x0[r]) for r in range(R_)], [dev(P0[r]) for r in range(R_)]

    def fill(k):
        for r in range(R_):
            s = raw[r][k]
            n = len(s.xyzi)
            xyzi[r, :n] = dev(s.xyzi); tms[r, :n] = dev(s.offset_ms); n_d[r].fill_(n)
            poses[r, :len(s.imu_pose)] = dev(s.imu_pose); np_d[r].fill_(len(s.imu_pose)); xend[r].copy_(dev(s.x_end))

    def fleet(x, P):
        for r, s in enumerate(fronts):
            s.upload_device(xyzi[r], tms[r], n_d[r], n_max)
            s.undistort_device(poses[r], np_d[r], xend[r])
            s.voxel_downsample_device(leaf)
        fg.update_scans_device(refs, x, P, n_max, pr.R, status)

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
        for r, s in enumerate(twins):                      # the twin chain: one robot at a time, single updates
            sr = raw[r][k]
            s.upload_device(dev(sr.xyzi), dev(sr.offset_ms))
            s.undistort_device(dev(sr.imu_pose), None, dev(sr.x_end))
            s.voxel_downsample_device(leaf)
            st = s.update_device(ft, xt[r], Pt[r], pr.R)
            assert host(st)[0] == 0
        x, p, st = host(xg), host(Pg), host(status)
        for r in range(R_):
            assert st[r][0] == 0, (k, r, st[r])
            assert x[r].tobytes() == host(xt[r]).tobytes() and p[r].tobytes() == host(Pt[r]).tobytes(), (k, r)


def test_busy_caller_stream_and_a_query_in_flight(problems):
    """The counts, x and P are produced on a stream that is still busy when the call is made, while a device query of the map runs
    on another stream."""
    pr = problems("small")
    t = tree(pr)
    n = len(pr.scan)
    fb, fs = esekf(t, pr, reserve=n), esekf(t, pr)
    scans, X, P = trajectory(pr, n, 6, seed=41)
    counts = [n, 900, 0, 257, 256, n]
    sl = Slots(scans, range(6), [0] * 6)
    want = {s: single(fs, scans[s][:counts[s]], X[s], P[s], pr.R) for s in range(6)}
    q = dev(pr.scan)
    pts0, d0, c0 = t.nearest_search_device(q, 5)
    ref_q = [host(v) for v in (pts0, d0, c0)]
    xb, Pb, cb = dev(X), dev(P), dev(np.asarray(counts, np.int32))
    other, side = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(other):
        torch.cuda._sleep(100_000_000)
        res = t.nearest_search_device(q, 5)
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                     # ~0.1 s: the call below is enqueued long before its inputs exist
        x, p = xb * 1.0, Pb * 1.0
        sl.cnt.copy_(cb)
        st, lg = fb.update_scans_device(sl.refs, x, p, n, pr.R, logs=True)
    side.synchronize(); other.synchronize()
    check_slots(want, (host(x), host(p), host(st), host(lg)))
    assert all(host(a).tobytes() == b.tobytes() for a, b in zip(res, ref_q))


def test_refusals(problems):
    pr = problems("small")
    L = api.load()
    t = tree(pr)
    n = len(pr.scan)
    f = esekf(t, pr, max_points=n)
    S = 3
    sd = dev(pr.scan)
    cnt = torch.full((S,), 100, dtype=torch.int32, device="cuda")
    refs = api.scan_refs([(sd, cnt.data_ptr() + 4 * s) for s in range(S)])
    xs = torch.full((S * 26 + 2,), -7.0, dtype=torch.float64, device="cuda")
    Ps = torch.full((S * 529 + 2,), -7.0, dtype=torch.float64, device="cuda")
    ss = torch.full((2 * S + 2,), -7, dtype=torch.int32, device="cuda")
    ls = torch.full((S * (pr.cfg.max_iter + 1) * api.C.sizeof(api.PassLog) + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    rh = refs.cpu().numpy().copy()
    xh, Ph, sh, lh = np.zeros(S * 26), np.zeros(S * 529), np.zeros(2 * S, np.int32), np.zeros(ls.numel(), np.uint8)
    s = torch.cuda.current_stream().cuda_stream
    r_, x_, P_, s_, l_ = refs.data_ptr(), xs.data_ptr(), Ps.data_ptr(), ss.data_ptr(), ls.data_ptr()

    def call(ff, tb, ns, nq, x, P, st, lg, stream=s):
        return L.fl_filter_update_scans_device(ff.h, tb, ns, nq, x, P, pr.R, st, lg, stream)

    def untouched():
        torch.cuda.synchronize()
        return (host(xs) == -7.0).all() and (host(Ps) == -7.0).all() and (host(ss) == -7).all() and (host(ls) == 0x5A).all()

    # before reserve_batch, also on a capturing stream: refused, nothing captured
    assert call(f, r_, S, n, x_, P_, s_, l_) == FL_ERR_STATE
    g = torch.cuda.CUDAGraph()
    rc = []
    marker = torch.zeros(1, device="cuda")
    with torch.cuda.graph(g):
        marker.add_(1.0)                                   # the graph's only node
        rc.append(call(f, r_, S, n, x_, P_, s_, l_, torch.cuda.current_stream().cuda_stream))
        rc.append(call(f, r_, -1, n, x_, P_, s_, l_, torch.cuda.current_stream().cuda_stream))
    assert rc == [FL_ERR_STATE, FL_ERR_ARG]
    g.replay()
    assert untouched() and host(marker)[0] == 1.0
    assert L.fl_filter_reserve_batch(f.h, n - 100) == 0
    m = n - 100
    refused = [
        (f, r_, S, n, x_, P_, s_, l_, FL_ERR_CAPACITY),                   # nq_max above the reserved one
        (f, rh.ctypes.data, S, m, x_, P_, s_, l_, FL_ERR_ARG),            # host table
        (f, r_, S, m, xh.ctypes.data, P_, s_, l_, FL_ERR_ARG),
        (f, r_, S, m, x_, Ph.ctypes.data, s_, l_, FL_ERR_ARG),
        (f, r_, S, m, x_, P_, sh.ctypes.data, l_, FL_ERR_ARG),
        (f, r_, S, m, x_, P_, s_, lh.ctypes.data, FL_ERR_ARG),
        (f, None, S, m, x_, P_, s_, l_, FL_ERR_ARG),
        (f, r_, S, m, None, P_, s_, l_, FL_ERR_ARG),
        (f, r_, S, m, x_, None, s_, l_, FL_ERR_ARG),
        (f, r_, S, m, x_, P_, None, l_, FL_ERR_ARG),
        (f, r_, -1, m, x_, P_, s_, l_, FL_ERR_ARG),
        (f, r_, S, -1, x_, P_, s_, l_, FL_ERR_ARG),
        (f, r_ + 4, S, m, x_, P_, s_, l_, FL_ERR_ARG),                    # misaligned table
        (f, r_, S, m, x_ + 4, P_, s_, l_, FL_ERR_ARG),                    # misaligned x
        (f, r_, S, m, x_, P_ + 4, s_, l_, FL_ERR_ARG),                    # misaligned P
        (f, r_, S, m, x_, P_, s_ + 2, l_, FL_ERR_ARG),                    # misaligned status
        (f, r_, S, m, x_, P_, s_, l_ + 4, FL_ERR_ARG),                    # misaligned logs
    ]
    sharded = esekf(t, pr, reserve=n); sharded.set_shard(0, n)
    solver0 = esekf(t, pr, solver=0, reserve=n)
    split = esekf(t, pr, fused=0, reserve=n)
    for ff in (sharded, solver0, split):
        refused.append((ff, r_, S, m, x_, P_, s_, l_, FL_ERR_STATE))
    for i, (ff, tb, ns, nq, x, P, st, lg, want) in enumerate(refused):
        assert call(ff, tb, ns, nq, x, P, st, lg) == want, i
    assert untouched()
    # n_scans = 0: FL_OK, nothing written (null outputs allowed)
    assert call(f, None, 0, m, None, None, None, None) == 0
    assert call(f, r_, 0, m, x_, P_, s_, l_) == 0
    assert untouched()
    # fl_scan_get_ref before fl_scan_reserve, and a null out
    sc = api.Scan(t)
    ref = api.ScanRef()
    assert L.fl_scan_get_ref(sc.h, api.C.byref(ref), None) == FL_ERR_STATE
    sc.reserve(64, 2)
    assert L.fl_scan_get_ref(sc.h, None, None) == FL_ERR_ARG
    assert L.fl_scan_get_ref(sc.h, api.C.byref(ref), None) == 0 and ref.body_xyzi and ref.n
    # the binding's checks
    with pytest.raises(ValueError):
        f.update_scans_device(refs[:1], xs[:26].view(1, 26), Ps[:1058].view(2, 23, 23), m)
    with pytest.raises(TypeError):
        f.update_scans_device(refs[:1].int(), xs[:26].view(1, 26), Ps[:529].view(1, 23, 23), m)
    assert untouched()
    # accepted: counts within nq_max
    x1, P1 = dev(pr.x_prior[None]), dev(pr.P_prior[None])
    st = f.update_scans_device(refs[:1], x1, P1, m, pr.R)
    assert host(st)[0][0] == 0 and host(st)[0][1] >= 2


def test_plain_c_program_runs_a_fleet_graph(problems, tmp_path):
    pr = problems("small")
    exe = tmp_path / "update_scans_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "facade", "update_scans_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    robots, steps = 4, 5
    raw = [[synth.make_raw_scan(pr.scene, 6_000, synth.true_state(pr.cfg.lidar, 2 * k + 25 * r), seed=800 + 50 * r + k)
            for k in range(steps)] for r in range(robots)]
    n_pose = len(raw[0][0].imu_pose)
    assert all(len(s.imu_pose) == n_pose and len(s.xyzi) == 6_000 for rs in raw for s in rs)
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as fo:
        fo.write(struct.pack("6i", len(pr.map_pts), robots, steps, 6_000, n_pose, pr.cfg.max_iter))
        fo.write(struct.pack("d", pr.R))
        fo.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes())
        for r in range(robots):
            x0, _ = synth.make_prior(synth.true_state(pr.cfg.lidar, 25 * r), seed=60 + r)
            fo.write(np.ascontiguousarray(x0, np.float64).tobytes())
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
