"""Batched form of the update (fl_filter_update_batch_device): one scan from many priors in waves of k_update_batch launches.
Every hypothesis must equal, byte for byte, fl_filter_update_device from its prior on a twin filter, and the batch must leave
the filter's own results (getters, map_incremental, later single updates) as they were."""
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
LARGE = {   # the large-correction priors of test_gpu_update_large_corrections.py: (make_prior options, extrinsic_est_en)
    "rot": (dict(rot_err_deg=(10.0, 10.0, 0.0)), 0),
    "grav": (dict(rot_err_deg=(9.0, 9.0, 0.0), grav_var=1e-2, grav_rot_corr=0.9, grav_deg=2.0), 0),
    "extr": (dict(rot_err_deg=(10.0, 10.0, 0.0), offr_deg=3.0), 1),
}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def tree(pr):
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return t


def esekf(t, pr, extr=0, max_points=None, reserve=True, **kw):
    f = api.Esekf(t, max_points=max_points or max(len(pr.scan), 1), max_iter=pr.cfg.max_iter, limit=pr.limit,
                  extrinsic_est_en=bool(extr), **kw)
    if reserve:
        f.reserve_batch(len(pr.scan))
    return f


def priors(pr, H, seed=0):
    """H priors around the truth: distinct make_prior seeds, with up to 0.3 m and 2 degrees of spread."""
    xs, Ps = [], []
    for h in range(H):
        x, P = synth.make_prior(pr.x_true, seed=1000 * seed + h, pos_sigma=0.3 * (h % 4) / 3 + 0.02, rot_sigma_deg=0.5 + 1.5 * (h % 3) / 2)
        xs.append(x); Ps.append(P)
    return np.stack(xs), np.stack(Ps)


def single(f, scan, x0, P0, R):
    """fl_filter_update_device from one prior: (x, P, status, pass logs)."""
    x, P = dev(x0), dev(P0)
    st = f.update_device(dev(scan), x, P, R)
    return host(x), host(P), host(st), f.pass_logs()


def same_logs(a, b):
    """Byte equality of pass logs; an entry of a pass without effective points (valid 0) has no HtH / Hth."""
    assert len(a) == len(b)
    for la, lb in zip(a, b):
        for k in la:
            if k in ("HtH", "Hth") and la["valid"] == 0:
                continue
            assert np.asarray(la[k]).tobytes() == np.asarray(lb[k]).tobytes(), k


def batch(f, scan, X, P, R, stream_scan=None):
    x, p = dev(X), dev(P)
    st, lg = f.update_batch_device(stream_scan if stream_scan is not None else dev(scan), x, p, R, logs=True)
    return host(x), host(p), host(st), host(lg)


def check_against(want, got, hyps=None):
    """want: list of single() results; got: (x, P, status, raw logs) of a batch over the same priors."""
    x, P, st, lg = got
    for h in (range(len(want)) if hyps is None else hyps):
        xw, Pw, sw, lw = want[h]
        assert x[h].tobytes() == xw.tobytes() and P[h].tobytes() == Pw.tobytes(), h
        assert list(st[h]) == list(sw), h
        same_logs(api.decode_pass_logs(lg[h], int(st[h][1])), lw)
        assert not lg[h][int(st[h][1]):].any(), h            # entries from `passes` on are not written


@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
def test_each_hypothesis_equals_its_single_update(problems, name, extr):
    pr = problems(name)
    t = tree(pr)
    fb, fs = esekf(t, pr, extr), esekf(t, pr, extr, reserve=False)
    n = len(pr.scan)
    workers, slots, _ = fb.batch_plan(n, 1)
    cap = 2 * torch.cuda.get_device_properties(0).multi_processor_count       # two k_update_batch blocks per SM
    assert workers == min(cap - 1, (n + 255) // 256) and slots == cap // (workers + 1)
    H = 2 * slots + 1                                      # three waves, the last one short
    assert fb.batch_plan(n, H)[2] == 3
    X, P = priors(pr, H, seed=extr)
    want = [single(fs, pr.scan, X[h], P[h], pr.R) for h in range(H)]
    assert all(w[2][0] == 0 and w[2][1] >= 2 for w in want)
    check_against(want, batch(fb, pr.scan, X, P, pr.R))


@pytest.mark.parametrize("extr", [0, 1])
def test_mixed_hypotheses_in_one_wave(problems, extr):
    """The default prior, the large-correction priors and a prior 5 000 m away (no effective point on any pass) share a wave."""
    pr = problems("small")
    t = tree(pr)
    fb, fs = esekf(t, pr, extr), esekf(t, pr, extr, reserve=False)
    xs, Ps = [pr.x_prior], [pr.P_prior]
    for opts, e in LARGE.values():
        if e == extr:
            x, P = synth.make_prior(pr.x_true, seed=pr.cfg.seed + 2, **opts)
            xs.append(x); Ps.append(P)
    far = pr.x_prior.copy()
    far[:3] += 5000.0
    xs.append(far); Ps.append(pr.P_prior)
    X, P = np.stack(xs), np.stack(Ps)
    assert fb.batch_plan(len(pr.scan), len(X))[2] == 1
    want = [single(fs, pr.scan, X[h], P[h], pr.R) for h in range(len(X))]
    got = batch(fb, pr.scan, X, P, pr.R)
    check_against(want, got)
    passes = [int(s[1]) for s in got[2]]
    assert len(set(passes)) > 1, passes
    assert list(got[2][-1]) == [0, pr.cfg.max_iter + 1] and got[0][-1].tobytes() == far.tobytes()


def test_wave_boundaries(problems):
    pr = problems("avia_2k_50k")
    t = tree(pr)
    fb, fs = esekf(t, pr), esekf(t, pr, reserve=False)
    n = len(pr.scan)
    _, slots, _ = fb.batch_plan(n, 1)
    X, P = priors(pr, 2 * slots + 3, seed=7)
    want = [single(fs, pr.scan, X[h], P[h], pr.R) for h in range(len(X))]
    for H in (1, slots, slots + 1, 2 * slots + 3):
        assert fb.batch_plan(n, H)[2] == (H + slots - 1) // slots
        check_against(want[:H], batch(fb, pr.scan, X[:H], P[:H], pr.R))
    # H = 0: FL_OK, nothing written
    assert fb.batch_plan(n, 0)[2] == 0
    xs = torch.full((4, 26), -7.0, dtype=torch.float64, device="cuda")
    Ps = torch.full((4, 23, 23), -7.0, dtype=torch.float64, device="cuda")
    ss = torch.full((4, 2), -7, dtype=torch.int32, device="cuda")
    ls = torch.full((4, pr.cfg.max_iter + 1, api.C.sizeof(api.PassLog)), 0x5A, dtype=torch.uint8, device="cuda")
    L = api.load()
    assert L.fl_filter_update_batch_device(fb.h, dev(pr.scan).data_ptr(), n, 0, xs.data_ptr(), Ps.data_ptr(), pr.R, ss.data_ptr(),
                                           ls.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    st = fb.update_batch_device(dev(pr.scan), xs[:0], Ps[:0], pr.R)
    assert tuple(st.shape) == (0, 2)
    torch.cuda.synchronize()
    assert (host(xs) == -7.0).all() and (host(Ps) == -7.0).all() and (host(ss) == -7).all() and (host(ls) == 0x5A).all()


def getters(f, n):
    pts, cnt = f.nearest(n)
    pd, cd = f.nearest_device(n)
    return [pts, cnt, f.selected(n), host(pd), host(cd), host(f.selected_device(n)), *f.download_state()]


def test_filter_results_are_untouched(problems):
    """single update -> batch -> every getter and map_incremental equals a twin filter with no batch; a single update after a
    batch equals one on a fresh filter."""
    pr = problems("small")
    n = len(pr.scan)
    ta, tb = tree(pr), tree(pr)
    fa, fb = esekf(ta, pr), esekf(tb, pr, reserve=False)
    X, P = priors(pr, 9, seed=3)
    ra, rb = single(fa, pr.scan, pr.x_prior, pr.P_prior, pr.R), single(fb, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    batch(fa, pr.scan[::-1].copy(), X, P, pr.R)            # another scan, other priors
    for a, b in zip(getters(fa, n), getters(fb, n)):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    same_logs(fa.pass_logs(), fb.pass_logs())
    assert fa.map_incremental(0.5, True) == fb.map_incremental(0.5, True)
    assert ta.validnum() == tb.validnum() and sort_rows(ta.flatten()).tobytes() == sort_rows(tb.flatten()).tobytes()
    # the device form of map_incremental after a batch
    tc, td = tree(pr), tree(pr)
    fc, fd = esekf(tc, pr), esekf(td, pr, reserve=False)
    single(fc, pr.scan, pr.x_prior, pr.P_prior, pr.R); single(fd, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    batch(fc, pr.scan, X, P, pr.R)
    assert host(fc.map_incremental_device(0.5, True)).tobytes() == host(fd.map_incremental_device(0.5, True)).tobytes()
    assert sort_rows(tc.flatten()).tobytes() == sort_rows(td.flatten()).tobytes()
    # a single update after a batch
    te, tf = tree(pr), tree(pr)
    fe, ff = esekf(te, pr), esekf(tf, pr, reserve=False)
    batch(fe, pr.scan, X, P, pr.R)
    x0 = X[4]
    re_, rf = single(fe, pr.scan, x0, P[4], pr.R), single(ff, pr.scan, x0, P[4], pr.R)
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(re_[:3], rf[:3]))
    same_logs(re_[3], rf[3])
    assert fe.nearest(n)[0].tobytes() == ff.nearest(n)[0].tobytes() and fe.selected(n).tobytes() == ff.selected(n).tobytes()
    assert ra[0].tobytes() == rb[0].tobytes()


def test_graph_capture_and_replay(problems):
    """One batch call captured, replayed with three sets of priors copied into the captured buffers, single updates on the same
    filter in between: each replay equals the uncaptured call on a twin filter, each single update its twin's."""
    pr = problems("avia_2k_50k")
    t = tree(pr)
    fg, fr, fs = esekf(t, pr), esekf(t, pr), esekf(t, pr, reserve=False)
    _, slots, _ = fg.batch_plan(len(pr.scan), 1)
    H = slots + 5                                          # two waves in the graph
    sd = dev(pr.scan)
    X0, P0 = priors(pr, H, seed=11)
    xs, Ps = dev(X0), dev(P0)
    status = torch.zeros((H, 2), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm-up outside capture
        fg.update_batch_device(sd, xs, Ps, pr.R, status)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fg.update_batch_device(sd, xs, Ps, pr.R, status)
    for rep in range(3):
        X, P = priors(pr, H, seed=20 + rep)
        xs.copy_(dev(X)); Ps.copy_(dev(P))
        g.replay()
        torch.cuda.synchronize()
        want = batch(fr, pr.scan, X, P, pr.R)
        assert host(xs).tobytes() == want[0].tobytes() and host(Ps).tobytes() == want[1].tobytes(), rep
        assert host(status).tobytes() == want[2].tobytes(), rep
        x1 = X[rep] + 0.0
        a, b = single(fg, pr.scan, x1, P[rep], pr.R), single(fs, pr.scan, x1, P[rep], pr.R)
        assert all(np.asarray(u).tobytes() == np.asarray(v).tobytes() for u, v in zip(a[:3], b[:3])), rep
        same_logs(a[3], b[3])


def test_busy_caller_stream_and_freed_scan(problems):
    """x, P and the scan are produced on a stream that is still busy when the call is made, and the scan is freed and its memory
    reused right after the call."""
    pr = problems("small")
    t = tree(pr)
    fb, fs = esekf(t, pr), esekf(t, pr, reserve=False)
    X, P = priors(pr, 60, seed=5)
    want = [single(fs, pr.scan, X[h], P[h], pr.R) for h in range(len(X))]
    xb, Pb, sb = dev(X), dev(P), dev(pr.scan)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                     # ~0.1 s: the call below is enqueued long before its inputs exist
        x, p, s = xb * 1.0, Pb * 1.0, sb * 1.0
        st, lg = fb.update_batch_device(s, x, p, pr.R, logs=True)
        del s
        junk = torch.full((len(pr.scan), 4), -3.0e5, dtype=torch.float32, device="cuda")
    side.synchronize()
    check_against(want, (host(x), host(p), host(st), host(lg)))
    del junk


def test_refusals(problems):
    pr = problems("small")
    L = api.load()
    t = tree(pr)
    n = len(pr.scan)
    f = esekf(t, pr, max_points=n, reserve=False)
    H = 3
    sd = dev(pr.scan)
    xs = torch.full((H * 26 + 2,), -7.0, dtype=torch.float64, device="cuda")
    Ps = torch.full((H * 529 + 2,), -7.0, dtype=torch.float64, device="cuda")
    ss = torch.full((2 * H + 2,), -7, dtype=torch.int32, device="cuda")
    ls = torch.full((H * (pr.cfg.max_iter + 1) * api.C.sizeof(api.PassLog) + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    xh, Ph, sh, lh = np.zeros(H * 26), np.zeros(H * 529), np.zeros(2 * H, np.int32), np.zeros(ls.numel(), np.uint8)
    s = torch.cuda.current_stream().cuda_stream
    x_, P_, s_, l_ = xs.data_ptr(), Ps.data_ptr(), ss.data_ptr(), ls.data_ptr()

    def call(ff, body, nq, nh, x, P, st, lg, stream=s):
        return L.fl_filter_update_batch_device(ff.h, body, nq, nh, x, P, pr.R, st, lg, stream)

    def untouched():
        torch.cuda.synchronize()
        return (host(xs) == -7.0).all() and (host(Ps) == -7.0).all() and (host(ss) == -7).all() and (host(ls) == 0x5A).all()

    # before reserve_batch, also on a capturing stream: refused, nothing captured
    assert call(f, sd.data_ptr(), n, H, x_, P_, s_, l_) == FL_ERR_STATE
    g = torch.cuda.CUDAGraph()
    rc = []
    marker = torch.zeros(1, device="cuda")
    with torch.cuda.graph(g):
        marker.add_(1.0)                                   # the graph's only node
        rc.append(call(f, sd.data_ptr(), n, H, x_, P_, s_, l_, torch.cuda.current_stream().cuda_stream))
    assert rc == [FL_ERR_STATE]
    g.replay()
    assert untouched() and host(marker)[0] == 1.0
    assert L.fl_filter_reserve_batch(f.h, -1) == FL_ERR_ARG
    assert L.fl_filter_reserve_batch(f.h, n + 1) == FL_ERR_CAPACITY        # above the filter's capacity (max_points = n)
    assert L.fl_filter_reserve_batch(f.h, n - 100) == 0
    refused = [
        (f, sd.data_ptr(), n, H, x_, P_, s_, l_, FL_ERR_CAPACITY),             # above the reserved nq_max
        (f, pr.scan.ctypes.data, n - 100, H, x_, P_, s_, l_, FL_ERR_ARG),      # host scan
        (f, sd.data_ptr(), n - 100, H, xh.ctypes.data, P_, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, x_, Ph.ctypes.data, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, x_, P_, sh.ctypes.data, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, x_, P_, s_, lh.ctypes.data, FL_ERR_ARG),
        (f, None, n - 100, H, x_, P_, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, None, P_, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, x_, None, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, H, x_, P_, None, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), -1, H, x_, P_, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr(), n - 100, -1, x_, P_, s_, l_, FL_ERR_ARG),
        (f, sd.data_ptr() + 4, n - 100, H, x_, P_, s_, l_, FL_ERR_ARG),       # misaligned scan
        (f, sd.data_ptr(), n - 100, H, x_ + 4, P_, s_, l_, FL_ERR_ARG),       # misaligned x
        (f, sd.data_ptr(), n - 100, H, x_, P_ + 4, s_, l_, FL_ERR_ARG),       # misaligned P
        (f, sd.data_ptr(), n - 100, H, x_, P_, s_ + 2, l_, FL_ERR_ARG),       # misaligned status
        (f, sd.data_ptr(), n - 100, H, x_, P_, s_, l_ + 4, FL_ERR_ARG),       # misaligned logs
    ]
    sharded = esekf(t, pr); sharded.set_shard(0, n)
    solver0 = esekf(t, pr, solver=0)
    split = esekf(t, pr, fused=0)
    for ff in (sharded, solver0, split):
        refused.append((ff, sd.data_ptr(), n, H, x_, P_, s_, l_, FL_ERR_STATE))
    for i, (ff, body, nq, nh, x, P, st, lg, want) in enumerate(refused):
        assert call(ff, body, nq, nh, x, P, st, lg) == want, i
    assert untouched()
    out3 = np.zeros(3, np.int32)
    assert L.fl_filter_batch_plan(f.h, -1, 1, out3) == FL_ERR_ARG and L.fl_filter_batch_plan(f.h, 1, -1, out3) == FL_ERR_ARG
    # the binding's checks
    with pytest.raises(ValueError):
        f.update_batch_device(sd[:50], xs[:26].view(1, 26), Ps[:1058].view(2, 23, 23))       # one x, two P
    with pytest.raises(TypeError):
        f.update_batch_device(sd[:50], xs[:26].view(1, 26).float(), Ps[:529].view(1, 23, 23))
    assert untouched()
    # accepted: nq within the reservation
    x1, P1 = dev(pr.x_prior[None]), dev(pr.P_prior[None])
    st = f.update_batch_device(sd[:n - 100], x1, P1, pr.R)
    assert host(st)[0][0] == 0 and host(st)[0][1] >= 2


def test_plain_c_program_captures_the_batch(problems, tmp_path):
    pr = problems("avia_2k_50k")
    exe = tmp_path / "update_batch_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "facade", "update_batch_device.cu"), "-o", str(exe), build.LIB,
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
