"""The config-4 scan stream (avia_stream_24k raw scans) through the whole per-scan chain -- lasermap_fov_segment, upload, de-skew,
voxel down-sampling, the iterated update, map_incremental -- on maps whose first clouds were built with different slot layouts,
for the deterministic map mode's stream test (test_gpu_deterministic.py) and benchmark (scripts/deterministic_bench.py).

Device chains run the six calls captured once into one CUDA graph and replayed scan after scan (recaptured after maintenance
moves the map); the host chain runs the host-buffer forms of the same calls."""
import numpy as np

from fast_lio_b200 import api, synth

N_MIN, N_MAX, LEAF, CUBE_LEN, DET_RANGE = 30_000, 60_000, 0.5, 6.0, 1.0


def pos_lid(x):
    """state.pos + state.rot * state.offset_T_L_I (laserMapping.cpp:890) in the order of Eigen's _transformVector."""
    q, v = x[3:6], x[11:14]
    cross = lambda a, b: np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])   # noqa: E731
    uv = cross(q, v)
    uv = uv + uv
    return x[0:3] + ((v + uv * x[6]) + cross(q, uv))


def problem(scans, seed=7):
    pr = synth.make_problem("avia_stream_24k")
    rng = np.random.default_rng(seed)
    raws = [synth.make_raw_scan(pr.scene, int(rng.integers(N_MIN, N_MAX + 1)), synth.true_state(pr.cfg.lidar, s),
                                seed=3000 + s, imu_hz=float(rng.choice([100.0, 200.0, 400.0]))) for s in range(scans)]
    return pr, raws


def build(pr, how, det):
    """The problem's map, the same point set reached two ways: 'build' (one Build) or 'build_add' (Build of a permuted first
    half, Add_Points of the rest without down-sampling: another slot layout)."""
    t = api.KdTree(0, 0.5)
    t.set_deterministic(det)
    if how == "build":
        t.Build(pr.map_pts)
    else:
        p = pr.map_pts[np.random.default_rng(23).permutation(len(pr.map_pts))]
        t.Build(p[: len(p) // 2])
        t.Add_Points(p[len(p) // 2:], False)
    return t


def run_graph(pr, raws, tree, timed=False):
    """The captured per-scan graph over `raws`.  Returns (x, P, per-scan status words [update status, passes, out4, seg3],
    per-scan graph times in seconds or None)."""
    import torch
    n_pose_max = max(len(r.imu_pose) for r in raws)
    f = api.Esekf(tree, max_points=N_MAX, max_iter=pr.cfg.max_iter)
    s = api.Scan(tree)
    s.reserve(N_MAX, n_pose_max)
    cube = api.LocalMap(CUBE_LEN, DET_RANGE)
    st = torch.cuda.Stream()
    dev = lambda **kw: {k: torch.zeros(v[0], dtype=v[1], device="cuda") for k, v in kw.items()}   # noqa: E731
    b = dev(xyzi=((N_MAX, 4), torch.float32), t=((N_MAX,), torch.float32), n=((1,), torch.int32),
            poses=((n_pose_max, 22), torch.float64), n_pose=((1,), torch.int32), x_end=((26,), torch.float64),
            status=((2,), torch.int32), out4=((4,), torch.int32), seg3=((3,), torch.int32), n_out=((1,), torch.int32))
    b["x"] = torch.from_numpy(pr.x_prior.copy()).cuda()
    b["P"] = torch.from_numpy(pr.P_prior.copy()).cuda()
    eye = torch.eye(23, dtype=torch.float64, device="cuda") * 1e-4

    def chain():
        cube.segment_device(tree, b["x"], b["seg3"], None, b["n"])
        s.upload_device(b["xyzi"], b["t"], b["n"], N_MAX)
        s.undistort_device(b["poses"], b["n_pose"], b["x_end"])
        s.voxel_downsample_device(LEAF, b["n_out"])
        s.update_device(f, b["x"], b["P"], pr.R, b["status"])
        f.map_incremental_device(0.5, True, b["out4"])

    def capture():
        torch.cuda.synchronize()
        tree.maintain()                             # the map's headroom for the captured inserts is reserved outside capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            chain()
        return g

    words, times, graph = [], [], None
    for i, r in enumerate(raws):
        with torch.cuda.stream(st):
            b["xyzi"][:len(r.xyzi)] = torch.from_numpy(r.xyzi).cuda(); b["t"][:len(r.xyzi)] = torch.from_numpy(r.offset_ms).cuda()
            b["n"].fill_(len(r.xyzi)); b["poses"][:len(r.imu_pose)] = torch.from_numpy(r.imu_pose).cuda()
            b["n_pose"].fill_(len(r.imu_pose)); b["x_end"].copy_(torch.from_numpy(r.x_end).cuda()); b["P"].add_(eye)
            if graph is None:                       # the first scan runs uncaptured, then the chain is captured
                chain()
            else:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                graph.replay()
                e1.record(st)
                times.append((e0, e1))
            words.append(torch.cat([b["status"], b["out4"], b["seg3"]]).clone())
        st.synchronize()
        if graph is None:
            graph = capture()
        w = words[-1].cpu().numpy()
        if w[5] != 0 or w[8] != 0:                  # maintenance fell due (map_incremental or the segment): settle, recapture
            if tree.maintain():
                graph = capture()
    torch.cuda.synchronize()
    t = [e0.elapsed_time(e1) * 1e-3 for e0, e1 in times] if timed else None
    out = (b["x"].cpu().numpy(), b["P"].cpu().numpy(), torch.stack(words).cpu().numpy(), t)
    f.close(); s.close()
    return out


def run_host(pr, raws, tree):
    """The host-buffer forms of the same chain.  Returns (x, P, per-scan (added, voxel-downsampled count))."""
    f = api.Esekf(tree, max_points=N_MAX, max_iter=pr.cfg.max_iter)
    s = api.Scan(tree)
    cube = api.LocalMap(CUBE_LEN, DET_RANGE)
    x, P = pr.x_prior.copy(), pr.P_prior.copy()
    words = []
    for r in raws:
        P = P + np.eye(23) * 1e-4
        cube.segment(pos_lid(x), tree)
        s.upload(r.xyzi, r.offset_ms)
        s.undistort(r.imu_pose, r.x_end)
        n_ds = s.voxel_downsample(LEAF)
        x, P, _ = s.update(f, x, P, pr.R)
        words.append((*f.map_incremental(0.5, True), n_ds))
    f.close(); s.close()
    return x, P, np.asarray(words)


def flat_sorted(tree):
    """The map's valid points as fl_map_flatten returns them (sorted by (x, y, z, intensity) in the deterministic mode)."""
    tree.maintain()
    return tree.flatten()
