"""The deterministic map mode (fl_map_set_deterministic) on the device: with it on, k-NN answers, the down-sampling survivor,
the update and flatten's rows depend only on the map's point set, whatever history of Build / Add_Points / Delete_Point_Boxes
/ Add_Point_Boxes produced it, and k-NN equals the numpy rule (det_rules.py) byte for byte."""
import ctypes as C
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import det_rules
from fast_lio_b200 import api

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
KS = [1, 5, 8, 16, 32]
MAX_DISTS = [np.inf, 0.6, 1.0, 2.5]
EXTRA_BOX = np.array([[20.0, 20.0, 20.0, 30.0, 30.0, 30.0]], dtype=F)      # holds the extra points, nothing of the lattice
CHURN_BOX = np.array([[-1.0, -1.0, 0.0, 1.0, 1.0, 1.5]], dtype=F)


def lattice_map():
    """Points on a 0.5 m lattice (bit-equal distances everywhere), two intensities per site on a few sites."""
    rng = np.random.default_rng(17)
    g = np.arange(-6, 6.01, 0.5, dtype=F)
    X, Y, Z = np.meshgrid(g, g, g[:9], indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel(), rng.integers(0, 3, X.size).astype(F)], axis=1).astype(F)
    dup = pts[rng.choice(len(pts), 200, replace=False)].copy()
    dup[:, 3] += 5
    return np.concatenate([pts, dup])


def queries(pts):
    rng = np.random.default_rng(3)
    on = pts[rng.choice(len(pts), 600, replace=False)].copy()
    mid = on.copy(); mid[:, :3] += F(0.25)                                       # cell centres: 8 equidistant sites
    off = on.copy(); off[:, :3] += rng.integers(-2, 3, (len(on), 3)).astype(F) * F(0.125)
    far = np.c_[rng.uniform(-40, 40, (100, 3)), np.zeros(100)].astype(F)          # nothing within a cell: the BVH walk
    return np.concatenate([on, mid, off, far]).astype(F)


def histories(pts, cell_directory):
    """The same valid point set, reached five ways."""
    rng = np.random.default_rng(11)
    def tree():
        t = api.KdTree(0, 0.5, cell_directory=cell_directory)
        t.set_deterministic(True)
        return t
    out = []
    t = tree(); t.Build(pts[rng.permutation(len(pts))]); out.append(("permuted_a", t))
    t = tree(); t.Build(pts[rng.permutation(len(pts))]); out.append(("permuted_b", t))
    p = pts[rng.permutation(len(pts))]
    t = tree(); t.Build(p[: len(p) // 2]); t.Add_Points(p[len(p) // 2:], False); out.append(("build_then_add", t))
    extra = np.c_[rng.uniform(21, 29, (3000, 3)), np.zeros(3000)].astype(F)
    both = np.concatenate([pts, extra]); both = both[rng.permutation(len(both))]
    t = tree(); t.Build(both); t.Delete_Point_Boxes(EXTRA_BOX); out.append(("build_then_delete", t))
    t = tree(); t.Build(pts[rng.permutation(len(pts))])
    for _ in range(3):
        t.Delete_Point_Boxes(CHURN_BOX); t.Add_Point_Boxes(CHURN_BOX)
    out.append(("delete_revive_churn", t))
    for _, t in out:
        assert t.validnum() == len(pts)
    return out


@pytest.fixture(scope="module")
def lattice():
    pts = lattice_map()
    return pts, queries(pts)


@pytest.mark.parametrize("cell_directory", [True, False])
def test_knn_bytes_do_not_depend_on_layout(lattice, cell_directory):
    import torch
    pts, q = lattice
    trees = histories(pts, cell_directory)
    qd = torch.from_numpy(q).cuda()
    for k, md in itertools.product(KS, MAX_DISTS):
        rule = det_rules.nearest(q, pts, k, md)
        assert rule[3].all()                                                      # the order is fixed on every row here
        for name, t in trees:
            got = t.Nearest_Search_K(q, k, md)
            for a, b in zip(got, rule[:3]):
                assert a.tobytes() == b.tobytes(), (name, k, md)
            dev = t.nearest_search_device(qd, k, md)
            torch.cuda.synchronize()
            for a, b in zip(dev, got):
                assert a.cpu().numpy().tobytes() == b.tobytes(), (name, k, md)
    rule = det_rules.nearest(q, pts, 5)
    for name, t in trees:                                                        # fl_map_knn (k_knn_batch)
        got = t.Nearest_Search(q, 5)
        for a, b in zip(got, rule[:3]):
            assert a.tobytes() == b.tobytes(), name
    # the lattice does put ties at the k-th place, where the default mode's answer follows the slot order
    assert det_rules.reference_arbitrary(q, pts, 5).any()


def test_flatten_rows_are_sorted_and_layout_free(lattice):
    pts, _ = lattice
    trees = histories(pts, True)
    want = pts[det_rules.key_order(pts)]
    for name, t in trees:
        assert t.flatten().tobytes() == want.tobytes(), name
    off = api.KdTree(0, 0.5); off.Build(pts)                                   # mode off: the same set, slot order
    got = off.flatten()
    assert got[det_rules.key_order(got)].tobytes() == want.tobytes()


def test_voxel_survivor_is_the_smallest_key_in_every_insertion_order():
    ds = F(0.5)
    mid = np.array([0.25, 0.25, 0.25], dtype=F)                               # centre of voxel [0, 0.5)^3
    offs = np.array([[1, 1, 1], [-1, 1, 1], [1, -1, 1], [-1, -1, 1]], dtype=F) * F(0.125)
    planted = np.c_[mid + offs, np.arange(4, dtype=F) + 1].astype(F)
    rest = np.c_[np.random.default_rng(2).uniform(2, 6, (500, 3)), np.zeros(500)].astype(F)
    batch = np.array([[0.49, 0.49, 0.49, 9.0], [3.0, 3.0, 3.0, 1.0]], dtype=F)  # far from the planted voxel's centre; a new voxel
    survivor = planted[det_rules.voxel_survivor(planted, mid)]
    results = set()
    for perm in itertools.permutations(range(4)):
        t = api.KdTree(0, float(ds)); t.set_deterministic(True)
        t.Build(np.concatenate([planted[list(perm)], rest]))
        added = t.Add_Points(batch, True)
        flat = t.flatten()
        inside = flat[(flat[:, :3] >= 0).all(1) & (flat[:, :3] < 0.5).all(1)]
        assert inside.tobytes() == survivor[None].tobytes(), perm
        results.add((added, flat.tobytes()))
    assert len(results) == 1


def update_maps(pr, mode_on, hows=("build", "build_add", "build_delete"), dup=False):
    """The problem's map reached through different histories, so the slot layouts really differ: one Build; Build of a permuted
    half, then Add_Points of the rest; Build with extra far points, then Delete_Point_Boxes of them.  dup: every map point twice,
    the copy with another intensity -- bit-equal d2 at every place, so the default mode's Nearest_Points follow the slots."""
    pts = pr.map_pts
    if dup:
        cp = pts.copy(); cp[:, 3] += 100
        pts = np.concatenate([pts, cp])
    rng = np.random.default_rng(4)
    out = []
    for how in hows:
        t = api.KdTree(0, 0.5)
        t.set_deterministic(mode_on)
        if how == "build":
            t.Build(pts)
        elif how == "build_add":
            p = pts[rng.permutation(len(pts))]
            t.Build(p[: len(p) // 2]); t.Add_Points(p[len(p) // 2:], False)
        else:
            far = np.c_[rng.uniform(1e4, 1e4 + 50, (20000, 3)), np.zeros(20000)].astype(F)
            both = np.concatenate([pts, far]); both = both[rng.permutation(len(both))]
            t.Build(both)
            assert t.Delete_Point_Boxes(np.array([[9e3, 9e3, 9e3, 2e4, 2e4, 2e4]], dtype=F)) == len(far)
        assert t.validnum() == len(pts)
        out.append(t)
    return out


def filt(pr, t, extr=0):
    return api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr))


def run_host(pr, f):
    x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)       # (the third is a host time)
    n = len(pr.scan)
    near, cnt = f.nearest(n)
    return [np.asarray(x), np.asarray(P), near, cnt, f.selected(n), repr(f.pass_logs()).encode()]


def run_device(pr, f):
    import torch
    x = torch.from_numpy(np.array(pr.x_prior, dtype=np.float64)).cuda()
    P = torch.from_numpy(np.array(pr.P_prior, dtype=np.float64)).cuda()
    st = f.update_device(torch.from_numpy(pr.scan).cuda(), x, P, pr.R)
    torch.cuda.synchronize()
    n = len(pr.scan)
    near, cnt = f.nearest(n)
    return [x.cpu().numpy(), P.cpu().numpy(), st.cpu().numpy(), near, cnt, f.selected(n), repr(f.pass_logs()).encode()]


def run_batch(pr, f):
    import torch
    H = 3
    x = torch.from_numpy(np.tile(np.array(pr.x_prior, dtype=np.float64), (H, 1))).cuda()
    x[:, 0] += torch.arange(H, dtype=torch.float64, device=x.device) * 0.01
    P = torch.from_numpy(np.tile(np.array(pr.P_prior, dtype=np.float64), (H, 1, 1))).cuda()
    f.reserve_batch(len(pr.scan))
    st, lg = f.update_batch_device(torch.from_numpy(pr.scan).cuda(), x, P, pr.R, logs=True)
    torch.cuda.synchronize()
    return [x.cpu().numpy(), P.cpu().numpy(), st.cpu().numpy(), lg.cpu().numpy()]


def same(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        u = u if isinstance(u, bytes) else np.ascontiguousarray(u).tobytes()
        v = v if isinstance(v, bytes) else np.ascontiguousarray(v).tobytes()
        assert u == v, i


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
@pytest.mark.parametrize("extr", [0, 1])
def test_update_equal_across_map_histories(problems, name, extr):
    """x, P, pass logs, Nearest_Points and selected of the host, device and batch forms are equal on maps whose slot layouts
    differ (one Build, Build + Add_Points, Build + Delete_Point_Boxes), and from run to run."""
    pr = problems(name)
    fs = [filt(pr, t, extr) for t in update_maps(pr, True)]
    for run in (run_host, run_device, run_batch):
        ref = run(pr, fs[0])
        for f in fs[1:]:
            same(ref, run(pr, f))
        same(ref, run(pr, fs[0]))


def test_update_on_planted_ties_follows_the_mode(problems):
    """Every map point twice (the copy with another intensity): the k-th place is a bit-equal tie on every row.  In the default
    mode Nearest_Points follow the slot layout and differ between the histories; in the mode they are equal, and each neighbour
    pair comes (y, z, intensity)-ordered, the smaller intensity first."""
    pr = problems("small")
    near = {}
    for on in (False, True):
        near[on] = []
        for t in update_maps(pr, on, hows=("build", "build_add"), dup=True):
            near[on].append(run_host(pr, filt(pr, t)))
    same(near[True][0], near[True][1])
    assert near[False][0][2].tobytes() != near[False][1][2].tobytes()      # the default mode does depend on the layout
    nb = near[True][0][2].reshape(len(pr.scan), 5, 4)
    cnt = near[True][0][3]
    full = cnt == 5
    assert full.any()
    # pairs (0, 1) and (2, 3): the same coordinates, the original intensity before its copy (+100)
    for a, b in ((0, 1), (2, 3)):
        assert (nb[full, a, :3] == nb[full, b, :3]).all() and (nb[full, a, 3] < nb[full, b, 3]).all()


def test_map_incremental_equal_across_map_histories(problems):
    """After the device update, map_incremental's device form (Add_Points with down-sampling on the stream, k_downsample_keyed)
    leaves the same point set, returns the same counts and flattens to the same rows on every history; so does the host form."""
    import torch
    pr = problems("small")
    ts = update_maps(pr, True)
    outs, flats = [], []
    for i, t in enumerate(ts):
        f = filt(pr, t)
        run_device(pr, f)
        if i < 2:
            o = f.map_incremental_device(0.5, True)
            torch.cuda.synchronize()
            outs.append(o.cpu().numpy())
        else:
            outs.append(np.array(list(f.map_incremental(0.5, True)) + [0], dtype=np.int32)[:4])
        t.maintain()
        flats.append(t.flatten())
    assert outs[0].tobytes() == outs[1].tobytes()
    assert outs[0][:3].tolist() == outs[2][:3].tolist()
    assert outs[0][0] > 0
    for fl in flats[1:]:
        assert fl.tobytes() == flats[0].tobytes()
    assert flats[0].tobytes() == flats[0][det_rules.key_order(flats[0])].tobytes()


def world(pr, x):
    """Scan points in the world at state x (the update's first search point), for the numpy rule."""
    from scipy.spatial.transform import Rotation
    R_il = Rotation.from_quat(x[7:11]).as_matrix(); t_il = x[11:14]
    R_wi = Rotation.from_quat(x[3:7]).as_matrix(); t_wi = x[0:3]
    p = pr.scan[:, :3].astype(np.float64) @ R_il.T + t_il
    p = p @ R_wi.T + t_wi
    return np.c_[p, np.zeros(len(p))].astype(F)


def test_update_mode_on_equals_mode_off_without_boundary_ties(problems):
    """Where the numpy rule finds no bit-equal tie at the 5th place, the two modes give the same bytes.  The rule is checked on
    the scan points at the prior and at the final state; the passes in between search from states between them."""
    pr = problems("tiny")
    (on,) = update_maps(pr, True, hows=("build",))
    (off,) = update_maps(pr, False, hows=("build",))
    a, b = run_host(pr, filt(pr, on)), run_host(pr, filt(pr, off))
    for x in (np.asarray(pr.x_prior), a[0]):
        assert not det_rules.reference_arbitrary(world(pr, x), pr.map_pts, 5).any()
    same(a, b)


def test_rows_where_the_modes_differ_are_the_rows_where_the_reference_is_arbitrary(problems):
    """Mode on against mode off on the scan queries of tiny and small, and on a lattice: any row that differs is one the numpy
    rule names as arbitrary for the reference (a bit-equal d2 at the k-th place, or a 1e-10 tie sharing x)."""
    from refknn import world_queries
    cases = [(problems(n).map_pts, world_queries(problems(n))) for n in ("tiny", "small")]
    pts = lattice_map(); cases.append((pts, queries(pts)))
    seen_arbitrary = 0
    for mp, q in cases:
        on = api.KdTree(0, 0.5); on.set_deterministic(True); on.Build(mp)
        off = api.KdTree(0, 0.5); off.Build(mp)
        for k, md in itertools.product(KS, [np.inf, 1.0]):
            a, b = on.Nearest_Search_K(q, k, md), off.Nearest_Search_K(q, k, md)
            assert np.array_equal(a[2], b[2]) and a[1].tobytes() == b[1].tobytes()        # counts and d2: every row
            differ = ~np.all(a[0].reshape(len(q), -1) == b[0].reshape(len(q), -1), axis=1)
            arbitrary = det_rules.reference_arbitrary(q, mp, k, md)
            bad = np.flatnonzero(differ & ~arbitrary)
            assert not len(bad), (k, md, bad[:10])
            seen_arbitrary += int(arbitrary.sum())
    assert seen_arbitrary > 0


def test_cpp_facade_mode_from_the_environment(tmp_path):
    from fast_lio_b200 import build
    exe = tmp_path / "facade_deterministic"
    cmd = ["/usr/bin/g++", "-O1", "-std=c++14", "-Wall", "-Wno-unused",
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "facade"), "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(ROOT, "tests", "facade", "facade_deterministic.cpp"), "-o", str(exe), build.LIB, "-Wl,-rpath," + os.path.dirname(build.LIB)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    import struct
    pts = lattice_map()
    q = queries(pts)[:800]
    k = 8
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("3i", len(pts), len(q), k) + pts.tobytes() + q.tobytes())
    rule = det_rules.nearest(q, pts, k)
    for env_on in (True, False):
        fout = tmp_path / f"out{int(env_on)}.bin"
        env = dict(os.environ)
        env.pop("FASTLIO_B200_DETERMINISTIC", None)
        if env_on:
            env["FASTLIO_B200_DETERMINISTIC"] = "1"
        run = subprocess.run([str(exe), str(fin), str(fout)], capture_output=True, text=True, timeout=300, env=env)
        assert run.returncode == 0, run.stdout + run.stderr
        raw = open(fout, "rb").read()
        mode = struct.unpack_from("i", raw, 0)[0]
        assert mode == int(env_on)
        cnt = np.frombuffer(raw, np.int32, len(q), 4)
        at = 4 + 4 * len(q)
        assert np.array_equal(cnt, rule[2])
        got = np.frombuffer(raw, np.float32, 4 * int(cnt.sum()), at).reshape(-1, 4); at += 16 * int(cnt.sum())
        want = np.concatenate([rule[0][i, :cnt[i]] for i in range(len(q))])
        nf = struct.unpack_from("i", raw, at)[0]; at += 4
        flat = np.frombuffer(raw, np.float32, 4 * nf, at).reshape(-1, 4)
        assert nf == len(pts)
        if env_on:
            assert got.tobytes() == want.tobytes()
            assert flat.tobytes() == pts[det_rules.key_order(pts)].tobytes()
        else:
            assert flat[det_rules.key_order(flat)].tobytes() == pts[det_rules.key_order(pts)].tobytes()


def test_scan_stream_graph_equal_across_layouts(problems):
    """60 config-4 raw scans through the captured per-scan graph (segment, upload, de-skew, down-sample, update,
    map_incremental) on two maps whose first clouds have different slot layouts, the host-form chain on a third, and the first
    graph run again: in the mode the final x and P, every scan's status words and the flattened point sets are equal."""
    import det_stream
    pr, raws = det_stream.problem(60)
    xa, Pa, wa, _ = det_stream.run_graph(pr, raws, ta := det_stream.build(pr, "build", True))
    xb, Pb, wb, _ = det_stream.run_graph(pr, raws, tb := det_stream.build(pr, "build_add", True))
    xh, Ph, wh = det_stream.run_host(pr, raws, th := det_stream.build(pr, "build_add", True))
    xa2, Pa2, wa2, _ = det_stream.run_graph(pr, raws, ta2 := det_stream.build(pr, "build", True))
    fa = det_stream.flat_sorted(ta)
    assert fa.tobytes() == fa[det_rules.key_order(fa)].tobytes()
    for x, P, w, t in ((xb, Pb, wb, tb), (xa2, Pa2, wa2, ta2)):
        assert x.tobytes() == xa.tobytes() and P.tobytes() == Pa.tobytes()
        assert w.tobytes() == wa.tobytes()
        assert det_stream.flat_sorted(t).tobytes() == fa.tobytes()
    assert xh.tobytes() == xa.tobytes() and Ph.tobytes() == Pa.tobytes()
    assert np.array_equal(wh[:, 2], wa[:, 4])                     # Add_Points' return value, scan by scan
    assert det_stream.flat_sorted(th).tobytes() == fa.tobytes()
    assert (wa[:, 0] == 0).all()


def test_setter_getter_and_errors():
    t = api.KdTree(0, 0.5)
    assert t.deterministic is False
    t.set_deterministic(True)
    assert t.deterministic is True
    t.set_deterministic(False)
    assert t.deterministic is False
    L = api.load()
    on = C.c_int(7)
    FL_ERR_ARG = -2
    assert L.fl_map_set_deterministic(None, 1) == FL_ERR_ARG
    assert L.fl_map_get_deterministic(None, C.byref(on)) == FL_ERR_ARG
    assert L.fl_map_get_deterministic(t.h, None) == FL_ERR_ARG
    assert on.value == 7


def test_filter_legacy_chain_refuses_the_mode(problems):
    pr = problems("tiny")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts); t.set_deterministic(True)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, fused=0)
    with pytest.raises(api.FastLioError):
        f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)


PARITY_FILES = ["tests/test_gpu_knn.py", "tests/test_gpu_knn_k.py", "tests/test_gpu_range_search.py", "tests/test_gpu_map_mutation.py"]


def test_reference_parity_holds_in_the_mode():
    """The existing k-NN, range and map-mutation tests against the reference's goldens, every map in the mode: they assert
    neighbours only on rows the reference's own rules decide, so they hold unchanged."""
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    res = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "det_mode_plugin", "-x", *PARITY_FILES],
                         cwd=ROOT, env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
