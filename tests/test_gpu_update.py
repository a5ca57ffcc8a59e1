"""Parity of the fused device update against the CPU oracle (north-star tolerance 1e-4 m / 1e-4 rad)."""
import numpy as np
import pytest

from fast_lio_b200 import api, synth
from oracle import bind
from refcalls import RefTree, digest

pytestmark = pytest.mark.gpu

POS_TOL = 1e-4      # metres   (BASELINE.json north_star)
ROT_TOL = 1e-4      # radians


def rot_err(qa, qb):
    """Angle of qa^-1 * qb (x,y,z,w)."""
    qa = qa / np.linalg.norm(qa); qb = qb / np.linalg.norm(qb)
    d = abs(float(np.dot(qa, qb)))
    return 2.0 * np.arccos(min(1.0, d))


def run_both(pr, solver=0, extr=0):
    o = RefTree(f"update_{pr.cfg.name}_e{extr}", pr.map_pts).update_iterated(pr.scan, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, extr)
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr), solver=solver)
    x, P, st = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    return o, (x, P, st, f)


def check_state(o, x, P):
    assert np.abs(x[0:3] - o.x[0:3]).max() <= POS_TOL
    assert rot_err(x[3:7], o.x[3:7]) <= ROT_TOL
    assert rot_err(x[7:11], o.x[7:11]) <= ROT_TOL
    assert np.abs(x[11:] - o.x[11:]).max() <= POS_TOL
    scale = np.sqrt(np.outer(np.diag(o.P), np.diag(o.P)))
    assert (np.abs(P - o.P) / scale).max() < 1e-3


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k"])
@pytest.mark.parametrize("solver", [0, 1])
def test_update_matches_oracle(problems, name, solver):
    pr = problems(name)
    o, (x, P, st, f) = run_both(pr, solver)
    logs = f.pass_logs()
    assert len(logs) == len(o.passes)
    for lg, op in zip(logs, o.passes):
        assert lg["searched"] == op["searched"]
        assert lg["effct"] == op["effct"]
        assert lg["converged"] == op["converged"]
        assert abs(lg["res_sum"] - op["res_sum"]) <= 1e-6 * max(1.0, abs(op["res_sum"]))
        assert np.allclose(lg["HtH"], op["HtH"], rtol=1e-9, atol=1e-9 * np.abs(op["HtH"]).max())
        assert np.allclose(lg["Hth"], op["Hth"], rtol=1e-9, atol=1e-9 * np.abs(op["Hth"]).max())
        assert np.abs(lg["x_after"] - op["x_after"]).max() < 1e-6
    check_state(o, x, P)
    npts = len(pr.scan)
    near, cnt = f.nearest(npts)
    assert digest(cnt) == o.nearest_cnt_digest
    assert digest(near) == o.nearest_digest
    assert digest(f.selected(npts)) == o.selected_digest
    assert st > 0.0


@pytest.mark.parametrize("name", ["velodyne_30k_1m", "ouster64_131k_5m"])
def test_headline_size_parity(problems, name):
    """North-star claim, at the sizes it is made on (BASELINE configs 2 and 3): the whole update against the CPU oracle
    (the reference's own ikd-Tree + the restated h_share_model / esekf update) on identical input -- per-pass search
    decisions, effective-point counts and convergence flags identical, point_selected_surf and Nearest_Points identical,
    state within 1e-4 m / 1e-4 rad, covariance within 1e-3 relative."""
    pr = problems(name)
    o, (x, P, st, f) = run_both(pr, solver=1)
    logs = f.pass_logs()
    assert len(logs) == len(o.passes)
    for lg, op in zip(logs, o.passes):
        assert (lg["searched"], lg["effct"], lg["converged"], lg["valid"]) == (op["searched"], op["effct"], op["converged"], op["valid"])
        assert abs(lg["res_sum"] - op["res_sum"]) <= 1e-6 * max(1.0, abs(op["res_sum"]))
        assert np.allclose(lg["HtH"], op["HtH"], rtol=1e-9, atol=1e-9 * np.abs(op["HtH"]).max())
        assert np.allclose(lg["Hth"], op["Hth"], rtol=1e-9, atol=1e-9 * np.abs(op["Hth"]).max())
        assert np.abs(lg["x_after"] - op["x_after"]).max() < 1e-6
    check_state(o, x, P)
    n = len(pr.scan)
    near, cnt = f.nearest(n)
    assert digest(cnt) == o.nearest_cnt_digest
    assert digest(near) == o.nearest_digest
    assert digest(f.selected(n)) == o.selected_digest


def test_update_extrinsic_est(problems):
    pr = problems("small")
    o, (x, P, st, f) = run_both(pr, 0, extr=1)
    check_state(o, x, P)
    assert np.allclose(f.pass_logs()[0]["HtH"], o.passes[0]["HtH"], rtol=1e-9, atol=1e-6)


def test_shard_equals_subscan(problems):
    """Multi-GPU building block on one GPU: processing the shard [lo, hi) of a bound scan gives the
    same normal equations as binding only scan[lo:hi] (what each rank contributes to the all-reduce)."""
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    n = len(pr.scan)
    total = None
    for rank in range(3):
        lo, hi = api.shard_range(n, 3, rank)
        fa = api.Esekf(t, max_points=n, max_iter=1)
        fa.upload_scan(pr.scan); fa.set_shard(lo, hi); fa.upload_state(pr.x_prior, pr.P_prior, pr.R); fa.run()
        fa.download_state()
        fb = api.Esekf(t, max_points=n, max_iter=1)
        fb.upload_scan(pr.scan[lo:hi]); fb.upload_state(pr.x_prior, pr.P_prior, pr.R); fb.run()
        fb.download_state()
        la, lb = fa.pass_logs()[0], fb.pass_logs()[0]
        assert la["effct"] == lb["effct"]
        assert np.array_equal(la["HtH"], lb["HtH"]) and np.array_equal(la["Hth"], lb["Hth"])
        total = la["HtH"] if total is None else total + la["HtH"]
    full = api.Esekf(t, max_points=n, max_iter=1)
    full.upload_scan(pr.scan); full.upload_state(pr.x_prior, pr.P_prior, pr.R); full.run(); full.download_state()
    assert np.allclose(total, full.pass_logs()[0]["HtH"], rtol=1e-12, atol=1e-9)


def test_sharded_update_completes_the_neighbours_of_the_whole_scan(problems):
    """Multi-GPU building block on one GPU (ADVICE r1): a rank searches only its shard during the update, but map_incremental
    and get_nearest need Nearest_Points of the WHOLE scan, from the state of the last searching pass -- the rank recomputes the
    others' on its own map replica.  They must be exactly what an unsharded search at that state returns."""
    pr = problems("small")
    n = len(pr.scan)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    lo, hi = api.shard_range(n, 3, 1)
    f = api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter)
    f.upload_scan(pr.scan); f.set_shard(lo, hi); f.upload_state(pr.x_prior, pr.P_prior, pr.R); f.run()
    x, P, npass = f.download_state()
    logs = f.pass_logs()
    last_search = max(i for i, l in enumerate(logs) if l["searched"])
    x_search = pr.x_prior if last_search == 0 else logs[last_search - 1]["x_after"]
    near, cnt = f.nearest(n)
    q = np.zeros((n, 4), dtype=np.float32)
    tmp = np.zeros(3, dtype=np.float32)
    for i in range(n):
        bind.lib().oracle_transform_point(np.ascontiguousarray(x_search), np.ascontiguousarray(pr.scan[i, :3]), tmp)
        q[i, :3] = tmp
    gp, gd, gc = t.Nearest_Search(q, 5)
    assert np.array_equal(cnt, gc)
    assert np.array_equal(near, gp)
    with pytest.raises(api.FastLioError):
        f.selected(n)                              # point_selected_surf of the other shards lives on their ranks
    # and the device-side map_incremental classifies the whole scan
    to_add, no_ds, added = f.map_incremental(0.5, True)
    assert to_add + no_ds > 0


def test_small_m_branch(problems):
    """Fewer than 23 effective points -> the K = P H^T (H P H^T / R + I)^-1 / R branch (esekfom.hpp:1715-1744)."""
    pr = problems("tiny")
    scan = pr.scan[:14].copy()
    o = RefTree("update_small_m", pr.map_pts).update_iterated(scan, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, 0)
    assert 0 < o.passes[0]["effct"] < 23
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=64, max_iter=pr.cfg.max_iter)
    x, P, _ = f.update_iterated_dyn_share_modified(scan, pr.x_prior, pr.P_prior, pr.R)
    assert len(f.pass_logs()) == len(o.passes)
    check_state(o, x, P)


def test_no_effective_points_leaves_state_untouched(problems):
    """effct_feat_num < 1 -> valid = false, every pass is skipped (laserMapping.cpp:708-713)."""
    pr = problems("tiny")
    far = pr.scan[:50].copy()
    far[:, :3] += 5000.0                       # nothing within sqrt(5) m of any 5 map points
    o = RefTree("update_no_effective_points", pr.map_pts).update_iterated(far, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, 0)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=64, max_iter=pr.cfg.max_iter)
    x, P, _ = f.update_iterated_dyn_share_modified(far, pr.x_prior, pr.P_prior, pr.R)
    assert np.array_equal(x, pr.x_prior) and np.array_equal(o.x, pr.x_prior)
    assert np.allclose(P, o.P, rtol=0, atol=0)
    logs = f.pass_logs()
    assert len(logs) == len(o.passes) == pr.cfg.max_iter + 1
    assert all(l["valid"] == 0 and l["effct"] == 0 for l in logs)


@pytest.mark.parametrize("extr", [0, 1])
def test_fused_kernel_equals_the_split_kernels(problems, extr):
    """k_update (one persistent launch, solver block with the one-right-hand-side gain) against the two-kernels-per-pass chain
    with the 6x6 / 12x12 solve it replaced: same per-pass sums bit for bit (same rows, same reduction order is NOT required --
    the block partition differs -- so 1e-12), same state to rounding."""
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    res = []
    for fused in (1, 0):
        f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, extrinsic_est_en=bool(extr), fused=fused)
        assert f.fused() == bool(fused)
        x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
        res.append((x, P, f.pass_logs(), f.nearest(len(pr.scan)), f.selected(len(pr.scan)), f.gpu_launches()))
    (xa, Pa, la, na, sa, launches_a), (xb, Pb, lb, nb, sb, launches_b) = res
    assert launches_a == 1 and launches_b >= 8
    assert len(la) == len(lb)
    for a, b in zip(la, lb):
        assert (a["searched"], a["effct"], a["converged"], a["valid"]) == (b["searched"], b["effct"], b["converged"], b["valid"])
        assert np.allclose(a["HtH"], b["HtH"], rtol=1e-12, atol=1e-12 * np.abs(b["HtH"]).max())
        assert np.abs(a["x_after"] - b["x_after"]).max() < 1e-11
    assert np.array_equal(na[0], nb[0]) and np.array_equal(na[1], nb[1]) and np.array_equal(sa, sb)
    assert np.abs(xa - xb).max() < 1e-11
    assert np.abs(Pa - Pb).max() <= 1e-9 * np.abs(Pb).max()


def test_update_is_deterministic(problems):
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    a = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    b = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_full_size_properties(problems):
    """BASELINE config 2 (30k points vs 1M-point map): size-independent checks -- the GPU kNN of a
    sample against the port oracle, filter contraction towards the truth, symmetric P."""
    pr = problems("velodyne_30k_1m")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, solver=1)
    x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert np.abs(x[:3] - pr.x_true[:3]).max() < 2e-3 < np.abs(pr.x_prior[:3] - pr.x_true[:3]).max()
    assert np.allclose(P, P.T, atol=1e-12) and (np.linalg.eigvalsh(0.5 * (P + P.T)) > 0).all()
    near, cnt = f.nearest(len(pr.scan))
    assert (cnt == 5).all()
    # the cached neighbours are the exact 5-NN of the LAST searched pose: re-query them on the device map
    logs = f.pass_logs()
    last_search = max(i for i, l in enumerate(logs) if l["searched"])
    x_search = pr.x_prior if last_search == 0 else logs[last_search - 1]["x_after"]
    idx = np.arange(0, len(pr.scan), 97)
    q = np.zeros((len(idx), 4), dtype=np.float32)
    tmp = np.zeros(3, dtype=np.float32)
    for k, i in enumerate(idx):
        bind.lib().oracle_transform_point(np.ascontiguousarray(x_search), np.ascontiguousarray(pr.scan[i, :3]), tmp)
        q[k, :3] = tmp
    port = bind.KdTree(pr.map_pts, "port")
    pp, pd, pc = port.knn(q, 5)
    assert np.array_equal(near[idx][:, :, :3], pp[:, :, :3])


def test_bvh_and_cell_directory_search_give_identical_update(problems):
    """The BVH walk (one warp per point) and the cell-directory search (one lane per point) are interchangeable."""
    pr = problems("small")
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    out = []
    for search in (0, 1):
        f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, search=search)
        x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
        near, cnt = f.nearest(len(pr.scan))
        out.append((x, P, near, cnt))
    for k in (1,):
        assert np.array_equal(out[0][3], out[k][3]) and np.array_equal(out[0][2], out[k][2])
        assert np.array_equal(out[0][0], out[k][0]) and np.array_equal(out[0][1], out[k][1])


@pytest.mark.parametrize("n_pts", [0, 1, 4])
def test_empty_and_tiny_scans(problems, n_pts):
    """laserMapping.cpp:930-934 skips scans with < 5 points before the update is ever called; called anyway, the update must
    behave like the reference's: an empty or tiny scan contributes few or no rows, the passes run, nothing crashes."""
    pr = problems("tiny")
    scan = pr.scan[:n_pts].copy()
    o = RefTree(f"update_tiny_scan_{n_pts}", pr.map_pts).update_iterated(scan, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, 0)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    f = api.Esekf(t, max_points=64, max_iter=pr.cfg.max_iter)
    x, P, _ = f.update_iterated_dyn_share_modified(scan, pr.x_prior, pr.P_prior, pr.R)
    logs = f.pass_logs()
    assert len(logs) == len(o.passes)
    assert [l["effct"] for l in logs] == [p["effct"] for p in o.passes]
    check_state(o, x, P)
    if n_pts == 0:
        assert np.array_equal(x, pr.x_prior)


def test_update_against_a_map_with_fewer_than_k_points(problems):
    """Nearest_Search returns < 5 neighbours: point_selected_surf stays false for every point (laserMapping.cpp:671)."""
    pr = problems("tiny")
    few = pr.map_pts[:3].copy()
    t = api.KdTree(0, 0.5); t.Build(few)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert np.array_equal(x, pr.x_prior)
    logs = f.pass_logs()
    assert all(l["effct"] == 0 for l in logs)
    near, cnt = f.nearest(len(pr.scan))
    assert (cnt == 3).all() and not f.selected(len(pr.scan)).any()
    e = api.KdTree(0, 0.5); e.Build(np.zeros((0, 4), np.float32))      # and against an empty map
    g = api.Esekf(e, max_points=len(pr.scan), max_iter=pr.cfg.max_iter)
    x, P, _ = g.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert np.array_equal(x, pr.x_prior)
    assert (g.nearest(len(pr.scan))[1] == 0).all()
