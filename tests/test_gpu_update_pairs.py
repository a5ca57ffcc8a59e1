"""The update with two threads per scan point (k_update<EXTR, 2>, chosen automatically when the scan's tiles fit the 512-thread
grid) against one thread per point (FASTLIO_B200_PAIR=1): x, P, the pass logs, Nearest_Points, their counts and
point_selected_surf must be byte-equal, and so must the number of queries the BVH walk answered."""
import os

import numpy as np
import pytest

from fast_lio_b200 import api

pytestmark = pytest.mark.gpu


def run(tree, pr, scan, pair1, extr=0, search=-1, shard=None):
    """One whole update; returns every output as bytes."""
    if pair1:
        os.environ["FASTLIO_B200_PAIR"] = "1"
    else:
        os.environ.pop("FASTLIO_B200_PAIR", None)
    try:
        n = len(scan)
        f = api.Esekf(tree, max_points=n, max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr), search=search)
        w0 = tree.dir_stats()["walked"]
        if shard is None:
            x, P, _ = f.update_iterated_dyn_share_modified(scan, pr.x_prior, pr.P_prior, pr.R)
            sel = f.selected(n).tobytes()
        else:
            f.upload_scan(scan); f.set_shard(*shard); f.upload_state(pr.x_prior, pr.P_prior, pr.R); f.run()
            x, P, _ = f.download_state()
            sel = b""
        near, cnt = f.nearest(n)                   # a sharded filter completes the other shards' neighbours here
        walked = tree.dir_stats()["walked"] - w0
        logs = [(l["searched"], l["valid"], l["effct"], l["converged"], np.float64(l["res_sum"]).tobytes(), l["HtH"].tobytes(),
                 l["Hth"].tobytes(), l["x_after"].tobytes()) for l in f.pass_logs()]
        return dict(x=x.tobytes(), P=P.tobytes(), logs=logs, near=near.tobytes(), cnt=cnt.tobytes(), sel=sel, walked=walked)
    finally:
        os.environ.pop("FASTLIO_B200_PAIR", None)


def assert_same(tree, pr, scan, **kw):
    a = run(tree, pr, scan, True, **kw)
    b = run(tree, pr, scan, False, **kw)
    for k in a:
        assert a[k] == b[k], k
    return a


def built(pr):
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    return t


@pytest.mark.parametrize("name", ["tiny", "small"])
@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("search", [0, 1])
def test_pairs_equal_single_threads(problems, name, extr, search):
    pr = problems(name)
    assert_same(built(pr), pr, pr.scan, extr=extr, search=search)


@pytest.mark.parametrize("extr,search", [(0, 1), (1, 1), (0, 0)])
def test_pairs_equal_single_threads_config2(problems, extr, search):
    pr = problems("velodyne_30k_1m")
    out = assert_same(built(pr), pr, pr.scan, extr=extr, search=search)
    assert out["logs"][0][0] == 1 and out["logs"][0][2] > 0


def test_pairs_after_deletes_and_reinserts(problems):
    """Deleted points keep their listings and re-used slots are listed again: halo lists name a slot twice."""
    pr = problems("small")
    t = built(pr)
    pts = pr.map_pts
    rng = np.random.default_rng(5)
    c = pts[rng.integers(0, len(pts), 12), :3]
    boxes = np.concatenate([c - 1.5, c + 1.5], axis=1).astype(np.float32)
    t.Delete_Point_Boxes(boxes)
    inside = np.zeros(len(pts), bool)
    for b in boxes:
        inside |= ((pts[:, :3] >= b[:3]) & (pts[:, :3] < b[3:])).all(axis=1)
    back = pts[inside].copy()
    back[:, :3] += rng.normal(0, 0.05, (len(back), 3)).astype(np.float32)
    t.Add_Points(np.ascontiguousarray(back), False)
    for search in (1, 0):
        assert_same(t, pr, pr.scan, search=search)


def test_pairs_on_a_lattice_map(problems):
    """Map points on a 0.25 m lattice, scan points on lattice nodes: many neighbours at exactly equal distances."""
    pr = problems("small")
    g = np.arange(-6.0, 6.0, 0.25, dtype=np.float32)
    X, Y = np.meshgrid(g, g, indexing="ij")
    plane = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, np.float32), np.ones(X.size, np.float32)], axis=1)
    lattice = np.concatenate([plane, plane + np.array([0, 0, 0.25, 0], np.float32)]).astype(np.float32)
    t = api.KdTree(0, 0.0)
    t.Build(np.ascontiguousarray(lattice))
    rng = np.random.default_rng(7)
    scan = np.zeros((3000, 4), np.float32)
    scan[:, 0] = rng.integers(-20, 20, 3000) * 0.25
    scan[:, 1] = rng.integers(-20, 20, 3000) * 0.25
    scan[:, 2] = 0.125
    pr0 = problems("small")
    x0 = pr0.x_prior.copy()
    x0[0:3] = 0.0; x0[3:7] = [0, 0, 0, 1]; x0[7:11] = [0, 0, 0, 1]; x0[11:14] = 0.0
    pr = type("P", (), dict(cfg=pr0.cfg, limit=pr0.limit, x_prior=x0, P_prior=pr0.P_prior, R=pr0.R))
    for search in (1, 0):
        assert_same(t, pr, scan, search=search)


def test_pairs_sharded_with_completed_neighbours(problems):
    pr = problems("small")
    t = built(pr)
    n = len(pr.scan)
    assert_same(t, pr, pr.scan, shard=api.shard_range(n, 3, 1))
