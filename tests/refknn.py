"""RefTree with the reference's KD_TREE::Nearest_Search(point, k, .., max_dist) (oracle/knn_ref.py), live or replayed.

KnnRefTree records and replays exactly as RefTree does (tests/refcalls.py, same call tags, same tests/golden/ref files).  It
runs the reference only where both oracle/_ref libraries are built -- the tree and its k-nearest wrapper -- and replays the
stored answers otherwise.
"""
import os

import numpy as np
import pytest

from oracle import bind, knn_ref
from refcalls import GOLD, RefTree, _f32, digest, row_digests


class KnnRefTree(RefTree):
    def __init__(self, key: str, pts4, downsample: float = 0.5):
        # RefTree.__init__, with "the reference is live" meaning both libraries
        self.key, self.n, self.rec = key, 0, {}
        path = os.path.join(GOLD, key + ".npz")
        self.record_dir = os.environ.get("FASTLIO_RECORD_REF")
        self.live = bind.KdTree(_f32(pts4), "reference", downsample=downsample) if knn_ref.available() else None
        if self.record_dir:
            assert self.live is not None, "recording needs oracle/_ref (the tree and its k-nearest wrapper)"
            self.stored = None
        elif os.path.exists(path):
            with np.load(path) as g:
                self.stored = dict(g)
        elif self.live is None:
            pytest.fail(f"no reference answers: neither oracle/_ref nor {path}")
        else:
            self.stored = None
        self._call("build", (_f32(pts4), np.float32(downsample)), lambda: ())

    def flatten_points(self):
        """The valid points, as a sort_rows array (stored in full)."""
        from semantics import sort_rows
        return self._call("flatten_points", (), lambda: (sort_rows(self.live.flatten()),))[0]

    def nearest_search(self, q4, k: int, max_dist: float = np.inf):
        """KD_TREE::Nearest_Search(q, k, .., max_dist) per row: (row_digests of the neighbour rows, one digest of the squared
        distances, the counts)."""
        q4 = _f32(q4).reshape(-1, 4)

        def run():
            p, d, c = knn_ref.nearest_search(self.live, q4, k, max_dist)
            return row_digests(p), np.bytes_(digest(d)), c
        rows, d, c = self._call("nearest_search", (q4, np.int32(k), np.float32(max_dist)), run)
        return rows, d.item().decode(), c


def world_queries(pr):
    """Scan points pushed through the prior pose (float32), as h_share_model does."""
    from oracle.bind import lib
    q = np.zeros((len(pr.scan), 4), dtype=np.float32)
    L = lib()
    tmp = np.zeros(3, dtype=np.float32)
    for i in range(len(pr.scan)):
        L.oracle_transform_point(pr.x_prior, np.ascontiguousarray(pr.scan[i, :3]), tmp)
        q[i, :3] = tmp
    return q


KS = (6, 8, 16, 32)
MAX_DISTS = (0.0, 0.3, 1.0, 2.236, np.inf, -1.0, np.nan)
GATED_KS = (3, 5, 8, 32)


def gated_queries(pr, n=400):
    """Scan queries plus some placed on map points (max_dist = 0 finds those)."""
    q = world_queries(pr)[:n]
    on = pr.map_pts[np.random.default_rng(31).integers(0, len(pr.map_pts), 40)].copy()
    on[:, 3] = 0
    return np.ascontiguousarray(np.concatenate([q, on]).astype(np.float32))


def mutation_batch(rng, base_pts, n):
    """New points: most near existing map points (they compete in their voxel), a fifth in fresh space."""
    b = base_pts[rng.integers(0, len(base_pts), n)].copy()
    b[:, :3] += rng.normal(0, 0.3, (n, 3)).astype(np.float32)
    far = rng.random(n) < 0.2
    b[far, :3] += rng.uniform(5, 30, (int(far.sum()), 3)).astype(np.float32)
    b[:, 3] = rng.uniform(100, 200, n).astype(np.float32)
    return np.ascontiguousarray(b.astype(np.float32))


def mutation_run(pr, dev=None):
    """Add_Points(.., true), Add_Points(.., false) and Delete_Point_Boxes on the reference (and on the device map `dev`, when
    given, checking that both return the same), then Nearest_Search_K.  Yields per step (the reference's valid points, the
    queries, {(k, max_dist): the reference's answer}), before the next step changes either map."""
    from semantics import sort_rows
    rng = np.random.default_rng(12)
    r = KnnRefTree("knnk_mutation", pr.map_pts)
    for step in range(2):
        batch = mutation_batch(rng, pr.map_pts, 900)
        ra, rb = r.add(batch[:600], True), r.add(batch[600:], False)
        c = pr.map_pts[rng.integers(0, len(pr.map_pts)), :3]
        box = np.array([[*(c - 5), *(c + 5)]], dtype=np.float32)
        rd = r.delete_boxes(box)
        if dev is not None:
            assert dev.Add_Points(batch[:600], True) == ra and dev.Add_Points(batch[600:], False) == rb
            assert dev.Delete_Point_Boxes(box) == rd
        live = r.flatten_points()
        q = np.zeros((300, 4), np.float32)
        q[:, :3] = live[rng.integers(0, len(live), 300), :3] + rng.normal(0, 1.0, (300, 3)).astype(np.float32)
        q[:20, :3] = c + rng.uniform(-4, 4, (20, 3)).astype(np.float32)         # inside the deleted box
        yield live, q, {(k, md): r.nearest_search(q, k, md) for k, md in ((8, np.inf), (32, 1.5), (5, 1.0))}
