"""CPU: the numpy statement of the deterministic mode's rules (det_rules.py) against brute force on lattice data, where
bit-equal squared distances are everywhere."""
import itertools

import numpy as np

import det_rules
from knn_rules import sq_dist

F = np.float32


def lattice(seed=3, n_dup=40):
    rng = np.random.default_rng(seed)
    g = np.arange(-2, 2.01, 0.5, dtype=F)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel(), rng.integers(0, 4, X.size).astype(F)], axis=1).astype(F)
    dup = pts[rng.choice(len(pts), n_dup, replace=False)].copy()       # same coordinates, other intensities
    dup[:, 3] += 7
    return np.concatenate([pts, dup])[rng.permutation(len(pts) + n_dup)]


def brute(q, pts, k, max_dist):
    """The k smallest by Python tuple comparison of (d2, ord x, ord y, ord z, ord intensity)."""
    md2 = F(F(max_dist) * F(max_dist))
    d = sq_dist(q, pts)
    o = det_rules.ord_bits(pts)
    rows = sorted((float(d[i]), int(o[i, 0]), int(o[i, 1]), int(o[i, 2]), int(o[i, 3]), i) for i in range(len(pts)) if d[i] <= md2)
    return [r[-1] for r in rows[:k]]


def test_ord_bits_orders_like_floats():
    v = np.array([-np.inf, -3.5, -1e-30, -0.0, 0.0, 1e-30, 2.0, np.inf], dtype=F)
    o = det_rules.ord_bits(v)
    assert (np.diff(o.astype(np.int64)) > 0).all()


def test_keyed_knn_equals_brute_force_on_lattice():
    pts = lattice()
    rng = np.random.default_rng(5)
    q = np.concatenate([pts[:20, :4], np.c_[rng.integers(-4, 5, (20, 3)) * F(0.25), np.zeros(20)]]).astype(F)
    for k, md in itertools.product([1, 5, 8, 16, 32], [np.inf, 0.5, 0.75]):
        p, d, c, exact = det_rules.nearest(q, pts, k, md)
        for i in range(len(q)):
            sel = brute(q[i], pts, k, md)
            assert c[i] == len(sel)
            assert d[i, :c[i]].tobytes() == sq_dist(q[i], pts[sel]).tobytes()
            # the set always; the order where d2 values are equal or apart by more than 1e-10 (always, on this lattice)
            assert exact[i]
            assert p[i, :c[i]].tobytes() == pts[sel].tobytes()
    # ties at the k-th place really occur here, so the rule is not vacuous
    assert det_rules.reference_arbitrary(q, pts, 5).any()


def test_keyed_knn_does_not_depend_on_point_order():
    pts = lattice()
    q = pts[:30]
    a = det_rules.nearest(q, pts, 8)
    b = det_rules.nearest(q, pts[::-1].copy(), 8)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def test_voxel_survivor_is_smallest_key_at_equal_distance():
    mid = np.array([0.25, 0.25, 0.25], dtype=F)
    offs = np.array([[1, 1, 1], [-1, 1, 1], [1, -1, 1], [1, 1, -1], [-1, -1, -1]], dtype=F) * F(0.125)
    pts = np.c_[mid + offs, np.arange(5, dtype=F)].astype(F)
    for perm in itertools.permutations(range(5)):
        s = det_rules.voxel_survivor(pts[list(perm)], mid)
        assert pts[list(perm)][s].tobytes() == pts[4].tobytes()      # (-,-,-): the smallest x, then y, then z
