"""Numpy restatement of the per-point rules of KD_TREE::Box_Search and Radius_Search (test infrastructure only).

  Box_Search     ikd_Tree.cpp:464-468 -> Search_by_range :1247-1289: vertex_min <= p < vertex_max on every axis.
  Radius_Search  ikd_Tree.cpp:470-475 -> Search_by_radius :1292-1332.  An interior node's own point is tested by
                 calc_dist(p, q) <= radius * radius (:1308) -- the "literal" rule, which the device map implements.  Leaves and
                 the subtrees caught by the short-cuts at :1302-1303 are decided by sqrtf(d2) compared with radius, so the
                 reference may also return points of the band B = {d2 > fl(r * r) and sqrtf(d2) <= r}.

Squared distances are float32 with every operation rounded, x + y first, then + z (calc_dist, ikd_Tree.cpp:1683-1689).
"""
from collections import Counter

import numpy as np

from semantics import sort_rows

F = np.float32


def sq_dist(c, pts):
    d = (pts[:, :3] - np.asarray(c[:3], dtype=F)).astype(F)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def box_mask(b, pts):
    b = np.asarray(b, dtype=F)
    return ((b[0] <= pts[:, 0]) & (pts[:, 0] < b[3]) & (b[1] <= pts[:, 1]) & (pts[:, 1] < b[4]) &
            (b[2] <= pts[:, 2]) & (pts[:, 2] < b[5]))


def radius_masks(q, pts):
    """(literal, band) masks over pts for one (x, y, z, r) query; both empty for NaN input or a negative radius."""
    q = np.asarray(q, dtype=F)
    if np.isnan(q).any() or not q[3] >= 0:
        z = np.zeros(len(pts), dtype=bool)
        return z, z
    d2 = sq_dist(q, pts)
    r = q[3]
    r2 = F(r * r)
    return d2 <= r2, (d2 > r2) & (np.sqrt(d2) <= r)


def box_sets(boxes6, pts):
    """The literal answer of every box, as sort_rows arrays."""
    pts = sort_rows(pts)
    return [pts[box_mask(b, pts)] for b in np.asarray(boxes6, dtype=F).reshape(-1, 6)]


def radius_sets(q4, pts):
    """(literal answers, band points) of every query, as sort_rows arrays."""
    pts = sort_rows(pts)
    lit, band = [], []
    for q in np.asarray(q4, dtype=F).reshape(-1, 4):
        l, b = radius_masks(q, pts)
        lit.append(pts[l]); band.append(pts[b])
    return lit, band


def members(rows, got):
    """For each row of `rows`: is a copy of it in `got` (multiset: each copy in got matches one row)?"""
    out = np.zeros(len(rows), dtype=bool)
    if len(rows) == 0:
        return out
    left = Counter(r.tobytes() for r in np.ascontiguousarray(got, dtype=F))
    for j, r in enumerate(np.ascontiguousarray(rows, dtype=F)):
        k = r.tobytes()
        if left[k] > 0:
            out[j] = True
            left[k] -= 1
    return out


def split(offsets, pts):
    """CSR output -> one sort_rows array per query."""
    return [sort_rows(pts[a:b]) for a, b in zip(offsets[:-1], offsets[1:])]


def make_queries(pts, rng, n):
    """n boxes and n spheres over the map: half random, half planted on the boundary -- box faces on point coordinates,
    radii equal to a point's float distance or the float just below it."""
    pts = np.asarray(pts, dtype=F)
    lo, hi = pts[:, :3].min(0), pts[:, :3].max(0)
    h = n // 2
    c = rng.uniform(lo, hi, (n, 3)).astype(F)
    half = rng.uniform(0.2, 6.0, (n, 3)).astype(F)
    boxes = np.concatenate([c - half, c + half], axis=1).astype(F)
    # planted boxes: min on a point's coordinates (that point is inside), or max on them (that point is outside)
    a = pts[rng.integers(0, len(pts), n - h), :3]
    on_min = (np.arange(n - h) % 2 == 0)[:, None]
    boxes[h:, :3] = np.where(on_min, a, a - half[h:])
    boxes[h:, 3:] = np.where(on_min, a + half[h:], a)
    spheres = np.zeros((n, 4), dtype=F)
    spheres[:, :3] = c
    spheres[:h, 3] = rng.uniform(0.3, 5.0, h).astype(F)
    # planted spheres: centre near a point, radius = the float distance of another nearby point (or one ulp below it)
    j = rng.integers(0, len(pts), n - h)
    spheres[h:, :3] = pts[j, :3] + rng.normal(0, 1.0, (n - h, 3)).astype(F)
    for i, jj in enumerate(j):
        d = np.sqrt(sq_dist(spheres[h + i], pts[jj:jj + 1]))[0]
        spheres[h + i, 3] = d if i % 2 == 0 else np.nextafter(d, F(0))
    return boxes, spheres
