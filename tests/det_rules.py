"""Numpy statement of the deterministic map mode's rules (fl_map_set_deterministic; test infrastructure only).

Keys: a point's (x, y, z, intensity), each float32 compared as an order-preserving integer of its bits (ord_bits: the float
order, with -0 below +0).  Squared distances are the float32 of calc_dist (knn_rules.sq_dist).

  k-NN   The answer is the k smallest candidates (d2 <= fl(max_dist^2)) under the total order (d2, x, y, z, intensity), d2
         compared as the float.  Order: ascending d2; entries within 1e-10 by x (PointType_CMP); entries equal on both by
         (y, z, intensity).  Where two adjacent entries differ in d2 by a nonzero amount below 1e-10 the device's sort of
         "near" ties is not a total order, so `exact` marks the rows whose order the rule fixes; the set is fixed on all rows.
  voxel  Of the valid points of a down-sampling voxel at equal distance from its centre, the smallest key is the nearest.
"""
import numpy as np

from knn_rules import sq_dist

F = np.float32


def ord_bits(a):
    """uint64 array ordering like the float32 values of `a` (-0 below +0)."""
    u = np.ascontiguousarray(a, dtype=F).view(np.uint32).astype(np.uint64)
    neg = (u & 0x80000000) != 0
    return np.where(neg, 0xFFFFFFFF - u, u | 0x80000000)


def key_order(pts, d=None):
    """Indices of pts sorted by (d, x, y, z, intensity) (d omitted: by the key alone)."""
    pts = np.asarray(pts, dtype=F).reshape(-1, 4)
    cols = [ord_bits(pts[:, 3]), ord_bits(pts[:, 2]), ord_bits(pts[:, 1]), ord_bits(pts[:, 0])]
    if d is not None:
        cols.append(np.asarray(d, dtype=F))
    return np.lexsort(cols)


def nearest(q4, pts, k, max_dist=np.inf):
    """(pts[nq, k, 4], d2[nq, k], cnt[nq], exact[nq]) of the keyed k-NN over the valid map points `pts`."""
    q4 = np.asarray(q4, dtype=F).reshape(-1, 4)
    pts = np.asarray(pts, dtype=F).reshape(-1, 4)
    md2 = F(F(max_dist) * F(max_dist))
    nq = len(q4)
    out_p = np.zeros((nq, k, 4), dtype=F)
    out_d = np.full((nq, k), np.inf, dtype=F)
    cnt = np.zeros(nq, dtype=np.int32)
    exact = np.ones(nq, dtype=bool)
    for i, q in enumerate(q4):
        if np.isnan(md2) or not np.isfinite(q[:3]).all():
            continue
        d = sq_dist(q, pts)
        ok = np.flatnonzero(d <= md2)
        if len(ok) > k:                              # every candidate at the k-th distance stays in the running
            kth = np.partition(d[ok], k - 1)[k - 1]
            ok = ok[d[ok] <= kth]
        ok = ok[key_order(pts[ok], d[ok])][:k]
        n = len(ok)
        out_p[i, :n], out_d[i, :n], cnt[i] = pts[ok], d[ok], n
        dd = d[ok]
        near = np.abs(np.diff(dd)) < 1e-10
        if (near & (np.diff(dd) != 0)).any():
            exact[i] = False
        elif near.any():                             # equal d2: the device orders by x as a float, then (y, z, intensity)
            sel = pts[ok]
            if (near & (sel[1:, 0] == sel[:-1, 0]) & (ord_bits(sel[1:, 0]) != ord_bits(sel[:-1, 0]))).any():
                exact[i] = False                     # -0 against +0: float-equal x, bit-different
    return out_p, out_d, cnt, exact


def reference_arbitrary(q4, pts, k, max_dist=np.inf):
    """Rows where the reference's own answer is arbitrary: the k-th and (k+1)-th candidates have bit-equal d2, or two
    adjacent neighbours within 1e-10 share x (knn_rules' undecided rows)."""
    import knn_rules
    return ~knn_rules.nearest(q4, pts, k, max_dist)[3]


def voxel_survivor(pts, mid):
    """Index (into pts) of the point nearest the voxel centre `mid` under (d2, x, y, z, intensity)."""
    pts = np.asarray(pts, dtype=F).reshape(-1, 4)
    d = sq_dist(np.asarray(mid, dtype=F), pts)
    return int(key_order(pts, d)[0])
