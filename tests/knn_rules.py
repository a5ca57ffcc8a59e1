"""Numpy restatement of KD_TREE::Nearest_Search(point, k, .., max_dist) (test infrastructure only).

  Nearest_Search ikd_Tree.cpp:426-461 -> Search :1062-1244.  md2 = max_dist * max_dist in float32 (:1067).  A point is a
                 candidate when calc_dist(p, q) <= md2 (:1088); the answer is the min(k, #candidates) nearest candidates,
                 nearest first, and neighbours whose squared distances differ by less than 1e-10 come in ascending x
                 (PointType_CMP, ikd_Tree.h:102-108).  A NaN max_dist or a query with a non-finite coordinate finds nothing.

Squared distances are float32 with every operation rounded, x + y first, then + z (calc_dist, ikd_Tree.cpp:1683-1689).

A row is *decided* when the reference's own rules fix its points: the k-th and the (k+1)-th candidate distances differ (else
the reference keeps whichever its traversal found first), and every two adjacent neighbours within 1e-10 of each other have
exactly equal distances and different x (else the heap's order is unspecified).  Distances and counts are fixed on every row.
"""
import numpy as np

F = np.float32


def sq_dist(q, pts):
    d = (pts[:, :3] - np.asarray(q[:3], dtype=F)).astype(F)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def nearest(q4, pts, k, max_dist=np.inf, cand=None):
    """(pts[nq, k, 4], d2[nq, k], cnt[nq], decided[nq]) over the valid map points `pts`.  cand (optional, [nq, m] indices into
    pts): each query's candidates are looked for among these only -- enough when they hold the k + 1 nearest."""
    q4 = np.asarray(q4, dtype=F).reshape(-1, 4)
    pts = np.asarray(pts, dtype=F).reshape(-1, 4)
    md2 = F(F(max_dist) * F(max_dist))
    nq = len(q4)
    out_p = np.zeros((nq, k, 4), dtype=F)
    out_d = np.full((nq, k), np.inf, dtype=F)
    cnt = np.zeros(nq, dtype=np.int32)
    decided = np.ones(nq, dtype=bool)
    for i, q in enumerate(q4):
        if np.isnan(md2) or not np.isfinite(q[:3]).all():
            continue
        sub = pts if cand is None else pts[cand[i]]
        d = sq_dist(q, sub)
        ok = np.flatnonzero(d <= md2)
        if len(ok) > k + 1:
            ok = ok[np.argpartition(d[ok], k)[:k + 1]]
        ok = ok[np.lexsort((sub[ok, 0], d[ok]))]          # ascending d2, equal d2 by ascending x
        n = min(k, len(ok))
        sel = ok[:n]
        out_p[i, :n], out_d[i, :n], cnt[i] = sub[sel], d[sel], n
        if len(ok) > k and d[ok[k - 1]] == d[ok[k]]:
            decided[i] = False
        dd, xx = d[sel], sub[sel, 0]
        near = np.abs(np.diff(dd)) < 1e-10
        if (near & ((np.diff(dd) != 0) | (np.diff(xx) == 0))).any():
            decided[i] = False
    return out_p, out_d, cnt, decided
