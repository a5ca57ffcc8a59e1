"""RefTree with the reference's KD_TREE::Box_Search and Radius_Search (oracle/range_ref.py), live or replayed.

RangeRefTree records and replays exactly as RefTree does (tests/refcalls.py, same call tags, same tests/golden/ref files).
It runs the reference only where both oracle/_ref libraries are built -- the tree and its range wrapper -- and replays the
stored answers otherwise.
"""
import os

import numpy as np
import pytest

import range_rules
from oracle import bind, range_ref
from refcalls import GOLD, RefTree, _f32, rows_digest
from semantics import sort_rows


class RangeRefTree(RefTree):
    def __init__(self, key: str, pts4, downsample: float = 0.5):
        # RefTree.__init__, with "the reference is live" meaning both libraries
        self.key, self.n, self.rec = key, 0, {}
        path = os.path.join(GOLD, key + ".npz")
        self.record_dir = os.environ.get("FASTLIO_RECORD_REF")
        self.live = bind.KdTree(_f32(pts4), "reference", downsample=downsample) if range_ref.available() else None
        if self.record_dir:
            assert self.live is not None, "recording needs oracle/_ref (the tree and its range wrapper)"
            self.stored = None
        elif os.path.exists(path):
            with np.load(path) as g:
                self.stored = dict(g)
        elif self.live is None:
            pytest.fail(f"no reference answers: neither oracle/_ref nor {path}")
        else:
            self.stored = None
        self._call("build", (_f32(pts4), np.float32(downsample)), lambda: ())

    def box_search(self, boxes6):
        """KD_TREE::Box_Search per box: (counts, rows_digest of each answer)."""
        boxes6 = _f32(boxes6).reshape(-1, 6)

        def run():
            off, got = range_ref.box_search(self.live, boxes6)
            return np.diff(off).astype(np.int32), np.array([rows_digest(got[a:b]).encode() for a, b in zip(off[:-1], off[1:])], dtype="S16")
        cnt, dig = self._call("box_search", (boxes6,), run)
        return cnt, [d.decode() for d in dig]

    def radius_search(self, centers_xyzr, map_pts):
        """KD_TREE::Radius_Search per (x, y, z, r) row: the answer of each query as a sort_rows array.  map_pts are the map's
        valid points now (they must be the reference's).  Stored: per query the count and rows_digest, and one bit per point
        of the band B (range_rules) saying whether the reference returned it; the answer is rebuilt as the literal set plus
        the flagged band points and checked against the count and digest -- so literal <= answer <= literal + B."""
        q = _f32(centers_xyzr).reshape(-1, 4)
        pts = sort_rows(_f32(map_pts))
        lit, band = range_rules.radius_sets(q, pts)

        def run():
            off, got = range_ref.radius_search(self.live, q)
            dig = np.array([rows_digest(got[a:b]).encode() for a, b in zip(off[:-1], off[1:])], dtype="S16")
            bits = [range_rules.members(band[i], got[off[i]:off[i + 1]]) for i in range(len(q))]
            return np.diff(off).astype(np.int32), dig, np.packbits(np.concatenate(bits + [np.zeros(0, bool)]))
        cnt, dig, bits = self._call("radius_search", (q, pts), run)
        flags = np.unpackbits(bits)[:sum(len(b) for b in band)].astype(bool)
        out, k = [], 0
        for i in range(len(q)):
            f = flags[k:k + len(band[i])]
            k += len(band[i])
            s = sort_rows(np.concatenate([lit[i], band[i][f]]))
            assert len(s) == cnt[i] and rows_digest(s) == dig[i].decode(), \
                f"{self.key}: query {i}: the reference's answer is not the literal set plus band points"
            out.append(s)
        return out
