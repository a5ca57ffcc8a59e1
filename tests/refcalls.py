"""The reference's own ikd-Tree (oracle/_ref, compiled from the original project), live or replayed.

Tests that compare with the reference call it through RefTree.  Where oracle/_ref is built, RefTree runs it and checks
each answer against tests/golden/ref/<key>.npz; with FASTLIO_RECORD_REF=DIR in the environment it writes the answers
to DIR/<key>.npz instead.  Where oracle/_ref is not built, RefTree replays the stored answers in call order.  Every
stored answer carries a digest of its call's inputs, so a test whose calls change fails instead of reading the wrong
answer; where oracle/_ref is built, such a call is judged by the live reference alone, with a warning.  Point sets (a
flattened map, the neighbours of a kNN query, a scan's Nearest_Points) are stored as SHA-256 digests of their bytes.
"""
import hashlib
import os
import warnings
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import bind
from semantics import sort_rows

PASS_FIELDS = ("searched", "valid", "effct", "converged", "res_sum", "HtH", "Hth", "x_after")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype}{a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()[:16]


def rows_digest(pts4) -> str:
    """Digest of a point set, independent of its order."""
    return digest(sort_rows(pts4))


def row_digests(a) -> np.ndarray:
    """One 32-bit digest per row of a (for comparing a subset of the rows)."""
    a = np.ascontiguousarray(a)
    return np.array([int.from_bytes(hashlib.sha256(r.tobytes()).digest()[:4], "little") for r in a.reshape(len(a), -1)],
                    dtype=np.uint32)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class RefTree:
    def __init__(self, key: str, pts4, downsample: float = 0.5):
        self.key, self.n, self.rec = key, 0, {}
        path = os.path.join(GOLD, key + ".npz")
        self.record_dir = os.environ.get("FASTLIO_RECORD_REF")
        self.live = bind.KdTree(_f32(pts4), "reference", downsample=downsample) if bind.have_ref() else None
        if self.record_dir:
            assert self.live is not None, "recording needs oracle/_ref"
            self.stored = None
        elif os.path.exists(path):
            with np.load(path) as g:
                self.stored = dict(g)
        elif self.live is None:
            pytest.fail(f"no reference answers: neither oracle/_ref nor {path}")
        else:
            self.stored = None
        self._call("build", (_f32(pts4), np.float32(downsample)), lambda: ())

    def _call(self, name, inputs, run):
        i = self.n
        self.n += 1
        tag = f"{name}:{digest(*inputs)}"
        out = tuple(np.asarray(o) for o in run()) if self.live is not None else None
        if self.stored is not None:
            recorded = self.stored.get(f"c{i}_in")
            if recorded is None or recorded.item().decode() != tag:
                why = f"{self.key}: call {i} ({name}) " + ("was not recorded" if recorded is None else f"is not the recorded {recorded}")
                if out is None:
                    pytest.fail(why + "; record the answers again (FASTLIO_RECORD_REF)")
                warnings.warn(why + "; judged by the live reference only")
            else:
                want = tuple(self.stored[f"c{i}_o{j}"] for j in range(int(self.stored[f"c{i}_n"])))
                if out is None:
                    out = want
                else:
                    assert all(np.array_equal(a, b) for a, b in zip(out, want)), f"{self.key}: call {i} ({name}) differs from the stored answer"
        if self.record_dir:
            self.rec[f"c{i}_in"] = np.bytes_(tag)
            self.rec[f"c{i}_n"] = np.int32(len(out))
            for j, o in enumerate(out):
                self.rec[f"c{i}_o{j}"] = o
            os.makedirs(self.record_dir, exist_ok=True)
            np.savez_compressed(os.path.join(self.record_dir, self.key + ".npz"), **self.rec)
        return out

    def add(self, pts4, downsample_on: bool) -> int:
        pts4 = _f32(pts4)
        return int(self._call("add", (pts4, np.int8(downsample_on)), lambda: (self.live.add(pts4, downsample_on),))[0])

    def delete_boxes(self, boxes6) -> int:
        boxes6 = _f32(boxes6).reshape(-1, 6)
        return int(self._call("delete_boxes", (boxes6,), lambda: (self.live.delete_boxes(boxes6),))[0])

    def validnum(self) -> int:
        return int(self._call("validnum", (), lambda: (self.live.validnum(),))[0])

    def flatten_digest(self) -> str:
        """rows_digest of the valid points."""
        return self._call("flatten", (), lambda: (np.bytes_(rows_digest(self.live.flatten())),))[0].item().decode()

    def knn(self, q4, k: int = 5, neighbours: str = "digest"):
        """(neighbours, squared distances, counts).  neighbours = "points": the arrays themselves; "rows": the
        neighbours as row_digests and the distances as one digest; "digest": both as one digest each."""
        q4 = _f32(q4)
        form = ("digest", "rows", "points").index(neighbours)

        def run():
            p, d, c = self.live.knn(q4, k)
            if form == 2:
                return p, d, c
            return (row_digests(p) if form == 1 else np.bytes_(digest(p))), np.bytes_(digest(d)), c
        p, d, c = self._call("knn", (q4, np.int32(k), np.int8(form)), run)
        return (p, d, c) if form == 2 else ((p if form == 1 else p.item().decode()), d.item().decode(), c)

    def update_iterated(self, scan4, x26, P, max_iter, R=0.001, limit=0.001, extrinsic_est_en=0):
        """bind.update_iterated on this tree: x, P, the pass logs, and digests of Nearest_Points, their counts and
        point_selected_surf."""
        scan4 = _f32(scan4)
        x26, P = np.array(x26, dtype=np.float64), np.array(P, dtype=np.float64)
        args = (max_iter, R, limit, extrinsic_est_en)

        def run():
            o = bind.update_iterated(self.live, scan4, x26, P, *args)
            logs = tuple(np.array([p[f] for p in o.passes]) for f in PASS_FIELDS)
            return (o.x, o.P, np.bytes_(digest(o.nearest)), np.bytes_(digest(o.nearest_cnt)), np.bytes_(digest(o.selected))) + logs
        out = self._call("update_iterated", (scan4, x26, P, np.array(args, dtype=np.float64)), run)
        x, Pn, near, cnt, sel = out[:5]
        passes = [{f: (a[i] if a.ndim > 1 else a[i].item()) for f, a in zip(PASS_FIELDS, out[5:])} for i in range(len(out[5]))]
        near, cnt, sel = (a.item().decode() for a in (near, cnt, sel))
        return SimpleNamespace(x=x, P=Pn, passes=passes, nearest_digest=near, nearest_cnt_digest=cnt, selected_digest=sel)
