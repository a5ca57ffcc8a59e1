"""Host-buffer map queries of two builds of libfastlio_b200.so, compared answer for answer and timed in turn.

    python scripts/host_query_ab.py OLD.so NEW.so [--reps N] [--out FILE]

Each library is loaded with ctypes (a binding of its own: fast_lio_b200.api loads one library only) and builds its own map
from the config-2 points (velodyne_30k_1m, 1 M points) with fl_map_build.  The two maps are then queried through the
host-buffer entry points on the workloads of scripts/knn_k_bench.py and scripts/range_bench.py:
  - fl_map_knn at k = 5 on the 30 000 world-frame scan points;
  - fl_map_nearest_search at k in {1, 3, 5, 8, 16, 32} x max_dist in {+inf, 1 m}, on the same queries with a few NaN and
    +-inf rows;
  - range workloads (a)-(d) of range_bench.py at cap in {0, total / 2, total, total + 7}.
Every output buffer starts filled with the same sentinel, so the bytes beyond what a call writes are compared too.  Return
values, counts, d2, offsets and padding must be byte-equal, and so must the points, except that a nearest-search row may
keep a different one of several points at an equal d2: such rows are counted and reported.  Timing: in each round every
library is called twice, old, new, old, new; per workload the script reports each library's median host-clock time of the
synchronous call and, as the spread between repeated runs of the same code, the relative gap between the medians of each
library's first and second call.  Prints one JSON line (also written to --out) with the card's name and power limit, read
in the same run.  Exits non-zero if any answer differs.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_lio_b200 import synth  # noqa: E402
from refknn import world_queries  # noqa: E402

F = np.float32
_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
SENTINEL = 0xDEADBEEF


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def filled(shape, dtype=np.float32):
    a = np.empty(shape, dtype)
    a.view(np.uint32)[...] = SENTINEL
    return a


class HostMap:
    """One library's map, queried through its host-buffer entry points."""

    def __init__(self, path, pts):
        L = self.L = C.CDLL(os.path.abspath(path))
        L.fl_last_error.restype = C.c_char_p
        L.fl_map_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_float]
        L.fl_map_build.argtypes = [C.c_void_p, _f32p, C.c_int]
        L.fl_map_knn.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, _f32p, _f32p, _i32p]
        L.fl_map_nearest_search.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_float, _f32p, _f32p, _i32p]
        for fn in (L.fl_map_box_search, L.fl_map_radius_search):
            fn.argtypes = [C.c_void_p, _f32p, C.c_int, _i32p, _f32p, C.c_int]
        self.h = C.c_void_p()
        self.check(L.fl_map_create(C.byref(self.h), 0, 0.5))
        self.check(L.fl_map_build(self.h, pts, len(pts)))

    def check(self, rc):
        if rc < 0:
            raise RuntimeError(f"error {rc}: {self.L.fl_last_error().decode(errors='replace')}")

    def knn(self, q, k, max_dist=None):
        nq = len(q)
        p, d, c = filled((nq, k, 4)), filled((nq, k)), filled(nq, np.int32)
        rc = (self.L.fl_map_knn(self.h, q, nq, k, p, d, c) if max_dist is None
              else self.L.fl_map_nearest_search(self.h, q, nq, k, max_dist, p, d, c))
        return rc, p, d, c

    def range(self, kind, q, cap):
        off, out = filled(len(q) + 1, np.int32), filled((max(cap, 1), 4))
        fn = self.L.fl_map_radius_search if kind == "radius" else self.L.fl_map_box_search
        return fn(self.h, q, len(q), off, out, cap), off, out


def timed_ab(fa, fb, reps):
    """Old, new, old, new in every round after one warm-up round: each library's median, and the spread of its two calls."""
    outs = [fa(), fb()]
    ts = [[], [], [], []]
    for _ in range(reps):
        for j, f in enumerate((fa, fb, fa, fb)):
            t0 = time.perf_counter()
            outs[j % 2] = f()
            ts[j].append(time.perf_counter() - t0)
    m = [statistics.median(t) for t in ts]
    res = {"old_s": statistics.median(ts[0] + ts[2]), "new_s": statistics.median(ts[1] + ts[3]),
           "old_repeat_spread": abs(m[0] - m[2]) / min(m[0], m[2]), "new_repeat_spread": abs(m[1] - m[3]) / min(m[1], m[3])}
    res["new_over_old"] = res["new_s"] / res["old_s"]
    return res, outs


def sq_dist(q, p):
    d = (p[..., :3] - q[:3]).astype(F)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def compare_knn(q, a, b):
    """(equal, rows whose points differ only by which of several points at an equal d2 was kept)"""
    if a[0] != b[0] or any(x.tobytes() != y.tobytes() for x, y in zip(a[2:], b[2:])):
        return False, 0
    pa, pb, d = a[1], b[1], a[2]
    rows = np.nonzero((pa.view(np.uint32) != pb.view(np.uint32)).any(axis=(1, 2)))[0]
    for i in rows:
        j = (pa[i].view(np.uint32) != pb[i].view(np.uint32)).any(axis=1)
        # both kept points lie at the entry's reported d2, so they tie
        if not (np.array_equal(sq_dist(q[i], pa[i][j]), d[i][j]) and np.array_equal(sq_dist(q[i], pb[i][j]), d[i][j])):
            return False, int(len(rows))
    return True, int(len(rows))


def range_workloads(pts, rng):
    lo, hi = pts[:, :3].min(0), pts[:, :3].max(0)

    def centres(n):
        return (pts[rng.integers(0, len(pts), n), :3] + rng.normal(0, 0.5, (n, 3))).astype(F)
    c = centres(64)
    return {
        "a_radius_1m_x30000": ("radius", np.concatenate([centres(30000), np.full((30000, 1), 1.0, F)], axis=1)),
        "b_radius_10m_x1000": ("radius", np.concatenate([centres(1000), np.full((1000, 1), 10.0, F)], axis=1)),
        "c_box_20m_x64": ("box", np.concatenate([c - 10, c + 10], axis=1).astype(F)),
        "d_box_whole_map_x1": ("box", np.array([[*(lo - 1), *(hi + 1)]], dtype=F)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old_lib")
    ap.add_argument("new_lib")
    ap.add_argument("--size", default="velodyne_30k_1m")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, power = card()
    pr = synth.make_problem(a.size)
    pts = np.ascontiguousarray(pr.map_pts, dtype=F)
    old, new = HostMap(a.old_lib, pts), HostMap(a.new_lib, pts)
    q = world_queries(pr)
    qbad = q.copy()
    qbad[0, :3] = np.nan
    qbad[1, 0] = np.inf
    qbad[2, 1] = -np.inf
    qbad[3, 2] = np.nan
    res = {"bench": "host_query_ab", "gpu": name, "power_limit": power, "old_lib": a.old_lib, "new_lib": a.new_lib,
           "map": a.size, "map_points": len(pts), "queries": len(q), "reps": a.reps,
           "timing": "host clock of each synchronous call; old, new, old, new in every round", "workloads": {}}
    all_equal = True

    def record(key, t, equal, **extra):
        nonlocal all_equal
        all_equal &= equal
        res["workloads"][key] = {**t, "equal": bool(equal), **extra}

    t, (ga, gb) = timed_ab(lambda: old.knn(q, 5), lambda: new.knn(q, 5), a.reps)
    eq, ties = compare_knn(q, ga, gb)
    record("knn_k5", t, eq, tie_rows=ties)
    for k in (1, 3, 5, 8, 16, 32):
        for md in (np.inf, 1.0):
            t, (ga, gb) = timed_ab(lambda: old.knn(qbad, k, md), lambda: new.knn(qbad, k, md), a.reps)
            eq, ties = compare_knn(qbad, ga, gb)
            record(f"nearest_k{k}_maxdist_{md:g}", t, eq, tie_rows=ties, neighbours=int(ga[3].sum()))
    for wname, (kind, rq) in range_workloads(pts, np.random.default_rng(2)).items():
        total = old.range(kind, rq, 0)[0]
        for cap in sorted({0, total // 2, total, total + 7}):
            t, (ga, gb) = timed_ab(lambda: old.range(kind, rq, cap), lambda: new.range(kind, rq, cap), a.reps)
            eq = ga[0] == gb[0] and all(x.tobytes() == y.tobytes() for x, y in zip(ga[1:], gb[1:]))
            record(f"{wname}_cap{cap}", t, eq, total=int(ga[0]), cap=cap)
    ws = res["workloads"].values()
    res["all_equal"] = bool(all_equal)
    res["worst_new_over_old"] = max(w["new_over_old"] for w in ws)
    res["max_repeat_spread"] = max(max(w["old_repeat_spread"], w["new_repeat_spread"]) for w in ws)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")
    if not all_equal:
        raise SystemExit("host_query_ab: the two libraries' answers differ")


if __name__ == "__main__":
    main()
