"""Box_Search / Radius_Search on the device map against the reference's ikd-Tree and the old flatten + host filter.

Map: the config-2 map (velodyne_30k_1m, 1 M points; --sizes adds ouster64_131k_5m).  Workloads:
  (a) 30 000 spheres of r = 1 m   (b) 1 000 spheres of r = 10 m   (c) 64 boxes with 20 m edges   (d) one box holding the map
Per workload: host-clock time of the synchronous batched call (median of --reps after a warm-up), points returned, and result
bytes (16 per point + 4 per offset) over that time; the reference's Box_Search / Radius_Search through oracle/_ref (oracle/range_ref.py), serial and
with OpenMP over the queries (reported only when its answers equal the serial ones); fl_map_flatten plus a numpy filter (what
the KD_TREE facade did before), timed on a few queries and scaled to the workload.  The device answers are checked: boxes equal
the reference's; spheres differ from it only on band points (d2 > fl(r * r) and sqrtf(d2) <= r); a sample of queries equals
the numpy rule.  Prints one JSON line (also written to --out) with the card's name and power limit.
"""
import argparse
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

from fast_lio_b200 import api, synth  # noqa: E402
import range_rules as rr  # noqa: E402
from semantics import sort_rows  # noqa: E402

F = np.float32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def timed(fn, reps, warmup=1):
    for _ in range(warmup):
        out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), out


def workloads(pts, rng):
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


def check(kind, q, dev, ref, pts, rng, n_sample=20):
    """boxes: equal multisets; spheres: the differences are band points the reference took; a sample equals the rule."""
    (do, dp), (ro, rp) = dev, ref
    if not np.array_equal(np.diff(do), np.diff(ro)) and kind == "box":
        return False
    for i in range(len(q)):
        g, r = sort_rows(dp[do[i]:do[i + 1]]), sort_rows(rp[ro[i]:ro[i + 1]])
        if g.tobytes() == r.tobytes():
            continue
        if kind == "box":
            return False
        only_g, only_r = g[~rr.members(g, r)], r[~rr.members(r, g)]
        d2 = rr.sq_dist(q[i], only_r)
        r_ = q[i, 3]
        if len(only_g) or not ((d2 > F(r_ * r_)) & (np.sqrt(d2) <= r_)).all():
            return False
    for i in rng.choice(len(q), min(n_sample, len(q)), replace=False):
        want = pts[rr.box_mask(q[i], pts)] if kind == "box" else pts[rr.radius_masks(q[i], pts)[0]]
        if sort_rows(dp[do[i]:do[i + 1]]).tobytes() != sort_rows(want).tobytes():
            return False
    return True


def run_size(name, reps, threads):
    from oracle import bind, range_ref
    pr = synth.make_problem(name)
    pts = pr.map_pts
    rng = np.random.default_rng(2)
    g = api.KdTree(0, 0.5); g.Build(pts)
    t_flat, flat = timed(g.flatten, reps)
    ref = bind.KdTree(pts, "reference") if range_ref.available() else None
    res = {"map": name, "map_points": len(pts), "flatten_s": t_flat, "flatten_bytes": 16 * len(flat), "workloads": {}}
    for wname, (kind, q) in workloads(pts, rng).items():
        call = (lambda: g.Box_Search(q)) if kind == "box" else (lambda: g.Radius_Search(q[:, :3], q[:, 3]))
        t_dev, (off, out) = timed(call, reps)
        n = int(off[-1])
        w = {"queries": len(q), "points": n, "device_s": t_dev, "result_bytes": 16 * n + 4 * len(off),
             "device_GBps": (16 * n + 4 * len(off)) / t_dev / 1e9}
        # the old facade: flatten, then filter on the host -- timed on a few queries, scaled to the workload
        k = min(len(q), 8)
        t0 = time.perf_counter()
        for i in range(k):
            allp = g.flatten()
            allp[rr.box_mask(q[i], allp)] if kind == "box" else allp[rr.radius_masks(q[i], allp)[0]]
        w["flatten_filter_s_scaled"] = (time.perf_counter() - t0) / k * len(q)
        if ref is not None:
            search = range_ref.box_search if kind == "box" else range_ref.radius_search
            fn = lambda q, nthreads: search(ref, q, nthreads)  # noqa: E731
            t0 = time.perf_counter()
            serial = fn(q, 1)
            w["reference_serial_s"] = time.perf_counter() - t0
            t0 = time.perf_counter()
            par = fn(q, threads)
            t_par = time.perf_counter() - t0
            same = np.array_equal(par[0], serial[0]) and par[1].tobytes() == serial[1].tobytes()
            w["reference_omp_threads"] = threads
            w["reference_omp_s"] = t_par if same else None
            w["reference_omp_answers_equal_serial"] = bool(same)
            w["matches_reference"] = bool(check(kind, q, (off, out), serial, pts, rng))
        else:
            w["matches_reference"] = None
        res["workloads"][wname] = w
    dw = res["workloads"]["d_box_whole_map_x1"]
    res["whole_map_box_over_flatten"] = dw["device_s"] / t_flat
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="velodyne_30k_1m", help="comma-separated synth configs")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("range_bench: no CUDA device (the device map has no CPU path)")
    name, power = card()
    line = {"bench": "range_search", "gpu": name, "power_limit": power, "host_cpus": os.cpu_count(),
            "sizes": [run_size(s, a.reps, a.threads) for s in a.sizes.split(",")]}
    txt = json.dumps(line)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
