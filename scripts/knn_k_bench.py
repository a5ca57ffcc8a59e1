"""Nearest_Search for k up to 32 with max_dist (fl_map_nearest_search) on the device map against the reference's ikd-Tree.

Map: the config-2 map (velodyne_30k_1m, 1 M points) and its 30 000 scan points pushed through the prior pose (world frame),
the queries of one FAST-LIO update.  Workloads: k in {5, 8, 16, 32} x max_dist in {+inf, 1 m}.  Per workload: host-clock
time of the synchronous batched call (median of --reps after a warm-up) with the cell directory on and off, the two maps
called alternately; the share of queries the directory proved (fl_map_dir_stats); result bytes (16 per neighbour + 4 per
distance + 4 per count) over that time; the reference's Nearest_Search(q, k, .., max_dist) through oracle/_ref
(oracle/knn_ref.py), serial and with OpenMP over the queries.  fl_map_knn at k = 5 (what the update runs) is timed the same
way for comparison.  The device answers are checked against the serial reference: counts and distances equal on every row,
neighbours equal on every decided row (tests/knn_rules.py, with each row's candidates taken from the k + 16 nearest by
scipy's cKDTree).  Prints one JSON line (also written to --out) with the card's name and power limit.
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
import knn_rules  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def world_queries(pr):
    from oracle.bind import lib
    q = np.zeros((len(pr.scan), 4), dtype=np.float32)
    L, tmp = lib(), np.zeros(3, dtype=np.float32)
    for i in range(len(pr.scan)):
        L.oracle_transform_point(pr.x_prior, np.ascontiguousarray(pr.scan[i, :3]), tmp)
        q[i, :3] = tmp
    return q


def alternate(fns, reps):
    """Median time of each callable, called in turn: one warm-up round, then `reps` rounds."""
    outs = [f() for f in fns]
    ts = [[] for _ in fns]
    for _ in range(reps):
        for j, f in enumerate(fns):
            t0 = time.perf_counter()
            outs[j] = f()
            ts[j].append(time.perf_counter() - t0)
    return [statistics.median(t) for t in ts], outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="velodyne_30k_1m")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("knn_k_bench: no CUDA device (the device map has no CPU path)")
    from oracle import bind, knn_ref
    from scipy.spatial import cKDTree
    name, power = card()
    pr = synth.make_problem(a.size)
    pts = pr.map_pts
    q = world_queries(pr)
    on = api.KdTree(0, 0.5); on.Build(pts)
    off = api.KdTree(0, 0.5, cell_directory=False); off.Build(pts)
    ref = bind.KdTree(pts, "reference") if knn_ref.available() else None
    _, cand = cKDTree(pts[:, :3].astype(np.float64)).query(q[:, :3].astype(np.float64), 32 + 16)
    (t_knn5,), _ = alternate([lambda: on.Nearest_Search(q, 5)], a.reps)
    res = {"bench": "nearest_search_k", "gpu": name, "power_limit": power, "host_cpus": os.cpu_count(), "map": a.size,
           "map_points": len(pts), "queries": len(q), "fl_map_knn_k5_s": t_knn5, "workloads": {}}
    for k in (5, 8, 16, 32):
        for md in (np.inf, 1.0):
            (t_on, t_off), (got, got_off) = alternate([lambda: on.Nearest_Search_K(q, k, md), lambda: off.Nearest_Search_K(q, k, md)], a.reps)
            on.dir_stats()
            on.Nearest_Search_K(q, k, md)
            walked = on.dir_stats()["walked"]
            nbytes = got[0].nbytes + got[1].nbytes + got[2].nbytes
            w = {"k": k, "max_dist": float(md), "device_dir_on_s": t_on, "device_dir_off_s": t_off,
                 "directory_proved": 1.0 - walked / len(q),
                 "neighbours": int(got[2].sum()), "result_bytes": nbytes, "result_GBps_dir_on": nbytes / t_on / 1e9,
                 "dir_on_equals_off": bool(all(x.tobytes() == y.tobytes() for x, y in zip(got[1:], got_off[1:])))}
            if ref is not None:
                t0 = time.perf_counter()
                rp, rd, rc = knn_ref.nearest_search(ref, q, k, md, nthreads=1)
                w["reference_serial_s"] = time.perf_counter() - t0
                t0 = time.perf_counter()
                par = knn_ref.nearest_search(ref, q, k, md, nthreads=a.threads)
                w["reference_omp_s"] = time.perf_counter() - t0
                w["reference_omp_threads"] = a.threads
                w["reference_omp_answers_equal_serial"] = bool(np.array_equal(par[2], rc) and par[1].tobytes() == rd.tobytes())
                decided = knn_rules.nearest(q, pts, k, md, cand=cand[:, :k + 16])[3]
                w["decided_rows"] = int(decided.sum())
                w["matches_reference"] = bool(np.array_equal(got[2], rc) and got[1].tobytes() == rd.tobytes()
                                              and np.array_equal(got[0][decided], rp[decided]))
            else:
                w["matches_reference"] = None
            res["workloads"][f"k{k}_maxdist_{md:g}"] = w
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
