"""How much of a searching pass the BVH walks of k_update_wave cost: the ceiling of any change that answers the walked queries
another way.

    python scripts/walk_tail_probe.py [--rounds N] [--steps K] [--out FILE]

A query whose cell's halo list does not prove its k nearest (tests/cell_directory_model.py, HaloRuleModel: the kernel's rule in
float32 numpy) goes to its block's walk pool and through the BVH.  For avia_2k_50k and config 2 (velodyne_30k_1m) the script
finds those queries at the two poses the update searches from -- the prior, and the x_after of the pass before the second
searching pass in the library's own pass logs -- and builds three scans:
    (a) the full scan;
    (b) the scan without those queries;
    (c) the scan without as many randomly chosen proven queries (a control for the point count).
In every round it times (a), (b) and (c) in turn: fl_filter_time_resident with the L2 flushed and warm, and
fl_filter_time_search_pass flushed, K steps each.  It reports per-step medians over the rounds, the repeat spread (relative gap
between the medians of the first and second half of the rounds), the passes and the queries walked per update.  (c) - (b) is the
most that removing the walk can gain.  Prints one JSON line (also written to --out) with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cell_directory_model import HaloRuleModel  # noqa: E402
from fast_lio_b200 import api, synth  # noqa: E402
from oracle import bind  # noqa: E402

WORKLOADS = ["avia_2k_50k", "velodyne_30k_1m"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, power


def world(x26, scan):
    q = np.zeros((len(scan), 3), dtype=np.float32)
    tmp = np.zeros(3, dtype=np.float32)
    x = np.ascontiguousarray(x26, dtype=np.float64)
    for i in range(len(scan)):
        bind.lib().oracle_transform_point(x, np.ascontiguousarray(scan[i, :3]), tmp)
        q[i] = tmp
    return q


def unproven(model, q):
    return np.array([not model.knn(qq)[2] for qq in q], dtype=bool)


class Run:
    def __init__(self, tree, pr, scan):
        self.tree, self.pr, self.scan = tree, pr, scan
        self.f = api.Esekf(tree, max_points=len(scan), max_iter=pr.cfg.max_iter, limit=pr.limit)

    def update(self):
        self.tree.dir_stats()                             # its walk counter restarts at every read
        self.f.update_iterated_dyn_share_modified(self.scan, self.pr.x_prior, self.pr.P_prior, self.pr.R)
        return self.f.pass_logs(), self.tree.dir_stats()["walked"]

    def times(self, steps):
        f = self.f
        f.upload_scan(self.scan)
        f.upload_state(self.pr.x_prior, self.pr.P_prior, self.pr.R)
        return {"step_flushed_us": 1e3 * f.time_resident(steps, flush_l2=True) / steps,
                "step_warm_us": 1e3 * f.time_resident(steps, flush_l2=False) / steps,
                "search_flushed_us": 1e3 * f.time_search_pass(steps, flush_l2=True) / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, power = card()
    res = {"bench": "walk_tail_probe", "gpu": name, "power_limit": power, "rounds": a.rounds, "steps_per_call": a.steps,
           "timing": "CUDA events inside fl_filter_time_resident / fl_filter_time_search_pass, per step; (a), (b), (c) in turn every round",
           "workloads": {}}
    for wl in a.workloads.split(","):
        pr = synth.make_problem(wl)
        tree = api.KdTree(0, 0.5)
        tree.Build(pr.map_pts)
        model = HaloRuleModel(pr.map_pts, 1.0)
        full = Run(tree, pr, pr.scan)
        logs, _ = full.update()
        searched = [i for i, lg in enumerate(logs) if lg["searched"]]
        poses = [pr.x_prior] + ([np.asarray(logs[searched[1] - 1]["x_after"], dtype=np.float64)] if len(searched) > 1 else [])
        masks = [unproven(model, world(x, pr.scan)) for x in poses]
        drop = np.logical_or.reduce(masks)
        rng = np.random.default_rng(1)
        ctrl = np.zeros(len(pr.scan), dtype=bool)
        ctrl[rng.choice(np.flatnonzero(~drop), int(drop.sum()), replace=False)] = True
        runs = {"a_full": full, "b_without_unproven": Run(tree, pr, pr.scan[~drop]), "c_without_random_proven": Run(tree, pr, pr.scan[~ctrl])}
        entry = {"scan_points": len(pr.scan), "map_points": len(pr.map_pts), "unproven_per_searching_pose": [int(m.sum()) for m in masks],
                 "removed": int(drop.sum()), "variants": {}}
        for k, r in runs.items():
            lg, walked = r.update()
            entry["variants"][k] = {"points": len(r.scan), "passes": len(lg), "searching_passes": int(sum(l["searched"] for l in lg)),
                                    "walked_per_update": int(walked)}
            r.times(max(3, a.steps // 10))                # warm-up
        ts = {k: [] for k in runs}
        for _ in range(a.rounds):
            for k, r in runs.items():
                ts[k].append(r.times(a.steps))
        h = a.rounds // 2
        for k in runs:
            for m in ts[k][0]:
                v = [t[m] for t in ts[k]]
                m1, m2 = statistics.median(v[:h]), statistics.median(v[h:])
                entry["variants"][k][m] = {"median": statistics.median(v), "repeat_spread": abs(m1 - m2) / min(m1, m2)}
        entry["ceiling_c_minus_b_us"] = {m: entry["variants"]["c_without_random_proven"][m]["median"] - entry["variants"]["b_without_unproven"][m]["median"]
                                         for m in ts["a_full"][0]}
        res["workloads"][wl] = entry
        print(json.dumps({wl: entry}), file=sys.stderr)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
