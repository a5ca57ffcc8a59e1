"""The fused update (k_update) of two builds of libfastlio_b200.so, compared output for output and timed in turn.

    python scripts/update_ab.py OLD.so NEW.so [--rounds N] [--steps K] [--out FILE]

Each library is bound through fast_lio_b200.api (rebound to that library's file; ctypes keeps the two libraries' symbols
apart) and builds its own map and filter for each workload: avia_2k_50k, velodyne_30k_1m (config 2) and ouster64_131k_5m
(config 3).  Outputs: one whole update through fl_filter_update with host buffers; x, P, the pass logs, Nearest_Points, their
counts and point_selected_surf must be byte-equal, and so must the number of queries the BVH walk answered.  Timing: in every
round, old, new, old, new, each call K resident steps of fl_filter_time_resident with the L2 flushed, K with it warm, and K
search-only launches of fl_filter_time_search_pass flushed and warm.  Per measure the script reports each library's median
over the rounds and, as the spread between repeated runs of the same code, the relative gap between the medians of each
library's first and second call in a round.  Prints one JSON line (also written to --out) with the card's name and power
limit, read in the same run.  Exits non-zero if any output differs.
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

from fast_lio_b200 import api, synth  # noqa: E402

WORKLOADS = ["avia_2k_50k", "velodyne_30k_1m", "ouster64_131k_5m"]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def bind(path):
    """Point fast_lio_b200.api at `path`; objects created afterwards keep that library."""
    api._lib = None
    api._build.LIB = os.path.abspath(path)
    return api.load()


class Run:
    """One library's map and filter for one workload."""

    def __init__(self, path, pr):
        bind(path)
        self.pr = pr
        self.tree = api.KdTree(0, 0.5)
        self.tree.Build(pr.map_pts)
        self.f = api.Esekf(self.tree, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit,
                           extrinsic_est_en=bool(pr.extrinsic_est_en))

    def outputs(self):
        pr, f = self.pr, self.f
        w0 = self.tree.dir_stats()["walked"]
        x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
        walked = self.tree.dir_stats()["walked"] - w0
        n = len(pr.scan)
        near, cnt = f.nearest(n)
        logs = b"".join(json.dumps({k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in lg.items()}).encode() for lg in f.pass_logs())
        return {"x": x.tobytes(), "P": P.tobytes(), "logs": logs, "nearest": near.tobytes(), "counts": cnt.tobytes(),
                "selected": f.selected(n).tobytes()}, walked

    def prepare(self):
        self.f.upload_scan(self.pr.scan)
        self.f.upload_state(self.pr.x_prior, self.pr.P_prior, self.pr.R)

    def times(self, steps):
        f = self.f
        return {"step_flushed_ms": f.time_resident(steps, flush_l2=True) / steps,
                "step_warm_ms": f.time_resident(steps, flush_l2=False) / steps,
                "search_flushed_ms": f.time_search_pass(steps, flush_l2=True) / steps,
                "search_warm_ms": f.time_search_pass(steps, flush_l2=False) / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old_lib")
    ap.add_argument("new_lib")
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, power = card()
    res = {"bench": "update_ab", "gpu": name, "power_limit": power, "old_lib": a.old_lib, "new_lib": a.new_lib,
           "rounds": a.rounds, "steps_per_call": a.steps,
           "timing": "CUDA events inside fl_filter_time_resident / fl_filter_time_search_pass, per step; old, new, old, new in every round",
           "workloads": {}}
    all_equal = True
    for wl in a.workloads.split(","):
        pr = synth.make_problem(wl)
        old, new = Run(a.old_lib, pr), Run(a.new_lib, pr)
        (oa, wa), (ob, wb) = old.outputs(), new.outputs()
        diff = [k for k in oa if oa[k] != ob[k]] + (["walked"] if wa != wb else [])
        all_equal &= not diff
        for r in (old, new):
            r.prepare()
            r.times(max(3, a.steps // 10))                 # warm-up
        ts = [[], [], [], []]
        for _ in range(a.rounds):
            for j, r in enumerate((old, new, old, new)):
                ts[j].append(r.times(a.steps))
        entry = {"scan_points": len(pr.scan), "map_points": len(pr.map_pts), "equal": not diff, "differs": diff,
                 "walked_per_update": [int(wa), int(wb)]}
        for key in ts[0][0]:
            m = [statistics.median(t[key] for t in ts[j]) for j in range(4)]
            o = statistics.median([t[key] for t in ts[0] + ts[2]])
            n = statistics.median([t[key] for t in ts[1] + ts[3]])
            entry[key] = {"old": o, "new": n, "new_over_old": n / o,
                          "old_repeat_spread": abs(m[0] - m[2]) / min(m[0], m[2]), "new_repeat_spread": abs(m[1] - m[3]) / min(m[1], m[3])}
        res["workloads"][wl] = entry
        print(json.dumps({wl: entry}), file=sys.stderr)
    res["all_equal"] = bool(all_equal)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")
    if not all_equal:
        raise SystemExit("update_ab: the two libraries' outputs differ")


if __name__ == "__main__":
    main()
