"""Device-buffer map queries (fl_map_*_device) against their host-buffer forms, on the config-2 map.

Map: velodyne_30k_1m (1 M points) with its 30 000 scan points pushed through the prior pose (world frame).  Workloads: the
nearest search at k in {5, 8, 16, 32} x max_dist in {+inf, 1 m} (scripts/knn_k_bench.py) and the range workloads (a)-(d) of
scripts/range_bench.py.  Per workload: the device form's time by CUDA events on the caller's stream around each call (inputs
and outputs already in HBM, explicit workspace and cap, so no call synchronises), median of --reps launches after a warm-up,
alternating with host-clock timings of the host form (host buffers in and out) in the same process; result bytes over the
device time.  Also one CUDA-graph replay of a captured k = 5 nearest query plus the r = 1 m radius query.  Every device answer
is checked byte for byte against the host form before anything is reported.  Prints one JSON line (also written to --out)
with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_lio_b200 import api, synth  # noqa: E402
from refknn import world_queries  # noqa: E402

F = np.float32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def measure(host_fn, dev_fn, reps, warmup=3):
    """Median host-clock seconds of host_fn and median CUDA-event seconds of dev_fn, called alternately."""
    for _ in range(warmup):
        host_fn(); dev_fn()
    torch.cuda.synchronize()
    th, evs = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        host_fn()
        th.append(time.perf_counter() - t0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dev_fn()
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(th), statistics.median(a.elapsed_time(b) for a, b in evs) / 1e3


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


def host_range(t, kind, q):
    return t.Radius_Search(q[:, :3], q[:, 3]) if kind == "radius" else t.Box_Search(q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="velodyne_30k_1m")
    ap.add_argument("--reps", type=int, default=31)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("device_query_bench: no CUDA device (the device map has no CPU path)")
    name, power = card()
    pr = synth.make_problem(a.size)
    pts = pr.map_pts
    q = world_queries(pr)
    t = api.KdTree(0, 0.5); t.Build(pts)
    qd = torch.from_numpy(q).cuda()
    res = {"bench": "device_queries", "gpu": name, "power_limit": power, "map": a.size, "map_points": len(pts), "queries": len(q),
           "timing": "device: CUDA events around each call on the caller's stream; host: host clock of the synchronous call",
           "nearest": {}, "range": {}}
    all_match = True
    for k in (5, 8, 16, 32):
        for md in (np.inf, 1.0):
            want = t.Nearest_Search_K(q, k, md)
            got = [x.cpu().numpy() for x in t.nearest_search_device(qd, k, md)]
            match = all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
            all_match &= match
            t_host, t_dev = measure(lambda: t.Nearest_Search_K(q, k, md), lambda: t.nearest_search_device(qd, k, md), a.reps)
            nbytes = sum(w.nbytes for w in want)
            res["nearest"][f"k{k}_maxdist_{md:g}"] = {"k": k, "max_dist": float(md), "device_s": t_dev, "host_form_s": t_host,
                                                      "host_over_device": t_host / t_dev, "result_bytes": nbytes,
                                                      "device_result_GBps": nbytes / t_dev / 1e9, "matches_host_form": bool(match)}
    rng = np.random.default_rng(2)
    graph_in = {}
    for wname, (kind, rq) in range_workloads(pts, rng).items():
        off_h, pts_h = host_range(t, kind, rq)
        rd = torch.from_numpy(rq).cuda()
        call = t.radius_search_device if kind == "radius" else t.box_search_device
        o, p, s = call(rd)                                     # sizes the workspace and cap (reads the status once)
        npairs, total = int(s[1]), int(s[0])
        ws = t.range_workspace(len(rq), npairs)
        cap = max(total, 1)
        o, p, s = call(rd, cap=cap, workspace=ws)
        torch.cuda.synchronize()
        match = (np.array_equal(o.cpu().numpy(), off_h) and p[:total].cpu().numpy().tobytes() == pts_h.tobytes()
                 and int(s[0].item()) == len(pts_h))
        all_match &= match
        t_host, t_dev = measure(lambda: host_range(t, kind, rq), lambda: call(rd, cap=cap, workspace=ws), a.reps)
        nbytes = 16 * total + 4 * (len(rq) + 1)
        res["range"][wname] = {"queries": len(rq), "points": total, "pairs": npairs, "workspace_bytes": ws.numel(),
                               "device_s": t_dev, "host_form_s": t_host, "host_over_device": t_host / t_dev,
                               "result_bytes": nbytes, "device_result_GBps": nbytes / t_dev / 1e9, "matches_host_form": bool(match)}
        if wname.startswith("a_"):
            graph_in = dict(rd=rd, ws=ws, cap=cap, off_h=off_h, pts_h=pts_h)
    # one graph replay: k = 5 nearest over the 30 000 queries + the 30 000 one-metre spheres
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        t.nearest_search_device(qd, 5); t.radius_search_device(graph_in["rd"], cap=graph_in["cap"], workspace=graph_in["ws"])
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ka = t.nearest_search_device(qd, 5)
        ra = t.radius_search_device(graph_in["rd"], cap=graph_in["cap"], workspace=graph_in["ws"])
    g.replay()
    torch.cuda.synchronize()
    want = t.Nearest_Search_K(q, 5)
    gmatch = (all(x.cpu().numpy().tobytes() == w.tobytes() for x, w in zip(ka, want)) and np.array_equal(ra[0].cpu().numpy(), graph_in["off_h"])
              and ra[1][:len(graph_in["pts_h"])].cpu().numpy().tobytes() == graph_in["pts_h"].tobytes())
    all_match &= gmatch
    _, t_graph = measure(lambda: None, g.replay, a.reps)
    _, t_pair = measure(lambda: None, lambda: (t.nearest_search_device(qd, 5),
                                               t.radius_search_device(graph_in["rd"], cap=graph_in["cap"], workspace=graph_in["ws"])), a.reps)
    res["graph_k5_plus_radius_1m"] = {"replay_s": t_graph, "same_calls_uncaptured_s": t_pair, "matches_host_form": bool(gmatch)}
    res["all_match_host_form"] = bool(all_match)
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")
    if not all_match:
        raise SystemExit("device_query_bench: a device answer differs from the host form")


if __name__ == "__main__":
    main()
