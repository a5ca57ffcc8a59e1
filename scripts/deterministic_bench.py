"""Cost of the deterministic map mode (fl_map_set_deterministic): mode off against mode on, in one run, alternating blocks.

    python scripts/deterministic_bench.py [--rounds N] [--steps K] [--out profiles/h100_deterministic_bench.json]

Workloads: the resident update (fl_filter_time_resident over K steps, L2 warm, per update) of config 1 (avia_2k_50k) and config 2
(velodyne_30k_1m); config 2's update captured into a CUDA graph (fl_filter_update_device) and replayed, CUDA events around K
replays; 30 000 Nearest_Search_K queries at k = 32 on config 2's 1 M-point map (wall time of the call, which ends in a device
synchronise).  Each round runs off, on, off, on; per measure the script reports each mode's median over the rounds and, as the
spread between repeated runs of the same code, the relative gap between the medians of each mode's first and second block.

The scan stream: --scans config-4 raw scans through the captured per-scan graph (tests/det_stream.py: segment, upload, de-skew,
down-sample, update, map_incremental), in the order off / on on a map from one Build, then off / on on a map of the same points
whose first half was built and the rest added (another slot layout).  Reported: the graph replay time per scan in each mode
(median and p90 over the scans of the Build maps), and for each mode whether the two layouts end with equal x, P and point set,
and how far apart their x and P end.  Prints one JSON line (also written to --out) with the card's name and power limit, read
in the same run.
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
import det_stream  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def make(pr, on, seed=1):
    t = api.KdTree(0, 0.5)
    t.set_deterministic(on)
    t.Build(pr.map_pts[np.random.default_rng(seed).permutation(len(pr.map_pts))])
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)
    f.upload_scan(pr.scan)
    f.upload_state(pr.x_prior, pr.P_prior, pr.R)
    return t, f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_deterministic_bench.json"))
    a = ap.parse_args()
    name, power = card()
    c1, c2 = synth.make_problem("avia_2k_50k"), synth.make_problem("velodyne_30k_1m")
    rng = np.random.default_rng(5)
    q = c2.map_pts[rng.choice(len(c2.map_pts), 30000, replace=False)].copy()
    q[:, :3] += rng.normal(0, 0.05, (len(q), 3)).astype(np.float32)
    objs = {on: {"c1": make(c1, on), "c2": make(c2, on)} for on in (False, True)}
    measures = {
        "config1_resident_update_ms": lambda on: objs[on]["c1"][1].time_resident(a.steps, flush_l2=False) / a.steps,
        "config2_resident_update_ms": lambda on: objs[on]["c2"][1].time_resident(a.steps, flush_l2=False) / a.steps,
        "nearest_search_k32_30k_on_1m_ms": None,
    }

    def knn(on):
        t = objs[on]["c2"][0]
        t0 = time.perf_counter()
        t.Nearest_Search_K(q, 32)
        return (time.perf_counter() - t0) * 1e3
    measures["nearest_search_k32_30k_on_1m_ms"] = knn
    import torch
    graphs = {}
    for on in (False, True):                          # config 2's device update, captured once per mode, on a filter of its own
        t = objs[on]["c2"][0]                         # (the resident timing's filter keeps its own launches)
        f = api.Esekf(t, max_points=len(c2.scan), max_iter=c2.cfg.max_iter, limit=c2.limit)
        g_st = torch.cuda.Stream()
        scan_d = torch.from_numpy(c2.scan).cuda()
        x_d, P_d = torch.from_numpy(c2.x_prior.copy()).cuda(), torch.from_numpy(c2.P_prior.copy()).cuda()
        with torch.cuda.stream(g_st):
            f.update_device(scan_d, x_d, P_d, c2.R)   # once outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=g_st):
            f.update_device(scan_d, x_d, P_d, c2.R)
        graphs[on] = (g, g_st, x_d, P_d, f, scan_d)          # the graph reads these buffers: they live as long as it does

    def replay(on):
        g, g_st, x_d, P_d = graphs[on][:4]
        with torch.cuda.stream(g_st):
            x_d.copy_(torch.from_numpy(c2.x_prior).cuda()); P_d.copy_(torch.from_numpy(c2.P_prior).cuda())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(g_st)
            for _ in range(a.steps):
                g.replay()
            e1.record(g_st)
        e1.synchronize()
        return e0.elapsed_time(e1) / a.steps
    measures["config2_update_graph_replay_ms"] = replay
    # outputs first: the two modes' k = 32 answers, for the record (they may differ only on tie rows)
    a_off, a_on = objs[False]["c2"][0].Nearest_Search_K(q, 32), objs[True]["c2"][0].Nearest_Search_K(q, 32)
    rows_differ = int((~np.all(a_off[0].reshape(len(q), -1) == a_on[0].reshape(len(q), -1), axis=1)).sum())
    for fn in measures.values():                                      # warm-up of every shape in both modes
        fn(False); fn(True)
    samples = {k: {False: [[], []], True: [[], []]} for k in measures}
    for _ in range(a.rounds):
        for blk in (0, 1):
            for on in (False, True):
                for k, fn in measures.items():
                    samples[k][on][blk].append(fn(on))
    res = {}
    for k in measures:
        med = {on: statistics.median(samples[k][on][0] + samples[k][on][1]) for on in (False, True)}
        spread = max(abs(statistics.median(samples[k][on][0]) - statistics.median(samples[k][on][1])) / med[on] for on in (False, True))
        res[k] = {"off": med[False], "on": med[True], "on_over_off": med[True] / med[False], "spread_same_code": spread}
    del graphs
    pr4, raws = det_stream.problem(a.scans)
    runs = {}
    for how in ("build", "build_add"):
        for on in (False, True):
            t = det_stream.build(pr4, how, on)
            x, P, w, times = det_stream.run_graph(pr4, raws, t, timed=True)
            runs[(how, on)] = (x, P, det_stream.flat_sorted(t), times)
            t.close()
    stream = {"scans": a.scans, "workload": "avia_stream_24k raw scans, 30k-60k points"}
    for on in (False, True):
        xa, Pa, fa, ta = runs[("build", on)]
        xb, Pb, fb, _ = runs[("build_add", on)]
        fa_s, fb_s = fa[np.lexsort(fa.T[::-1])], fb[np.lexsort(fb.T[::-1])]
        stream["on" if on else "off"] = {
            "graph_ms_per_scan_p50": float(np.median(ta)) * 1e3, "graph_ms_per_scan_p90": float(np.percentile(ta, 90)) * 1e3,
            "layouts_equal": {"x": xa.tobytes() == xb.tobytes(), "P": Pa.tobytes() == Pb.tobytes(),
                              "points": len(fa) == len(fb) and fa_s.tobytes() == fb_s.tobytes()},
            "max_abs_dx": float(np.abs(xa - xb).max()), "max_abs_dP": float(np.abs(Pa - Pb).max()),
            "validnum": [int(len(fa)), int(len(fb))]}
    stream["graph_on_over_off"] = stream["on"]["graph_ms_per_scan_p50"] / stream["off"]["graph_ms_per_scan_p50"]
    out = {"card": name, "power_limit": power, "rounds": a.rounds, "steps": a.steps, "measures": res,
           "knn_k32_rows_differing_between_modes": rows_differ, "config4_scan_graph": stream}
    line = json.dumps(out)
    print(line)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as fh:
        fh.write(line + "\n")


if __name__ == "__main__":
    main()
