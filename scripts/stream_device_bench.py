"""The config-4 stream (avia_stream_24k: ~1 M-point map, 24 000-point scans, the sensor 0.1 m further each scan, no segment
step), update + map_incremental per scan, in three forms that do the same work per scan:
  (a) host forms: fl_filter_update + fl_filter_map_incremental, host clock around the two calls (both end in a synchronise);
  (b) device forms uncaptured: fl_filter_update_device + fl_filter_map_incremental_device, CUDA events around the two calls;
  (c) one CUDA-graph replay of the two captured calls per scan (the scan copied into the captured buffer first), CUDA events
      around the replay.
A fourth loop (a2) repeats (a) on a twin map and filter, untimed, to show how far two host-form runs agree with each other.
(b)'s enqueue is also timed by host clock.  It holds the launch overhead of every kernel of the two calls and, on the calls
where the host's headroom bound runs out, the wait of the settle for the stream; that wait is inside (b)'s CUDA-event time too.
The loops run over the same scans in alternating blocks of --block scans, each on its own map and filter.  (b) and (c)
read their statuses at the end of a block and call fl_map_maintain when one was due ((c) captures again when it reports a
layout change); the maintenance calls are counted and timed (host clock).  Reports per-scan p50 / p90 / p99 / max per loop and
whether the final x, P and the map's point set are equal across the three.  Prints one JSON line (also written to --out) with
the card's name and power limit, read in the same run.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_lio_b200 import api, synth  # noqa: E402
from semantics import sort_rows  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def pct(v):
    a = np.asarray(v) * 1e6
    return {k: round(float(x), 1) for k, x in zip(("p50_us", "p90_us", "p99_us", "max_us"), (*np.percentile(a, [50, 90, 99]), a.max()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=500)
    ap.add_argument("--block", type=int, default=25)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    pr = synth.make_problem("avia_stream_24k")
    scans = [synth.make_scan(pr.scene, pr.cfg.n_scan, synth.true_state(pr.cfg.lidar, s), seed=1000 + s) for s in range(args.scans)]
    n = min(len(s) for s in scans)
    scans = [np.ascontiguousarray(s[:n]) for s in scans]
    trees = [api.KdTree(0, 0.5) for _ in range(4)]          # (a), (b), (c), (a2)
    for t in trees:
        t.Build(pr.map_pts)
    filt = [api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter) for t in trees]
    eye = np.eye(23) * 1e-4
    # (a)
    xa, Pa = pr.x_prior.copy(), pr.P_prior.copy()
    xa2, Pa2 = pr.x_prior.copy(), pr.P_prior.copy()
    enqueue = []
    # (b), (c): state and scan in HBM
    st = torch.cuda.Stream()
    xs = [torch.from_numpy(pr.x_prior.copy()).cuda() for _ in range(2)]
    Ps = [torch.from_numpy(pr.P_prior.copy()).cuda() for _ in range(2)]
    sb = [torch.from_numpy(scans[0]).cuda() for _ in range(2)]
    out4 = [torch.zeros(4, dtype=torch.int32, device="cuda") for _ in range(2)]
    stat = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(2)]
    eye_d = torch.eye(23, dtype=torch.float64, device="cuda") * 1e-4
    times = {"a": [], "b": [], "c": []}
    maint = {"b": [], "c": []}
    recaptures = 0
    graph = None
    statuses = {"b": [], "c": []}
    first_diff = {"a2": None, "b": None, "c": None}            # the end of the first block after which x differed from (a)'s

    def step_device(k, scan_i):
        with torch.cuda.stream(st):
            Ps[k].add_(eye_d)
            sb[k].copy_(torch.from_numpy(scans[scan_i]).to("cuda", non_blocking=False))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            if k == 0:
                h0 = time.perf_counter()
                filt[1].update_device(sb[0], xs[0], Ps[0], pr.R, stat[0])
                filt[1].map_incremental_device(0.5, True, out4[0])
                enqueue.append(time.perf_counter() - h0)
            else:
                graph.replay()
            e1.record(st)
            o = out4[k].clone()
        return e0, e1, o

    def capture():
        nonlocal graph
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            filt[2].update_device(sb[1], xs[1], Ps[1], pr.R, stat[1])
            filt[2].map_incremental_device(0.5, True, out4[1])
        graph = g

    for b0 in range(0, args.scans, args.block):
        idx = range(b0, min(b0 + args.block, args.scans))
        for i in idx:                                                   # (a)
            Pa = Pa + eye
            t0 = time.perf_counter()
            xa, Pa, _ = filt[0].update_iterated_dyn_share_modified(scans[i], xa, Pa, pr.R)
            filt[0].map_incremental(0.5, True)
            times["a"].append(time.perf_counter() - t0)
        for i in idx:                                                   # (a2)
            Pa2 = Pa2 + eye
            xa2, Pa2, _ = filt[3].update_iterated_dyn_share_modified(scans[i], xa2, Pa2, pr.R)
            filt[3].map_incremental(0.5, True)
        if first_diff["a2"] is None and xa2.tobytes() != xa.tobytes():
            first_diff["a2"] = idx[-1]
        for k, name in ((0, "b"), (1, "c")):
            ev = []
            for i in idx:
                if k == 1 and graph is None:                            # first scan of (c): once outside capture, then capture
                    with torch.cuda.stream(st):
                        Ps[1].add_(eye_d)
                        sb[1].copy_(torch.from_numpy(scans[i]).cuda())
                        filt[2].update_device(sb[1], xs[1], Ps[1], pr.R, stat[1])
                        filt[2].map_incremental_device(0.5, True, out4[1])
                        statuses["c"].append(out4[1].clone())
                    capture()
                    continue
                e0, e1, o = step_device(k, i)
                ev.append((e0, e1))
                statuses[name].append(o)
            torch.cuda.synchronize()
            times[name] += [e0.elapsed_time(e1) * 1e-3 for e0, e1 in ev]
            if first_diff[name] is None and xs[k].cpu().numpy().tobytes() != xa.tobytes():
                first_diff[name] = idx[-1]
            due = any(int(s[3]) != 0 for s in torch.stack(statuses[name][-len(idx):]).cpu())
            if due:
                t0 = time.perf_counter()
                changed = trees[1 + k].maintain()
                maint[name].append(time.perf_counter() - t0)
                if k == 1 and changed:
                    capture()
                    recaptures += 1
    torch.cuda.synchronize()
    all_st = {k: torch.stack(v).cpu().numpy() for k, v in statuses.items()}
    refused = {k: int((v[:, 3] == -5).sum()) for k, v in all_st.items()}
    xb, Pb = xs[0].cpu().numpy(), Ps[0].cpu().numpy()
    xc, Pc = xs[1].cpu().numpy(), Ps[1].cpu().numpy()
    for t in trees:
        t.maintain()
    dig = [hashlib.sha256(sort_rows(t.flatten()).tobytes()).hexdigest()[:16] for t in trees]
    name, power = card()
    res = {
        "workload": "avia_stream_24k", "scans": args.scans, "points_per_scan": n, "block": args.block,
        "gpu": name, "power_limit": power,
        "a_host_forms": pct(times["a"]), "b_device_forms": pct(times["b"]), "c_graph_replay": pct(times["c"]),
        "maintenance_calls": {k: len(v) for k, v in maint.items()},
        "maintenance_ms": {k: [round(x * 1e3, 2) for x in v] for k, v in maint.items()},
        "recaptures_c": recaptures, "refused_calls": refused,
        "b_enqueue_host": pct(enqueue),
        "final_x_equal": {"ab": xa.tobytes() == xb.tobytes(), "ac": xa.tobytes() == xc.tobytes(), "bc": xb.tobytes() == xc.tobytes(),
                          "a_a2": xa.tobytes() == xa2.tobytes()},
        "final_P_equal": {"ab": Pa.tobytes() == Pb.tobytes(), "ac": Pa.tobytes() == Pc.tobytes(), "bc": Pb.tobytes() == Pc.tobytes()},
        "final_pos_max_abs_diff_m": {"ab": float(np.abs(xa[:3] - xb[:3]).max()), "ac": float(np.abs(xa[:3] - xc[:3]).max()),
                                     "a_a2": float(np.abs(xa[:3] - xa2[:3]).max())},
        "map_digest_equal": {"ab": dig[0] == dig[1], "ac": dig[0] == dig[2], "bc": dig[1] == dig[2], "a_a2": dig[0] == dig[3]},
        "first_state_difference_scan": first_diff, "validnum": [t.validnum() for t in trees],
        "map_stats": [t.stats() for t in trees], "dir_relists": [t.dir_stats()["relists"] for t in trees],
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
