"""The device-buffer update (fl_filter_update_device) against the host-buffer fl_filter_update.

Workloads: avia_2k_50k (config 1) and velodyne_30k_1m (config 2), extrinsic_est_en 0.  Per workload:
  - host form: fl_filter_update with host buffers, called from native code (fl_filter_time_e2e with one repetition), host
    clock, median;
  - device form: CUDA events around one fl_filter_update_device call on the caller's stream (scan, x, P and status already in
    HBM; the prior is copied back into x and P before the first event), median;
  - one graph replay of the captured update, and one of the update plus a k = 5 nearest_search_device over the scan's world
    points, timed the same way;
  - for context, the resident update (fl_filter_time_resident, warm L2, no copies at all), mean over the same repetitions.
Every device result (x, P, status, and the nearest search in the graph) is checked byte for byte against the host form before
the line is written.  Prints one JSON line (also written to --out) with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_lio_b200 import api, synth  # noqa: E402
from refknn import world_queries  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown"


def event_median(reset, call, reps, warmup):
    """Median CUDA-event seconds of call(), each preceded (outside the events) by reset() on the same stream."""
    for _ in range(warmup):
        reset(); call()
    torch.cuda.synchronize()
    evs = []
    for _ in range(reps):
        reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in evs) / 1e3


def workload(name, reps, warmup):
    pr = synth.make_problem(name)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    mk = lambda: api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)  # noqa: E731
    fh, fd = mk(), mk()
    xh, Ph, _ = fh.update_iterated_dyn_share_modified(pr.scan, pr.x_prior, pr.P_prior, pr.R)
    n_pass = fh.download_state()[2]
    # host form, from native code: one fl_filter_update per sample
    for _ in range(warmup):
        fh.time_e2e(pr.scan, pr.x_prior, pr.P_prior, pr.R, 1)
    t_host = statistics.median(fh.time_e2e(pr.scan, pr.x_prior, pr.P_prior, pr.R, 1)[0] for _ in range(reps))
    # resident, for context
    fh.upload_scan(pr.scan); fh.upload_state(pr.x_prior, pr.P_prior, pr.R)
    fh.time_resident(warmup, flush_l2=False)
    t_res = fh.time_resident(reps, flush_l2=False) / reps / 1e3

    x0, P0 = torch.from_numpy(pr.x_prior).cuda(), torch.from_numpy(pr.P_prior).cuda()
    sd = torch.from_numpy(pr.scan).cuda()
    qd = torch.from_numpy(world_queries(pr)).cuda()
    xs, Ps = x0.clone(), P0.clone()
    status = torch.zeros(2, dtype=torch.int32, device="cuda")

    def reset():
        xs.copy_(x0); Ps.copy_(P0)

    def same():
        torch.cuda.synchronize()
        return (xs.cpu().numpy().tobytes() == xh.tobytes() and Ps.cpu().numpy().tobytes() == Ph.tobytes()
                and status.cpu().tolist() == [0, n_pass])

    reset(); fd.update_device(sd, xs, Ps, pr.R, status)
    match = {"device": same()}
    t_dev = event_median(reset, lambda: fd.update_device(sd, xs, Ps, pr.R, status), reps, warmup)
    match["device_timed"] = same()
    # graphs (warmed up on a side stream, captured, then replayed on the current stream)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        reset(); fd.update_device(sd, xs, Ps, pr.R, status); t.nearest_search_device(qd, 5)
    torch.cuda.current_stream().wait_stream(side)
    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1):
        fd.update_device(sd, xs, Ps, pr.R, status)
    with torch.cuda.graph(g2):
        fd.update_device(sd, xs, Ps, pr.R, status)
        nn = t.nearest_search_device(qd, 5)
    reset(); g1.replay()
    match["graph_update"] = same()
    t_g1 = event_median(reset, g1.replay, reps, warmup)
    match["graph_update_timed"] = same()
    reset(); g2.replay()
    want_nn = t.Nearest_Search_K(qd.cpu().numpy(), 5)
    match["graph_update_knn5"] = same() and all(a.cpu().numpy().tobytes() == w.tobytes() for a, w in zip(nn, want_nn))
    t_g2 = event_median(reset, g2.replay, reps, warmup)
    match["graph_update_knn5_timed"] = same()
    return {"scan_points": len(pr.scan), "map_points": len(pr.map_pts), "passes": n_pass,
            "host_form_s": t_host, "device_form_s": t_dev, "graph_update_s": t_g1, "graph_update_plus_knn5_s": t_g2,
            "resident_warm_mean_s": t_res, "host_over_device": t_host / t_dev,
            "matches_host_form": match, "all_match": all(match.values())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=201)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("filter_device_bench: no CUDA device (the filter has no CPU path)")
    name, power = card()
    res = {"bench": "filter_device", "gpu": name, "power_limit": power, "extrinsic_est_en": 0, "reps": a.reps,
           "timing": "device forms: CUDA events around one call / replay on the caller's stream, median; host form: host clock "
                     "around one native fl_filter_update, median; resident: fl_filter_time_resident, warm L2, mean",
           "workloads": {}}
    for wl in ("avia_2k_50k", "velodyne_30k_1m"):
        res["workloads"][wl] = workload(wl, a.reps, a.warmup)
    res["all_match_host_form"] = all(w["all_match"] for w in res["workloads"].values())
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")
    if not res["all_match_host_form"]:
        raise SystemExit("filter_device_bench: a device result differs from the host form")


if __name__ == "__main__":
    main()
