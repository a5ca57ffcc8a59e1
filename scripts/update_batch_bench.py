"""The batched update (fl_filter_update_batch_device) against the same hypotheses run one fl_filter_update_device call each.

Workloads: avia_2k_50k (config 1) and velodyne_30k_1m (config 2), extrinsic_est_en 0, H in {1, 8, one full wave, 64, 256}
hypotheses.  The priors come from synth.make_prior with distinct seeds and a spread of 1 m and 2 degrees (standard deviations)
around the truth.  Per workload and H, all timed with CUDA events on the caller's stream, median over --reps repetitions after
--warmup, the priors copied back into x and P before the first event of each repetition:
  (a) H back-to-back fl_filter_update_device calls on one stream, one per hypothesis;
  (b) one fl_filter_update_batch_device call;
  (c) one replay of a CUDA graph that captured (b).
Before the line is written, the x, P and status of (b) and (c), of the first and of the timed runs, are checked byte for byte
against (a).  Prints one JSON line (also written to --out) with the card's name and power limit, read in the same run.
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

from fast_lio_b200 import api, synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30)
        name, power, clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power, clock
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown", "unknown"


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


def priors(pr, H):
    xs, Ps = [], []
    for h in range(H):
        x, P = synth.make_prior(pr.x_true, seed=10_000 + h, pos_sigma=1.0, rot_sigma_deg=2.0)
        xs.append(x); Ps.append(P)
    return np.stack(xs), np.stack(Ps)


def workload(name, hyps, reps, warmup):
    pr = synth.make_problem(name)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    mk = lambda: api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)  # noqa: E731
    fs, fb = mk(), mk()
    n = len(pr.scan)
    fb.reserve_batch(n)
    workers, slots, _ = fb.batch_plan(n, 1)
    sd = torch.from_numpy(pr.scan).cuda()
    out = {"scan_points": n, "map_points": len(pr.map_pts), "workers_per_hypothesis": workers, "hypotheses_per_wave": slots, "H": {}}
    for H in sorted(set(h if h > 0 else slots for h in hyps)):
        X, P = priors(pr, H)
        x0, P0 = torch.from_numpy(X).cuda(), torch.from_numpy(P).cuda()
        xs, Ps = x0.clone(), P0.clone()
        status = torch.zeros((H, 2), dtype=torch.int32, device="cuda")

        def reset():
            xs.copy_(x0); Ps.copy_(P0); status.zero_()

        def singles():
            for h in range(H):
                fs.update_device(sd, xs[h], Ps[h], pr.R, status[h])

        def snap():
            torch.cuda.synchronize()
            return xs.cpu().numpy().tobytes(), Ps.cpu().numpy().tobytes(), status.cpu().numpy().tobytes()

        reset(); singles()
        want = snap()
        passes = status.cpu().numpy()[:, 1]
        ok_status = int((status.cpu().numpy()[:, 0] == 0).sum())
        t_a = event_median(reset, singles, reps, warmup)
        match = {"singles_timed": snap() == want}
        reset(); fb.update_batch_device(sd, xs, Ps, pr.R, status)
        match["batch"] = snap() == want
        t_b = event_median(reset, lambda: fb.update_batch_device(sd, xs, Ps, pr.R, status), reps, warmup)
        match["batch_timed"] = snap() == want
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            reset(); fb.update_batch_device(sd, xs, Ps, pr.R, status)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fb.update_batch_device(sd, xs, Ps, pr.R, status)
        reset(); g.replay()
        match["graph"] = snap() == want
        t_c = event_median(reset, g.replay, reps, warmup)
        match["graph_timed"] = snap() == want
        waves = fb.batch_plan(n, H)[2]
        out["H"][str(H)] = {
            "waves": waves, "status_ok": ok_status, "passes_min": int(passes.min()), "passes_max": int(passes.max()),
            "singles_s": t_a, "batch_s": t_b, "graph_s": t_c,
            "singles_us_per_hyp": t_a / H * 1e6, "batch_us_per_hyp": t_b / H * 1e6, "graph_us_per_hyp": t_c / H * 1e6,
            "batch_us_per_wave": t_b / waves * 1e6, "singles_over_batch": t_a / t_b, "singles_over_graph": t_a / t_c,
            "matches_singles": match, "all_match": all(match.values())}
        del g
    out["all_match"] = all(v["all_match"] for v in out["H"].values())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=51)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--hyps", default="1,8,0,64,256", help="hypothesis counts; 0 = one full wave")
    ap.add_argument("--workloads", default="avia_2k_50k,velodyne_30k_1m")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.reps < 51:
        raise SystemExit("update_batch_bench: at least 51 repetitions")
    if api.device_count() < 1:
        raise SystemExit("update_batch_bench: no CUDA device (the filter has no CPU path)")
    name, power, clock = card()
    res = {"bench": "update_batch", "gpu": name, "power_limit": power, "max_sm_clock": clock, "extrinsic_est_en": 0, "reps": a.reps,
           "warmup": a.warmup,
           "timing": "CUDA events on the caller's stream, median over reps; (a) H back-to-back fl_filter_update_device calls, "
                     "(b) one fl_filter_update_batch_device call, (c) one graph replay of (b); priors reset outside the events",
           "priors": "synth.make_prior(x_true, seed=10000 + h, pos_sigma=1.0 m, rot_sigma_deg=2.0)",
           "workloads": {}}
    hyps = [int(h) for h in a.hyps.split(",")]
    for wl in a.workloads.split(","):
        res["workloads"][wl] = workload(wl, hyps, a.reps, a.warmup)
    res["all_match_singles"] = all(w["all_match"] for w in res["workloads"].values())
    txt = json.dumps(res)
    if not res["all_match_singles"]:
        print(txt, file=sys.stderr)
        raise SystemExit("update_batch_bench: a batch result differs from the single updates; no line written")
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
