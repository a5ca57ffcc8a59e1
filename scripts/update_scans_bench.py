"""The batched update over many scans (fl_filter_update_scans_device) against the same (scan, prior) pairs run one
fl_filter_update_device call each.

Workloads: avia_2k_50k (2 000-point scans, 50 000-point map) and avia_stream_24k (24 000-point scans, 1 M-point map),
extrinsic_est_en 0, S in {1, 2, 8, 29, 64, 256} slots.  Slot s holds a scan of its own, synth.make_scan from the true state s
steps (0.1 m each) along the trajectory, and a prior from synth.make_prior around that state; nq_max is the workload's scan size.
Distinct scans touch different map lines, so the L2 reuse of fl_filter_update_batch_device's single shared scan is not there.
Per workload and S, all timed with CUDA events on the caller's stream, median over --reps repetitions after --warmup, the priors
copied back into x and P before the first event of each repetition:
  (a) S back-to-back fl_filter_update_device calls on one stream, one per slot;
  (b) one fl_filter_update_scans_device call;
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


def workload(name, sizes, reps, warmup):
    pr = synth.make_problem(name)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    n = len(pr.scan)
    mk = lambda: api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter, limit=pr.limit)  # noqa: E731
    fs, fb = mk(), mk()
    fb.reserve_batch(n)
    S_max = max(sizes)
    scans, xs0, Ps0 = [], [], []
    for s in range(S_max):
        xt = synth.true_state(pr.cfg.lidar, s)
        scans.append(synth.make_scan(pr.scene, n, xt, seed=20_000 + s))
        x, P = synth.make_prior(xt, seed=30_000 + s)
        xs0.append(x); Ps0.append(P)
    bodies = [torch.from_numpy(sc).cuda() for sc in scans]
    counts = torch.full((S_max,), n, dtype=torch.int32, device="cuda")
    refs_all = api.scan_refs([(bodies[s], counts[s:s + 1]) for s in range(S_max)])
    workers, slots, _ = fb.batch_plan(n, 1)
    out = {"scan_points": n, "map_points": len(pr.map_pts), "workers_per_slot": workers, "slots_per_wave": slots, "S": {}}
    for S in sorted(set(sizes)):
        x0, P0 = torch.from_numpy(np.stack(xs0[:S])).cuda(), torch.from_numpy(np.stack(Ps0[:S])).cuda()
        xs, Ps = x0.clone(), P0.clone()
        status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
        refs = refs_all[:S]

        def reset():
            xs.copy_(x0); Ps.copy_(P0); status.zero_()

        def singles():
            for s in range(S):
                fs.update_device(bodies[s], xs[s], Ps[s], pr.R, status[s])

        def scans_call():
            fb.update_scans_device(refs, xs, Ps, n, pr.R, status)

        def snap():
            torch.cuda.synchronize()
            return xs.cpu().numpy().tobytes(), Ps.cpu().numpy().tobytes(), status.cpu().numpy().tobytes()

        reset(); singles()
        want = snap()
        passes = status.cpu().numpy()[:, 1]
        ok_status = int((status.cpu().numpy()[:, 0] == 0).sum())
        t_a = event_median(reset, singles, reps, warmup)
        match = {"singles_timed": snap() == want}
        reset(); scans_call()
        match["scans"] = snap() == want
        t_b = event_median(reset, scans_call, reps, warmup)
        match["scans_timed"] = snap() == want
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            reset(); scans_call()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            scans_call()
        reset(); g.replay()
        match["graph"] = snap() == want
        t_c = event_median(reset, g.replay, reps, warmup)
        match["graph_timed"] = snap() == want
        waves = fb.batch_plan(n, S)[2]
        out["S"][str(S)] = {
            "waves": waves, "status_ok": ok_status, "passes_min": int(passes.min()), "passes_max": int(passes.max()),
            "singles_s": t_a, "scans_s": t_b, "graph_s": t_c,
            "singles_us_per_scan": t_a / S * 1e6, "scans_us_per_scan": t_b / S * 1e6, "graph_us_per_scan": t_c / S * 1e6,
            "scans_us_per_wave": t_b / waves * 1e6, "singles_over_scans": t_a / t_b, "singles_over_graph": t_a / t_c,
            "matches_singles": match, "all_match": all(match.values())}
        del g
    out["all_match"] = all(v["all_match"] for v in out["S"].values())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=31)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sizes", default="1,2,8,29,64,256", help="slot counts S")
    ap.add_argument("--workloads", default="avia_2k_50k,avia_stream_24k")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.reps < 21:
        raise SystemExit("update_scans_bench: at least 21 repetitions")
    if api.device_count() < 1:
        raise SystemExit("update_scans_bench: no CUDA device (the filter has no CPU path)")
    name, power, clock = card()
    res = {"bench": "update_scans", "gpu": name, "power_limit": power, "max_sm_clock": clock, "extrinsic_est_en": 0, "reps": a.reps,
           "warmup": a.warmup,
           "timing": "CUDA events on the caller's stream, median over reps; (a) S back-to-back fl_filter_update_device calls, "
                     "(b) one fl_filter_update_scans_device call, (c) one graph replay of (b); priors reset outside the events",
           "scans": "slot s: synth.make_scan(scene, n, true_state(lidar, s), seed=20000 + s), all n rows; "
                    "prior synth.make_prior(true_state(lidar, s), seed=30000 + s)",
           "workloads": {}}
    sizes = [int(s) for s in a.sizes.split(",")]
    for wl in a.workloads.split(","):
        res["workloads"][wl] = workload(wl, sizes, a.reps, a.warmup)
    res["all_match_singles"] = all(w["all_match"] for w in res["workloads"].values())
    txt = json.dumps(res)
    if not res["all_match_singles"]:
        print(txt, file=sys.stderr)
        raise SystemExit("update_scans_bench: a slot's result differs from the single updates; no line written")
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
