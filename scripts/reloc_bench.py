"""Relocalisation (fl_reloc_expand_grid_device + fl_filter_relocalize_device) against the batched update over every hypothesis.

Workloads: avia_2k_50k (config 1) and velodyne_30k_1m (config 2), extrinsic_est_en 0.  The prior is the truth moved by
(2.2 m, -1.3 m) and turned by 27 degrees of yaw about gravity; the grid is 9 x 9 x 1 x 36 around it (0.75 m steps over +-3 m,
2 degree steps over +-35 degrees: 2 916 hypotheses), every scan point screened with r_inlier = 0.2 m, min_effct = 100, and
keep in {16, 64}.  Per workload, timed with CUDA events on the caller's stream, median over --reps after --warmup:
  (a) the whole call: expansion + relocalisation;
  (b) one replay of a CUDA graph that captured (a);
  (c) fl_filter_update_batch_device over all 2 916 hypotheses, then the same ranking of their last passes on the host (the
      ranking is not timed).
The screen alone is k_reloc_screen's device time, read with torch.profiler in a run of its own.  Both routes' winners are
reported with their position and rotation error against the truth.  Before the line is written, each graph replay's outputs are
checked byte for byte against the uncaptured call.  Prints one JSON line (also written to --out) with the card's name and power
limit, read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fast_lio_b200 import api, synth  # noqa: E402

GRID_N = (9, 9, 1, 36)
GRID_STEP = (0.75, 0.75, 0.0, math.radians(2.0))
R_INLIER, MIN_EFFCT = 0.2, 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30)
        name, power, clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return name, power, clock
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})", "unknown", "unknown"


def event_median(call, reps, warmup):
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    evs = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in evs) / 1e3


def offset_prior(pr):
    x = pr.x_true.copy()
    x[0] += 2.2; x[1] -= 1.3
    u = -x[23:26] / np.linalg.norm(x[23:26])
    half = math.radians(27.0) / 2
    x[3:7] = synth.quat_mul(np.r_[u * math.sin(half), math.cos(half)], x[3:7])
    return x


def pose_error(x, x_true):
    dq = synth.quat_mul(np.r_[-x_true[3:6], x_true[6]], x[3:7])
    return {"dpos_m": float(np.linalg.norm(x[:3] - x_true[:3])),
            "drot_deg": float(np.degrees(2 * np.arcsin(min(1.0, float(np.linalg.norm(dq[:3]))))))}


def rank(status, effct, res_sum):
    """the winner of fl_filter_relocalize_device's rule over (status, last-pass effct, res_sum) rows, or -1"""
    best = -1
    for s in range(len(status)):
        if status[s] != 0 or effct[s] < MIN_EFFCT:
            continue
        ratio = res_sum[s] / effct[s]
        if best < 0 or effct[s] > effct[best] or (effct[s] == effct[best] and ratio < res_sum[best] / effct[best]):
            best = s
    return best


def screen_kernel_s(call, reps):
    from torch.profiler import ProfilerActivity, profile
    call(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    ts = [e.device_time_total for e in prof.events() if "k_reloc_screen" in e.name and e.device_type.name == "CUDA"]
    return statistics.median(ts) / 1e6 if ts else None


def workload(name, keeps, reps, warmup):
    pr = synth.make_problem(name)
    t = api.KdTree(0, 0.5); t.Build(pr.map_pts)
    n, H = len(pr.scan), int(np.prod(GRID_N))
    f = api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter, limit=pr.limit)
    f.reserve_reloc(n, H, max(keeps))
    fb = api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter, limit=pr.limit)
    fb.reserve_batch(n)
    sd, Pd, prior = torch.from_numpy(pr.scan).cuda(), torch.from_numpy(pr.P_prior).cuda(), torch.from_numpy(offset_prior(pr)).cuda()
    X = torch.empty((H, 26), dtype=torch.float64, device="cuda")
    g_ = api.RelocGrid((api.C.c_int * 4)(*GRID_N), (api.C.c_double * 4)(*GRID_STEP))
    out = {"scan_points": n, "map_points": len(pr.map_pts), "hypotheses": H, "stride": 1, "keep": {}}
    L = api.load()

    for keep in keeps:
        res = {}

        def call():
            assert L.fl_reloc_expand_grid_device(prior.data_ptr(), api.C.byref(g_), X.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
            res["r"] = f.relocalize_device(sd, X, Pd, keep, R_INLIER, MIN_EFFCT, stride=1, R=pr.R)

        call()
        want = [v.cpu().numpy().tobytes() for v in res["r"]]
        st4 = res["r"][2].cpu().numpy()
        t_call = event_median(call, reps, warmup)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            call()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        g.replay(); torch.cuda.synchronize()
        match = [v.cpu().numpy().tobytes() for v in res["r"]] == want
        t_graph = event_median(g.replay, reps, warmup)
        match = match and [v.cpu().numpy().tobytes() for v in res["r"]] == want
        del g
        t_screen = screen_kernel_s(call, max(5, reps // 4))
        out["keep"][str(keep)] = {"call_s": t_call, "graph_s": t_graph, "screen_kernel_s": t_screen, "graph_matches_call": match,
                                  "status": int(st4[0]), "winner": int(st4[1]), "effct": int(st4[2]), "inliers": int(st4[3]),
                                  "error": pose_error(np.frombuffer(want[0], np.float64), pr.x_true)}

    # (c) the batched update over every hypothesis
    xs, Ps = X.clone(), Pd.expand(H, 23, 23).contiguous()
    status = torch.zeros((H, 2), dtype=torch.int32, device="cuda")
    x0 = X.clone()
    lg = {}

    def batch():
        xs.copy_(x0); Ps.copy_(Pd.expand(H, 23, 23))
        lg["st"], lg["logs"] = fb.update_batch_device(sd, xs, Ps, pr.R, status, logs=True)

    t_batch = event_median(batch, max(3, reps // 10), 1)
    stb, logs = lg["st"].cpu().numpy(), lg["logs"].cpu().numpy()
    last = [api.decode_pass_logs(logs[h], int(stb[h][1]))[-1] if stb[h][1] > 0 else {"effct": 0, "res_sum": 0.0} for h in range(H)]
    w = rank(stb[:, 0], [l["effct"] for l in last], [l["res_sum"] for l in last])
    out["batch_all"] = {"batch_s": t_batch, "note": "includes resetting x and P on the stream", "winner": int(w),
                        "effct": int(last[w]["effct"]) if w >= 0 else 0,
                        "error": pose_error(xs[w].cpu().numpy(), pr.x_true) if w >= 0 else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--keeps", default="16,64")
    ap.add_argument("--workloads", default="avia_2k_50k,velodyne_30k_1m")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("reloc_bench: no CUDA device (the relocalisation has no CPU path)")
    name, power, clock = card()
    res = {"bench": "reloc", "gpu": name, "power_limit": power, "max_sm_clock": clock, "extrinsic_est_en": 0, "reps": a.reps,
           "warmup": a.warmup, "grid_n": GRID_N, "grid_step": GRID_STEP, "r_inlier": R_INLIER, "min_effct": MIN_EFFCT,
           "prior": "x_true + (2.2, -1.3, 0) m, turned 27 deg about gravity",
           "timing": "CUDA events on the caller's stream, median over reps: call = expansion + relocalisation, graph = its replay, "
                     "batch_all = fl_filter_update_batch_device over every hypothesis; screen_kernel_s = k_reloc_screen by torch.profiler",
           "workloads": {}}
    keeps = [int(k) for k in a.keeps.split(",")]
    for wl in a.workloads.split(","):
        res["workloads"][wl] = workload(wl, keeps, a.reps, a.warmup)
    res["graph_matches_call"] = all(k["graph_matches_call"] for w in res["workloads"].values() for k in w["keep"].values())
    txt = json.dumps(res)
    if not res["graph_matches_call"]:
        print(txt, file=sys.stderr)
        raise SystemExit("reloc_bench: a graph replay differs from the uncaptured call; no line written")
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fo:
            fo.write(txt + "\n")


if __name__ == "__main__":
    main()
