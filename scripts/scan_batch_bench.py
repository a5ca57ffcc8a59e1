"""The scan front end of S robots: S single front ends (fl_scan_t) against one fl_scan_batch_run_device, alone and in the whole
fleet step with fl_filter_update_scans_device.  Writes profiles/h100_scan_batch_bench.json (or --out).

Workloads, S in {1, 4, 16, 64, 256}:
  avia_2k_50k      raw scans of 2 000 - 9 000 points on the 50 000-point map
  avia_stream_24k  config-4 raw scans of 30 000 - 60 000 points on the 1 M-point map
Timings, CUDA events around graph replays, median of --reps after --warmup replays:
  (a) a graph of S single chains: fl_scan_upload_device -> undistort_device -> voxel_downsample_device per robot
  (b) a graph of one fl_scan_batch_run_device
  (c) the fleet step as a graph: (a) + fl_filter_update_scans_device over the S front ends' refs, against (b) + the same update
      over the batch's refs
Equality flags: every slot's status, feats_down_size and both clouds of (b) equal those of (a); the x and P of both (c) graphs
are byte-equal.  The raw scans are a pool of 16 per workload at distinct poses, cycled over the robots.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast_lio_b200 import api, synth  # noqa: E402

WORKLOADS = {"avia_2k_50k": (2_000, 9_000), "avia_stream_24k": (30_000, 60_000)}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(torch, g, warmup, reps):
    for _ in range(warmup):
        g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def capture(torch, fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                      # warm-up outside capture
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g


def run_workload(torch, name, S_list, warmup, reps, leaf=0.5):
    pr = synth.make_problem(name)
    lo, hi = WORKLOADS[name]
    n_max = hi
    rng = np.random.default_rng(5)
    pool = [synth.make_raw_scan(pr.scene, int(rng.integers(lo, hi + 1)), synth.true_state(pr.cfg.lidar, 3 * k), seed=100 + k,
                                imu_hz=float(rng.choice([100.0, 200.0]))) for k in range(16)]
    n_pose_max = max(len(r.imu_pose) for r in pool)
    tree = api.KdTree(0, 0.5)
    tree.Build(pr.map_pts)
    rows = []
    for S in S_list:
        raw = [pool[r % len(pool)] for r in range(S)]
        xyzi = torch.zeros((S, n_max, 4), dtype=torch.float32, device="cuda")
        tms = torch.zeros((S, n_max), dtype=torch.float32, device="cuda")
        n_d = torch.zeros((S, 1), dtype=torch.int32, device="cuda")
        poses = torch.zeros((S, n_pose_max, 22), dtype=torch.float64, device="cuda")
        np_d = torch.zeros((S, 1), dtype=torch.int32, device="cuda")
        xend = torch.zeros((S, 26), dtype=torch.float64, device="cuda")
        for r, s in enumerate(raw):
            n = len(s.xyzi)
            xyzi[r, :n] = torch.from_numpy(s.xyzi).cuda(); tms[r, :n] = torch.from_numpy(s.offset_ms).cuda(); n_d[r].fill_(n)
            poses[r, :len(s.imu_pose)] = torch.from_numpy(s.imu_pose).cuda(); np_d[r].fill_(len(s.imu_pose))
            xend[r].copy_(torch.from_numpy(s.x_end).cuda())
        fronts = [api.Scan(tree) for _ in range(S)]
        for f in fronts:
            f.reserve(n_max, n_pose_max)
        batch = api.ScanBatch(tree)
        batch.reserve(S, n_max, n_pose_max)
        raws = api.scan_raws([(xyzi[r], tms[r], n_d[r], poses[r], np_d[r], xend[r]) for r in range(S)])
        status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
        single_refs = api.scan_refs(fronts)
        batch_refs = batch.refs(1)[0][:S]
        filt = api.Esekf(tree, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
        filt.reserve_batch(n_max)
        x0 = np.stack([synth.make_prior(synth.true_state(pr.cfg.lidar, 3 * (r % len(pool))), seed=60 + r)[0] for r in range(S)])
        P0 = np.stack([pr.P_prior] * S)
        xa, Pa = torch.from_numpy(x0).cuda(), torch.from_numpy(P0).cuda()
        xb, Pb = xa.clone(), Pa.clone()
        ust = torch.zeros((S, 2), dtype=torch.int32, device="cuda")

        def chains():
            for r, f in enumerate(fronts):
                f.upload_device(xyzi[r], tms[r], n_d[r], n_max)
                f.undistort_device(poses[r], np_d[r], xend[r])
                f.voxel_downsample_device(leaf)

        def one_batch():
            batch.run_device(raws, n_max, n_pose_max, leaf, status=status)

        ga, gb = capture(torch, chains), capture(torch, one_batch)
        gca = capture(torch, lambda: (chains(), filt.update_scans_device(single_refs, xa, Pa, n_max, pr.R, ust)))
        gcb = capture(torch, lambda: (one_batch(), filt.update_scans_device(batch_refs, xb, Pb, n_max, pr.R, ust)))
        row = {"workload": name, "S": S, "n_max": n_max, "n_pose_max": n_pose_max,
               "points": int(sum(len(s.xyzi) for s in raw))}
        row["a_single_chains_us"] = timed(torch, ga, warmup, reps)
        row["b_batch_us"] = timed(torch, gb, warmup, reps)
        # equality of (b) with (a): both graphs replayed once more on the same inputs
        ga.replay(); gb.replay()
        torch.cuda.synchronize()
        st = status.cpu().numpy()
        eq = bool((st[:, 0] == 0).all())
        for r, f in enumerate(fronts):
            d1 = f.download(1)
            eq = eq and int(st[r, 1]) == len(d1) and batch.download(1, r).tobytes() == d1.tobytes()
            eq = eq and batch.download(0, r).tobytes() == f.download(0).tobytes()
        row["b_equals_a"] = eq
        row["c_fleet_single_us"] = timed(torch, gca, warmup, reps)
        row["c_fleet_batch_us"] = timed(torch, gcb, warmup, reps)
        # equality of the two fleet steps: one replay each from the same priors
        for x, P in ((xa, Pa), (xb, Pb)):
            x.copy_(torch.from_numpy(x0)); P.copy_(torch.from_numpy(P0))
        gca.replay(); torch.cuda.synchronize()
        ua = ust.cpu().numpy().copy()
        gcb.replay(); torch.cuda.synchronize()
        row["c_equal"] = bool(xa.cpu().numpy().tobytes() == xb.cpu().numpy().tobytes() and
                              Pa.cpu().numpy().tobytes() == Pb.cpu().numpy().tobytes() and (ua[:, 0] == 0).all() and
                              (ust.cpu().numpy() == ua).all())
        row["update_share_of_single_fleet"] = (row["c_fleet_single_us"] - row["a_single_chains_us"]) / row["c_fleet_single_us"]
        row["a_over_b"] = row["a_single_chains_us"] / row["b_batch_us"]
        row["c_single_over_batch"] = row["c_fleet_single_us"] / row["c_fleet_batch_us"]
        print(json.dumps(row), flush=True)
        rows.append(row)
        del ga, gb, gca, gcb, fronts, batch, filt
        torch.cuda.synchronize()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--S", default="1,4,16,64,256")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles",
                                                  "h100_scan_batch_bench.json"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("scan_batch_bench: no CUDA device (there is no CPU path)")
    info = gpu_info()
    t0 = time.time()
    rows = []
    for w in a.workloads.split(","):
        rows += run_workload(torch, w, [int(s) for s in a.S.split(",")], a.warmup, a.reps)
    out = {"gpu": info, "nvcc_arch": "sm_90a", "warmup": a.warmup, "reps": a.reps, "statistic": "median of CUDA-event times of graph "
           "replays, microseconds", "rows": rows, "all_equal": all(r["b_equals_a"] and r["c_equal"] for r in rows),
           "wall_s": time.time() - t0}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f)
    print(json.dumps({k: v for k, v in out.items() if k != "rows"}))


if __name__ == "__main__":
    main()
