"""Preprocess::process of S LiDAR frames: S single fl_preprocess_device calls against one fl_preprocess_batch_run_device, alone and
at the head of the fleet step (scan batch + fl_filter_update_scans_device).  Writes profiles/h100_preprocess_batch_bench.json (or
--out).

Workloads, S in {1, 4, 16, 64, 256}:
  avia       Livox CustomPoint frames of 2 000 - 24 000 points (random per slot)
  ouster     64 x 1024 ouster_ros::Point frames
  velo_yaw   32 x 1800 velodyne_ros::Point frames without point times (the ring sort and the scan by key)
Timings, CUDA events around graph replays, median of --reps after --warmup replays:
  (a) a graph of S fl_preprocess_device calls (one handle, each call into its own output region)
  (b) a graph of one fl_preprocess_batch_run_device
  fleet: on avia_2k_50k, raw Avia frames of 2 000 - 9 000 points -> (a) or (b), then one fl_scan_batch_run_device (no
         de-skew) and one fl_filter_update_scans_device from a prior near each frame's pose, each route captured into one graph
Equality flags: every slot's rows, offset times, out2 and last_ms of (b) equal those of (a); the fleet routes' x and P are
byte-equal.  The frames are a pool of 16 per workload, cycled over the slots.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast_lio_b200 import api, synth  # noqa: E402
from scan_batch_bench import capture, gpu_info, timed  # noqa: E402

# (lidar type, n_scans, time unit, frame maker)
WORKLOADS = {
    "avia": (api.LIDAR_AVIA, 6, api.TIME_NS, lambda rng, k: synth.raw_frame("avia", seed=k, n=int(rng.integers(2_000, 24_001)))),
    "ouster": (api.LIDAR_OUST64, 64, api.TIME_NS, lambda rng, k: synth.raw_frame("ouster", seed=k)),
    "velo_yaw": (api.LIDAR_VELO16, 32, api.TIME_US, lambda rng, k: synth.raw_frame("velodyne", seed=k, yaw0_deg=float(k * 37 % 360 - 180),
                                                                                  times=False)),
}


def avia_from_scan(r, seed):
    """A raw CustomPoint frame of a synthetic scan: a dummy row 0 (never output), tag 0x10, lines 0-5."""
    rng = np.random.default_rng(seed)
    n = len(r.xyzi)
    a = np.zeros(n + 1, api.CUSTOM_POINT)
    a["x"][1:], a["y"][1:], a["z"][1:] = r.xyzi[:, 0], r.xyzi[:, 1], r.xyzi[:, 2]
    a["offset_time"][1:] = (np.clip(r.offset_ms, 0, None) * 1e6).astype(np.uint32)
    a["reflectivity"][1:] = rng.integers(0, 256, n)
    a["tag"] = 0x10
    a["line"] = np.arange(n + 1) % 6
    return a


class Inputs:
    """S raw frames padded to n_max rows in one device tensor, their counts, and per-slot outputs for the single calls."""

    def __init__(self, torch, pool, S, n_max, step):
        self.raw = torch.zeros((S, n_max, step), dtype=torch.uint8, device="cuda")
        self.n = torch.zeros((S, 1), dtype=torch.int32, device="cuda")
        for s in range(S):
            a = pool[s % len(pool)]
            self.raw[s, :len(a)] = torch.from_numpy(a.view(np.uint8).reshape(len(a), -1)).cuda()
            self.n[s].fill_(len(a))
        self.xyzi = torch.zeros((S, n_max, 4), dtype=torch.float32, device="cuda")
        self.ms = torch.zeros((S, n_max), dtype=torch.float32, device="cuda")
        self.out2 = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
        self.last = torch.zeros((S, 1), dtype=torch.float32, device="cuda")
        self.table = api.preprocess_raws([(self.raw[s], self.n[s]) for s in range(S)])

    def singles(self, pp, S, n_max):
        for s in range(S):
            pp.process_device(self.raw[s], self.n[s], n_max, self.xyzi[s], self.ms[s], self.out2[s], self.last[s])


def same_outputs(torch, inp, pb, S):
    torch.cuda.synchronize()
    xyzi, ms, out2, last = (t.cpu().numpy() for t in pb.outputs())
    ax, am, ao, al = (t.cpu().numpy() for t in (inp.xyzi, inp.ms, inp.out2, inp.last))
    for s in range(S):
        k = int(ao[s, 0])
        if tuple(out2[s]) != tuple(ao[s]) or xyzi[s, :k].tobytes() != ax[s, :k].tobytes() or ms[s, :k].tobytes() != am[s, :k].tobytes() \
                or last[s].tobytes() != al[s, 0].tobytes():
            return False
    return True


def bench_frames(torch, args):
    rows = []
    for name, (t, n_scans, unit, make) in WORKLOADS.items():
        rng = np.random.default_rng(7)
        pool = [make(rng, 100 + k) for k in range(16)]
        n_max = max(len(a) for a in pool)
        for S in args.slots:
            pp = api.Preprocess(0, t, n_scans, 10, unit, 1, 0.5, n_raw_max=n_max)
            pb = api.PreprocessBatch(0, t, n_scans, 10, unit, 1, 0.5, n_slots_max=S, n_raw_max=n_max)
            inp = Inputs(torch, pool, S, n_max, pp.layout.itemsize)
            status = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
            ga = capture(torch, lambda: inp.singles(pp, S, n_max))
            gb = capture(torch, lambda: pb.run_device(inp.table, S, n_max, status))
            ta, tb = timed(torch, ga, args.warmup, args.reps), timed(torch, gb, args.warmup, args.reps)
            ga.replay(); gb.replay()
            eq = same_outputs(torch, inp, pb, S) and bool((status.cpu().numpy()[:, 0] == 0).all())
            kept = int(inp.out2[:, 0].sum().item())
            rows.append(dict(workload=name, S=S, n_max=n_max, raw_points=int(inp.n.sum().item()), kept=kept, singles_us=ta,
                             batch_us=tb, speedup=ta / tb, equal=eq))
            print(json.dumps(rows[-1]), flush=True)
            del ga, gb, inp, pb, pp
            torch.cuda.empty_cache()
    return rows


def bench_fleet(torch, args):
    pr = synth.make_problem("avia_2k_50k")
    rng = np.random.default_rng(11)
    pool = [avia_from_scan(synth.make_raw_scan(pr.scene, int(rng.integers(2_000, 9_001)), synth.true_state(pr.cfg.lidar, 3 * k), seed=500 + k),
                           k) for k in range(16)]
    priors = [synth.make_prior(synth.true_state(pr.cfg.lidar, 3 * k), seed=60 + k)[0] for k in range(16)]
    n_max = max(len(a) for a in pool)
    rows = []
    for S in args.slots:
        tree = api.KdTree(0, 0.5)
        tree.Build(pr.map_pts)
        f = api.Esekf(tree, max_points=n_max, max_iter=pr.cfg.max_iter, limit=pr.limit)
        f.reserve_batch(n_max)
        pp = api.Preprocess(0, api.LIDAR_AVIA, 6, 10, api.TIME_NS, 1, 0.5, n_raw_max=n_max)
        pb = api.PreprocessBatch(0, api.LIDAR_AVIA, 6, 10, api.TIME_NS, 1, 0.5, n_slots_max=S, n_raw_max=n_max)
        inp = Inputs(torch, pool, S, n_max, 20)
        sb_a, sb_b = api.ScanBatch(tree), api.ScanBatch(tree)
        sb_a.reserve(S, n_max, 0)
        sb_b.reserve(S, n_max, 0)
        raws_a = api.scan_raws([(inp.xyzi[s], inp.ms[s], inp.out2[s, :1]) for s in range(S)])
        raws_b = pb.scan_raws(n_slots=S)
        refs_a, m = sb_a.refs(1)
        refs_b, _ = sb_b.refs(1)
        # each robot's prior near the pose of the frame it gets (the pool is cycled over the robots)
        x0 = torch.from_numpy(np.stack([priors[s % len(pool)] for s in range(S)])).cuda()
        P0 = torch.from_numpy(np.stack([pr.P_prior] * S)).cuda()
        xa, Pa, xb, Pb = x0.clone(), P0.clone(), x0.clone(), P0.clone()
        st = [torch.zeros((S, 2), dtype=torch.int32, device="cuda") for _ in range(5)]

        def route_a():
            xa.copy_(x0); Pa.copy_(P0)
            inp.singles(pp, S, n_max)
            sb_a.run_device(raws_a, n_max, 0, 0.5, undistort=False, status=st[0])
            f.update_scans_device(refs_a[:S], xa, Pa, m, pr.R, st[1])

        def route_b():
            xb.copy_(x0); Pb.copy_(P0)
            pb.run_device(inp.table, S, n_max, st[2])
            sb_b.run_device(raws_b, n_max, 0, 0.5, undistort=False, status=st[3])
            f.update_scans_device(refs_b[:S], xb, Pb, m, pr.R, st[4])

        ga, gb = capture(torch, route_a), capture(torch, route_b)
        ta, tb = timed(torch, ga, args.warmup, args.reps), timed(torch, gb, args.warmup, args.reps)
        ga.replay(); gb.replay()
        torch.cuda.synchronize()
        eq = xa.cpu().numpy().tobytes() == xb.cpu().numpy().tobytes() and Pa.cpu().numpy().tobytes() == Pb.cpu().numpy().tobytes() \
            and all(bool((s.cpu().numpy()[:, 0] == 0).all()) for s in st)
        rows.append(dict(workload="fleet_avia_2k_50k", S=S, n_max=n_max, per_robot_preprocess_us=ta, batched_preprocess_us=tb,
                         speedup=ta / tb, equal=eq))
        print(json.dumps(rows[-1]), flush=True)
        del ga, gb
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[1, 4, 16, 64, 256])
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles",
                                                  "h100_preprocess_batch_bench.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    doc = dict(gpu=gpu_info(), warmup=args.warmup, reps=args.reps, frames=bench_frames(torch, args), fleet=bench_fleet(torch, args))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(doc, fh)
        fh.write("\n")


if __name__ == "__main__":
    main()
