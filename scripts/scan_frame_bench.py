"""The scan's clouds in a frame on the device (fl_scan_frame_device), measured on:
  (a) the device form alone, by CUDA events around replays of a graph of 100 calls, for each (which, frame) on config-4 raw
      scans (the avia_stream_24k scene) of 20 000, 40 000 and 65 000 points and on synth.raw_frame's Ouster 64 x 1024 frame
      (65 536 rows), with the achieved bytes/s of n * 32 B (one float4 read, one written) + 208 B (the state); and, for
      comparison, --reps eager calls back to back from Python with a memset of the position before each (`_eager_us`), which
      the host's enqueue rate bounds;
  (b) one scan's CUDA-graph replay of upload -> undistort -> down-sample -> update -> map_incremental on config 4's map, with and
      without the three output calls of a shipped config (a memset of the publish positions, the dense world cloud, the dense
      IMU-frame cloud and the dense world cloud appended to an accumulation buffer), replays alternated in one run;
  (c) the host route those calls replace, by host clock: fl_scan_download of feats_undistort, the state's download, and the
      three transforms on the CPU (numpy, FP64, vectorised).
Writes profiles/h100_scan_frame_bench.json (or --out) with the card's name and power limit, read in the same run.

    python scripts/scan_frame_bench.py [--reps 500] [--out PATH]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fast_lio_b200 import api, synth  # noqa: E402
from preprocess_bench import card  # noqa: E402

NAMES = {api.FRAME_LIDAR: "lidar", api.FRAME_IMU: "imu", api.FRAME_WORLD: "world"}


def cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def qrot(q, v):
    qv = np.broadcast_to(q[:3], v.shape)
    uv = cross(qv, v)
    uv = uv + uv
    return (v + uv * q[3]) + cross(qv, uv)


def cpu_frames(cloud, x):
    """The three loops of a shipped config on the CPU: dense world, dense IMU frame, dense world again for pcl_wait_save."""
    p = cloud[:, :3].astype(np.float64)
    p_this = qrot(x[7:11], p) + x[11:14]
    w = np.empty_like(cloud); w[:, 3] = cloud[:, 3]; w[:, :3] = qrot(x[3:7], p_this) + x[0:3]
    b = np.empty_like(cloud); b[:, 3] = cloud[:, 3]; b[:, :3] = p_this
    s = np.empty_like(cloud); s[:, 3] = cloud[:, 3]; s[:, :3] = qrot(x[3:7], qrot(x[7:11], p) + x[11:14]) + x[0:3]
    return w, b, s


def kernel_bench(torch, pr, tree, reps):
    sources = [(f"config4_raw_{n // 1000}k", synth.make_raw_scan(pr.scene, n, synth.true_state(pr.cfg.lidar, 2), seed=500 + n))
               for n in (20_000, 40_000, 65_000)]
    o = synth.raw_frame("ouster", seed=4)
    oxyzi = np.ascontiguousarray(np.stack([o["x"], o["y"], o["z"], o["intensity"]], 1), np.float32)
    sources.append(("raw_frame_ouster64x1024", synth.RawScan(oxyzi, np.zeros(len(o), np.float32), np.zeros((0, 22)), pr.x_prior, None)))
    x = torch.from_numpy(pr.x_prior.copy()).cuda()
    out = {}
    for name, r in sources:
        n = len(r.xyzi)
        s = api.Scan(tree)
        s.reserve(n, max(len(r.imu_pose), 1))
        s.upload_device(torch.from_numpy(r.xyzi).cuda(), torch.from_numpy(r.offset_ms).cuda())
        if len(r.imu_pose):
            s.undistort_device(torch.from_numpy(r.imu_pose).cuda(), None, torch.from_numpy(r.x_end).cuda())
        n_down = int(s.voxel_downsample_device(0.5).cpu()[0])
        # G appends per graph into a buffer of G clouds, so each replay times G calls (both launches) and nothing else; the
        # position is zeroed before each replay, outside the events
        G = 100
        buf = torch.empty((G * n, 4), device="cuda")
        n_io = torch.zeros(1, dtype=torch.int32, device="cuda")
        st = torch.zeros(2, dtype=torch.int32, device="cuda")
        row = dict(n_rows=n, n_down=n_down, calls_per_graph=G)
        for which in (0, 1):
            rows = n if which == 0 else n_down
            for frame in (api.FRAME_LIDAR, api.FRAME_IMU, api.FRAME_WORLD):
                xs = None if frame == api.FRAME_LIDAR else x
                key = f"which{which}_{NAMES[frame]}"
                # (a1) eager, back to back from Python: bounded by the host's enqueue rate, kept for comparison
                for _ in range(20):
                    n_io.zero_(); s.frame_device(which, frame, xs, buf, n_io, st)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(reps):
                    n_io.zero_()
                    s.frame_device(which, frame, xs, buf, n_io, st)
                e1.record()
                torch.cuda.synchronize()
                row[f"{key}_eager_us"] = e0.elapsed_time(e1) * 1e3 / reps
                # (a) device time: G calls in one graph
                n_io.zero_()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for _ in range(G):
                        s.frame_device(which, frame, xs, buf, n_io, st)
                ts = []
                for _ in range(max(reps // G, 5)):
                    n_io.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); g.replay(); e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1) * 1e3 / G)
                assert int(st[0]) == 0 and int(n_io[0]) == G * rows, (st, n_io)
                us = float(np.median(ts))
                row[f"{key}_us"] = us
                row[f"{key}_GBps"] = (rows * 32 + 208) / (us * 1e-6) / 1e9
                del g
        out[name] = row
        print(name, row, flush=True)
    return out


def graph_bench(torch, pr, trees, reps):
    """(b) and (c) on one 40 000-point config-4 raw scan; every replay starts from the same prior and adds no map points."""
    r = synth.make_raw_scan(pr.scene, 40_000, synth.true_state(pr.cfg.lidar, 1), seed=77)
    n_max, leaf = len(r.xyzi), 0.5
    x0, P0 = torch.from_numpy(pr.x_prior.copy()).cuda(), torch.from_numpy(pr.P_prior.copy()).cuda()
    graphs, keep = {}, []
    for form, tree in zip(("chain", "chain_with_frames"), trees):
        fd = api.Esekf(tree, max_points=n_max, max_iter=pr.cfg.max_iter)
        sd = api.Scan(tree)
        sd.reserve(n_max, len(r.imu_pose))
        b = dict(xyzi=torch.from_numpy(r.xyzi).cuda(), t=torch.from_numpy(r.offset_ms).cuda(), n=torch.tensor([n_max], dtype=torch.int32, device="cuda"),
                 poses=torch.from_numpy(r.imu_pose).cuda(), n_pose=torch.tensor([len(r.imu_pose)], dtype=torch.int32, device="cuda"),
                 x_end=torch.from_numpy(r.x_end).cuda(), x=x0.clone(), P=P0.clone(), status=torch.zeros(2, dtype=torch.int32, device="cuda"),
                 out4=torch.zeros(4, dtype=torch.int32, device="cuda"), world=torch.empty((n_max, 4), device="cuda"),
                 imu=torch.empty((n_max, 4), device="cuda"), save=torch.empty((n_max * (reps + 50), 4), device="cuda"),
                 pub=torch.zeros(2, dtype=torch.int32, device="cuda"), n_save=torch.zeros(1, dtype=torch.int32, device="cuda"),
                 fst=torch.zeros((3, 2), dtype=torch.int32, device="cuda"))

        def chain(b=b, sd=sd, fd=fd, frames=form != "chain"):
            sd.upload_device(b["xyzi"], b["t"], b["n"], n_max)
            sd.undistort_device(b["poses"], b["n_pose"], b["x_end"])
            sd.voxel_downsample_device(leaf)
            sd.update_device(fd, b["x"], b["P"], pr.R, b["status"])
            fd.map_incremental_device(0.5, False, b["out4"])
            if frames:
                b["pub"].zero_()
                sd.frame_device(0, api.FRAME_WORLD, b["x"], b["world"], b["pub"][0:1], b["fst"][0])
                sd.frame_device(0, api.FRAME_IMU, b["x"], b["imu"], b["pub"][1:2], b["fst"][1])
                sd.frame_device(0, api.FRAME_WORLD, b["x"], b["save"], b["n_save"], b["fst"][2])

        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            chain()
        torch.cuda.synchronize()
        tree.maintain()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            chain()
        graphs[form] = (g, b)
        keep.append((fd, sd))
    ts = {k: [] for k in graphs}
    for i in range(reps):
        for form in (("chain", "chain_with_frames") if i % 2 == 0 else ("chain_with_frames", "chain")):
            g, b = graphs[form]
            b["x"].copy_(x0); b["P"].copy_(P0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record()
            torch.cuda.synchronize()
            ts[form].append(e0.elapsed_time(e1) * 1e3)
    b = graphs["chain_with_frames"][1]
    assert b["fst"][:, 0].abs().sum().item() == 0, b["fst"]
    res = {f"graph_{k}_us": dict(p50=float(np.median(v)), p10=float(np.percentile(v, 10)), p90=float(np.percentile(v, 90)))
           for k, v in ts.items()}
    res["graph_frames_added_p50_us"] = res["graph_chain_with_frames_us"]["p50"] - res["graph_chain_us"]["p50"]
    res["n_raw"] = n_max
    # (c) the host route: download feats_undistort and x, then the three loops on the CPU
    sd = keep[1][1]
    xd = graphs["chain_with_frames"][1]["x"]
    L = api.load()
    cloud = np.empty((n_max, 4), np.float32)
    tt = []
    for _ in range(max(reps // 5, 20)):
        t0 = time.perf_counter()
        n = L.fl_scan_download(sd.h, 0, cloud, n_max)
        x = xd.cpu().numpy()
        cpu_frames(cloud[:n], x)
        tt.append(time.perf_counter() - t0)
    res["host_route_us"] = dict(p50=float(np.median(tt) * 1e6), p90=float(np.percentile(tt, 90) * 1e6))
    print(res, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=500)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_scan_frame_bench.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("scan_frame_bench: no CUDA device (there is no CPU path)")
    pr = synth.make_problem("avia_stream_24k")
    trees = [api.KdTree(0, 0.5) for _ in range(2)]
    for t in trees:
        t.Build(pr.map_pts)
    rec = dict(card=card(), kernel=kernel_bench(torch, pr, trees[0], args.reps), graph_config4_40k=graph_bench(torch, pr, trees, args.reps // 2))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
