"""Preprocess::process on realistic raw frames: the reference's CPU preprocess (oracle/_ref/libpreprocess_ref.so, on this host),
the host form fl_preprocess (host clock, copies included), the device form fl_preprocess_device (CUDA events), and one graph
replay of raw -> preprocess -> upload -> undistort -> down-sample -> update -> map_incremental against today's replay that
starts from fl_scan_upload_device.  Writes profiles/h100_preprocess_bench.json (or --out) with the card and its power limit.

    python scripts/preprocess_bench.py [--reps 200] [--out PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fast_lio_b200 import api, synth  # noqa: E402
from oracle import preprocess_ref  # noqa: E402

KINDS = [("avia_24k", api.LIDAR_AVIA, dict(kind="avia"), dict(n_scans=6, time_unit=api.TIME_NS)),
         ("velodyne32x1800_times", api.LIDAR_VELO16, dict(kind="velodyne"), dict(n_scans=32, time_unit=api.TIME_US)),
         ("velodyne32x1800_yaw", api.LIDAR_VELO16, dict(kind="velodyne", times=False), dict(n_scans=32, time_unit=api.TIME_US)),
         ("ouster64x1024", api.LIDAR_OUST64, dict(kind="ouster"), dict(n_scans=64, time_unit=api.TIME_NS)),
         ("marsim_20k", api.LIDAR_MARSIM, dict(kind="marsim"), dict(n_scans=1, time_unit=api.TIME_US))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def median_us(f, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts) * 1e6)


def frames_bench(torch, reps):
    out = {}
    for name, t, fk, cfg in KINDS:
        raw = synth.raw_frame(seed=1, **fk)
        pfn = 1
        pp = api.Preprocess(0, t, cfg["n_scans"], 10, cfg["time_unit"], pfn, 0.5, n_raw_max=len(raw))
        row = dict(n_raw=len(raw))
        if preprocess_ref.available():
            off = api.layout_offsets(raw.dtype, t)
            secs = [preprocess_ref.process(raw, off, t, cfg["n_scans"], 10, cfg["time_unit"], pfn, 0.5, timed=True)[2] for _ in range(20)]
            row["reference_cpu_us"] = float(np.median(secs) * 1e6)
        else:
            row["reference_cpu_us"] = None                         # not measured: oracle/_ref absent
        for _ in range(5):
            xyzi, ms, _ = pp.process(raw)
        row["n_kept"] = len(ms)
        row["host_form_us"] = median_us(lambda: pp.process(raw), reps // 4)
        d = torch.from_numpy(raw.view(np.uint8).copy()).cuda()
        n = torch.tensor([len(raw)], dtype=torch.int32, device="cuda")
        outs = [torch.empty((len(raw), 4), device="cuda"), torch.empty(len(raw), device="cuda"),
                torch.empty(2, dtype=torch.int32, device="cuda"), torch.empty(1, device="cuda")]
        for _ in range(10):
            pp.process_device(d, n, len(raw), *outs)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            pp.process_device(d, n, len(raw), *outs)
        e1.record()
        torch.cuda.synchronize()
        row["device_form_us"] = e0.elapsed_time(e1) * 1e3 / reps
        assert int(outs[2][0]) == len(ms)
        out[name] = row
        print(name, row, flush=True)
    return out


def graph_bench(torch, reps):
    """One scan's graph from raw Avia points against the graph that starts from the already-preprocessed cloud."""
    from test_gpu_frontend_device import stream_of_raw_scans, twins
    from test_gpu_preprocess import _avia_from_scan
    pr = synth.make_problem("small")
    n_max, leaf = 9_000, 0.5
    r = stream_of_raw_scans(pr, 1, n_max - 1)[0]
    a = _avia_from_scan(r, 100)
    res = {}
    for form in ("upload", "raw"):
        _, td = twins(pr)
        fd = api.Esekf(td, max_points=n_max, max_iter=3)
        sd = api.Scan(td)
        sd.reserve(n_max, 2)
        pp = api.Preprocess(0, api.LIDAR_AVIA, 6, 10, api.TIME_NS, 1, 0.5, n_raw_max=n_max)
        raw_d = torch.zeros((n_max, 20), dtype=torch.uint8, device="cuda")
        raw_d[:len(a)] = torch.from_numpy(a.view(np.uint8).reshape(len(a), -1)).cuda()
        n_d = torch.tensor([len(a)], dtype=torch.int32, device="cuda")
        xyzi = torch.zeros((n_max, 4), device="cuda")
        tms = torch.zeros(n_max, device="cuda")
        out2 = torch.zeros(2, dtype=torch.int32, device="cuda")
        last = torch.zeros(1, device="cuda")
        pp.process_device(raw_d, n_d, n_max, xyzi, tms, out2, last)
        torch.cuda.synchronize()
        poses = torch.zeros((2, 22), dtype=torch.float64, device="cuda")
        np_d = torch.zeros(1, dtype=torch.int32, device="cuda")
        xend = torch.from_numpy(pr.x_prior.copy()).cuda()
        x0, P0 = torch.from_numpy(pr.x_prior.copy()).cuda(), torch.from_numpy(pr.P_prior.copy()).cuda()
        xd, Pd = x0.clone(), P0.clone()
        status = torch.zeros(2, dtype=torch.int32, device="cuda")
        out4 = torch.zeros(4, dtype=torch.int32, device="cuda")

        def chain():
            if form == "raw":
                pp.process_device(raw_d, n_d, n_max, xyzi, tms, out2, last)
            sd.upload_device(xyzi, tms, out2[:1], n_max)
            sd.undistort_device(poses, np_d, xend)
            sd.voxel_downsample_device(leaf)
            sd.update_device(fd, xd, Pd, pr.R, status)
            fd.map_incremental_device(0.5, False, out4)       # no points added, so every replay does the same work

        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            chain()
        torch.cuda.synchronize()
        td.maintain()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            chain()
        ts = []
        for _ in range(reps // 4):
            xd.copy_(x0); Pd.copy_(P0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        res[f"graph_from_{form}_us"] = float(np.median(ts))
        res["n_raw"] = len(a)
        print(form, res, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_preprocess_bench.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench: no CUDA device (there is no CPU path)")
    rec = dict(card=card(), frames=frames_bench(torch, args.reps), graph_avia_small=graph_bench(torch, args.reps))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
