"""The whole per-scan chain of laserMapping.cpp on the config-4 stream (avia_stream_24k: ~1 M-point map, the sensor 0.1 m further
each scan) from raw points of varying size: lasermap_fov_segment (Delete_Point_Boxes when the cube moves) -> upload -> de-skew ->
voxel down-sample (leaf 0.5) -> update -> map_incremental, in three forms that do the same work per scan:
  (a) host forms: fl_localmap_segment with pos_lid computed on the host, fl_scan_upload / undistort / voxel_downsample,
      fl_filter_update_scan, fl_filter_map_incremental, host clock around the six calls;
  (b) device forms uncaptured: fl_localmap_segment_device, fl_scan_*_device, fl_filter_update_scan_device,
      fl_filter_map_incremental_device on one stream, CUDA events around the six calls (the raw scan is copied into the device
      buffers first, outside the events);
  (c) one CUDA-graph replay of the six captured calls per scan (captured once with n_max), CUDA events around the replay.
The cube (--cube-len, --det-range: 6 m and 1 m by default, so that it slides every 13-14 scans) starts where the first scan
places it.  Each form runs on its own map, cube, filter and scan handle over the same scans.  (b) and (c) read their statuses at
the end of a block of --block scans and call fl_map_maintain when one was due ((c) captures again when it reports a layout
change).  Reports per-scan p50 / p90 / p99 / max per form, separately for the scans where the cube slid and those where it did
not, and whether the final x, P and the map's point set are equal across the three.  (a2) runs the host forms again on a twin
map, cube, filter and scan, untimed: whether (a) and (a2) agree tells the host forms' own run-to-run determinism apart from
a difference of the device forms.  Then the cost of the segment call on a
scan where the cube does not move: the graph of the six calls and the graph of the last five, captured on (c)'s handles and
replayed alternately on one scan.  Prints one JSON line (also written to --out) with the card's name and power limit, read in
the same run.
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fast_lio_b200 import api, synth  # noqa: E402
from semantics import sort_rows  # noqa: E402
from stream_device_bench import card, pct  # noqa: E402


def pos_lid(x):
    """state.pos + state.rot * state.offset_T_L_I (laserMapping.cpp:890) in the order of Eigen's _transformVector."""
    q, v = x[3:6], x[11:14]
    cross = lambda a, b: np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])   # noqa: E731
    uv = cross(q, v)
    uv = uv + uv
    return x[0:3] + ((v + uv * x[6]) + cross(q, uv))


def segment_cost(reps, chain, capture, graph, b, st):
    """The six-call graph and the five-call graph (no segment) of (c), replayed alternately on the last scan, whose state stays
    away from the cube's faces: the difference of their medians is what the segment call costs on a scan where nothing moves."""
    torch.cuda.synchronize()
    without = torch.cuda.CUDAGraph()
    with torch.cuda.graph(without, stream=st):
        chain(1, segment=False)
    t = {"with": [], "without": []}
    moved = 0
    for r in range(2 * reps):
        which = "with" if r % 2 == 0 else "without"
        with torch.cuda.stream(st):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            (graph if which == "with" else without).replay()
            e1.record(st)
        e1.synchronize()
        if which == "with":
            moved += int(b["seg3"][0].item()) > 0
        t[which].append(e0.elapsed_time(e1) * 1e-3)
    return {"with_segment": pct(t["with"]), "without_segment": pct(t["without"]), "reps": reps, "scans_where_it_moved": moved,
            "segment_us_p50": (float(np.median(t["with"])) - float(np.median(t["without"]))) * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--block", type=int, default=25)
    ap.add_argument("--n-min", type=int, default=30_000)
    ap.add_argument("--n-max", type=int, default=60_000)
    ap.add_argument("--leaf", type=float, default=0.5)
    ap.add_argument("--cube-len", type=float, default=6.0)
    ap.add_argument("--det-range", type=float, default=1.0)
    ap.add_argument("--ab-reps", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    pr = synth.make_problem("avia_stream_24k")
    rng = np.random.default_rng(7)
    raws = [synth.make_raw_scan(pr.scene, int(rng.integers(args.n_min, args.n_max + 1)), synth.true_state(pr.cfg.lidar, s),
                                seed=3000 + s, imu_hz=float(rng.choice([100.0, 200.0, 400.0]))) for s in range(args.scans)]
    n_max, leaf = args.n_max, args.leaf
    n_pose_max = max(len(r.imu_pose) for r in raws)
    trees = [api.KdTree(0, 0.5) for _ in range(3)]
    for t in trees:
        t.Build(pr.map_pts)
    filt = [api.Esekf(t, max_points=n_max, max_iter=pr.cfg.max_iter) for t in trees]
    scans = [api.Scan(t) for t in trees]
    cubes = [api.LocalMap(args.cube_len, args.det_range) for _ in trees]
    twin = api.KdTree(0, 0.5)                                   # (a2)
    twin.Build(pr.map_pts)
    twin_f, twin_s, twin_c = api.Esekf(twin, max_points=n_max, max_iter=pr.cfg.max_iter), api.Scan(twin), api.LocalMap(args.cube_len, args.det_range)
    for s in scans[1:]:
        s.reserve(n_max, n_pose_max)
    eye = np.eye(23) * 1e-4
    eye_d = torch.eye(23, dtype=torch.float64, device="cuda") * 1e-4
    st = torch.cuda.Stream()
    # device inputs of (b) and (c): the captured buffers
    buf = [dict(xyzi=torch.zeros((n_max, 4), dtype=torch.float32, device="cuda"), t=torch.zeros(n_max, dtype=torch.float32, device="cuda"),
                n=torch.zeros(1, dtype=torch.int32, device="cuda"), poses=torch.zeros((n_pose_max, 22), dtype=torch.float64, device="cuda"),
                n_pose=torch.zeros(1, dtype=torch.int32, device="cuda"), x_end=torch.zeros(26, dtype=torch.float64, device="cuda"),
                x=torch.from_numpy(pr.x_prior.copy()).cuda(), P=torch.from_numpy(pr.P_prior.copy()).cuda(),
                status=torch.zeros(2, dtype=torch.int32, device="cuda"), out4=torch.zeros(4, dtype=torch.int32, device="cuda"),
                seg3=torch.zeros(3, dtype=torch.int32, device="cuda"))
           for _ in range(2)]

    def fill(b, r):
        with torch.cuda.stream(st):
            b["xyzi"][:len(r.xyzi)] = torch.from_numpy(r.xyzi).cuda(); b["t"][:len(r.xyzi)] = torch.from_numpy(r.offset_ms).cuda()
            b["n"].fill_(len(r.xyzi)); b["poses"][:len(r.imu_pose)] = torch.from_numpy(r.imu_pose).cuda()
            b["n_pose"].fill_(len(r.imu_pose)); b["x_end"].copy_(torch.from_numpy(r.x_end).cuda()); b["P"].add_(eye_d)

    def chain(k, segment=True):
        b, s, f = buf[k], scans[1 + k], filt[1 + k]
        if segment:
            cubes[1 + k].segment_device(trees[1 + k], b["x"], b["seg3"], None, b["n"])
        s.upload_device(b["xyzi"], b["t"], b["n"], n_max)
        s.undistort_device(b["poses"], b["n_pose"], b["x_end"])
        s.voxel_downsample_device(leaf, b.get("n_out"))
        s.update_device(f, b["x"], b["P"], pr.R, b["status"])
        f.map_incremental_device(0.5, True, b["out4"])

    for b in buf:
        b["n_out"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    times = {"a": [], "b": [], "c": []}
    statuses = {"b": [], "c": []}
    seg_st = {"b": [], "c": []}
    slid = []
    maint = {"b": 0, "c": 0}
    recaptures = 0
    graph = None
    xa, Pa = pr.x_prior.copy(), pr.P_prior.copy()
    xa2, Pa2 = pr.x_prior.copy(), pr.P_prior.copy()

    def capture():
        nonlocal graph
        torch.cuda.synchronize()
        trees[2].maintain()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            chain(1)
        graph = g

    for b0 in range(0, args.scans, args.block):
        idx = range(b0, min(b0 + args.block, args.scans))
        for i in idx:                                                   # (a)
            r = raws[i]
            Pa = Pa + eye
            t0 = time.perf_counter()
            boxes, _ = cubes[0].segment(pos_lid(xa), trees[0])
            scans[0].upload(r.xyzi, r.offset_ms)
            scans[0].undistort(r.imu_pose, r.x_end)
            scans[0].voxel_downsample(leaf)
            xa, Pa, _ = scans[0].update(filt[0], xa, Pa, pr.R)
            filt[0].map_incremental(0.5, True)
            times["a"].append(time.perf_counter() - t0)
            slid.append(len(boxes) > 0)
            Pa2 = Pa2 + eye                                             # (a2), untimed
            twin_c.segment(pos_lid(xa2), twin)
            twin_s.upload(r.xyzi, r.offset_ms); twin_s.undistort(r.imu_pose, r.x_end); twin_s.voxel_downsample(leaf)
            xa2, Pa2, _ = twin_s.update(twin_f, xa2, Pa2, pr.R)
            twin_f.map_incremental(0.5, True)
        for k, name in ((0, "b"), (1, "c")):
            ev = []
            for i in idx:
                fill(buf[k], raws[i])
                if k == 1 and graph is None and i == 0:                 # first scan of (c): once outside capture, then capture
                    with torch.cuda.stream(st):
                        chain(1)
                        statuses["c"].append(buf[1]["out4"].clone())
                        seg_st["c"].append(buf[1]["seg3"].clone())
                    capture()
                    continue
                with torch.cuda.stream(st):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    if k == 0:
                        chain(0)
                    else:
                        graph.replay()
                    e1.record(st)
                    statuses[name].append(buf[k]["out4"].clone())
                    seg_st[name].append(buf[k]["seg3"].clone())
                ev.append((e0, e1))
            torch.cuda.synchronize()
            times[name] += [e0.elapsed_time(e1) * 1e-3 for e0, e1 in ev]
            if any(int(s[3]) != 0 for s in torch.stack(statuses[name][-len(idx):]).cpu()) or \
                    any(int(s[2]) != 0 for s in torch.stack(seg_st[name][-len(idx):]).cpu()):
                maint[name] += 1
                if trees[1 + k].maintain() and k == 1:
                    capture()
                    recaptures += 1
    torch.cuda.synchronize()
    all_st = {k: torch.stack(v).cpu().numpy() for k, v in statuses.items()}
    refused = {k: int((v[:, 3] == -5).sum()) for k, v in all_st.items()}
    all_seg = {k: torch.stack(v).cpu().numpy() for k, v in seg_st.items()}
    seg_equal = {k: bool(all(int(v[i, 0]) == 0 for i in range(len(v)) if not slid[i]) and
                         all(int(v[i, 0]) > 0 for i in range(len(v)) if slid[i])) for k, v in all_seg.items()}
    xb, Pb = buf[0]["x"].cpu().numpy(), buf[0]["P"].cpu().numpy()
    xc, Pc = buf[1]["x"].cpu().numpy(), buf[1]["P"].cpu().numpy()
    for t in trees + [twin]:
        t.maintain()
    dig = [hashlib.sha256(sort_rows(t.flatten()).tobytes()).hexdigest()[:16] for t in trees + [twin]]
    split = lambda ts, want: [t for t, s in zip(ts, slid) if s == want]      # noqa: E731
    valid = [t.validnum() for t in trees + [twin]]
    ab = segment_cost(args.ab_reps, chain, capture, graph, buf[1], st)
    name, power = card()
    res = {
        "workload": "avia_stream_24k raw scans", "scans": args.scans, "raw_points": [args.n_min, args.n_max], "n_max": n_max,
        "n_pose_max": n_pose_max, "leaf": leaf, "block": args.block, "gpu": name, "power_limit": power,
        "cube_len": args.cube_len, "det_range": args.det_range, "slides": int(sum(slid)),
        "a_host_forms": {"slide": pct(split(times["a"], True)), "no_slide": pct(split(times["a"], False))},
        "b_device_forms": {"slide": pct(split(times["b"], True)), "no_slide": pct(split(times["b"], False))},
        "c_graph_replay": {"slide": pct([t for t, s in zip(times["c"], slid[1:]) if s]),          # scan 0 ran uncaptured
                           "no_slide": pct([t for t, s in zip(times["c"], slid[1:]) if not s])},
        "segment_cost_no_slide": ab, "segment_slides_match_host": seg_equal,
        "maintenance_calls": maint, "recaptures_c": recaptures, "refused_calls": refused,
        "final_x_equal": {"ab": xa.tobytes() == xb.tobytes(), "ac": xa.tobytes() == xc.tobytes()},
        "final_P_equal": {"ab": Pa.tobytes() == Pb.tobytes(), "ac": Pa.tobytes() == Pc.tobytes()},
        "map_digest_equal": {"ab": dig[0] == dig[1], "ac": dig[0] == dig[2]},
        "host_forms_twin_a2_equal": {"x": xa.tobytes() == xa2.tobytes(), "P": Pa.tobytes() == Pa2.tobytes(), "map": dig[0] == dig[3]},
        "max_abs_dx": {"ab": float(np.abs(xa - xb).max()), "ac": float(np.abs(xa - xc).max()), "aa2": float(np.abs(xa - xa2).max())},
        "validnum": valid,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
