"""Tiny driver for ncu: builds one workload and runs a few resident updates."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast_lio_b200 import api, synth

name = sys.argv[1] if len(sys.argv) > 1 else "velodyne_30k_1m"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
solver = int(sys.argv[3]) if len(sys.argv) > 3 else 1
search = int(sys.argv[4]) if len(sys.argv) > 4 else -1
pr = synth.make_problem(name)
t = api.KdTree(0, 0.5)
t.Build(pr.map_pts)
f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, solver=solver, search=search,
              fused=int(sys.argv[5]) if len(sys.argv) > 5 else -1)
f.upload_scan(pr.scan)
f.upload_state(pr.x_prior, pr.P_prior, pr.R)
ms = f.time_resident(reps, flush_l2=True)
x, P, n = f.download_state()
print(f"{name}: {ms / reps:.3f} ms/scan, passes={n}, stats={t.stats()}")

import ctypes as C, numpy as np
L = api.load()
prof = (C.c_longlong * 16)()
L.fl_filter_debug_prof.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
# one more scan, then read the stamps of its last pass
f.time_resident(1, flush_l2=True)
L.fl_filter_debug_prof(f.h, prof)
p = np.array(list(prof), dtype=np.int64)
if f.fused():
    print("last-pass cycles (k_update solver block): prepare", p[8] - p[0], "wait for tickets", p[9] - p[8], "reduce(+exchange)", p[1] - p[9],
          "gain", p[4] - p[1], "dx+converge", p[6] - p[4], "pose boxplus", p[10] - p[6], "publish", p[5] - p[10], "after publication (log, covariance)", p[7] - p[5], "total", p[7] - p[0])
    if p[11] and p[2] and p[3]:
        # k_update_wave only (%globaltimer ns, comparable across SMs): the pass that ends the update
        print("last pass ns (k_update_wave): every partial row in -> publication visible", p[2] - p[11],
              "publication -> last worker block has it", p[3] - p[2])
else:
    print("last-pass cycles: prepare", p[8] - p[0], "wait", p[9] - p[8], "reduce", p[1] - p[9], "gain", p[4] - p[1],
          "dxu", p[5] - p[4], "boxplus", p[6] - p[5], "tail", p[7] - p[6], "total", p[7] - p[0])
