"""Mint the golden vectors of tests/golden/ from the CPU oracle.

The reference ships no fixtures (SURVEY.md section 4), so the goldens are produced here from
(a) the reference's own unmodified ikd-Tree compiled into oracle/_ref -- kNN results -- and
(b) the CPU restatement in oracle/fastlio_oracle.cpp -- per-pass normal equations and final state.
Run from the repository root with the original project's sources present (oracle/_ref is built from them):

    python tests/golden/make_golden.py

The reference answers of tests/golden/ref/ (see tests/refcalls.py) are written by running the suite on a GPU with
oracle/_ref built and FASTLIO_RECORD_REF=<dir>, then copying <dir>/*.npz here.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from fast_lio_b200 import synth  # noqa: E402
from oracle import bind  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    assert bind.have_ref(), "oracle/_ref missing: build it here (make -C oracle) before minting goldens"
    for name in ("tiny", "small"):
        pr = synth.make_problem(name)
        tree = bind.KdTree(pr.map_pts, "reference")
        # kNN of the scan at the prior pose (what the first pass of h_share_model asks for)
        q = np.zeros((len(pr.scan), 4), dtype=np.float32)
        tmp = np.zeros(3, dtype=np.float32)
        for i in range(len(pr.scan)):
            bind.lib().oracle_transform_point(pr.x_prior, np.ascontiguousarray(pr.scan[i, :3]), tmp)
            q[i, :3] = tmp
        kp, kd, kc = tree.knn(q, 5)
        res = {}
        for extr in (0, 1):
            o = bind.update_iterated(tree, pr.scan, pr.x_prior, pr.P_prior, pr.cfg.max_iter, pr.R, pr.limit, extr)
            res[f"x_{extr}"] = o.x
            res[f"P_{extr}"] = o.P
            res[f"effct_{extr}"] = np.array([p["effct"] for p in o.passes], dtype=np.int32)
            res[f"searched_{extr}"] = np.array([p["searched"] for p in o.passes], dtype=np.int32)
            res[f"converged_{extr}"] = np.array([p["converged"] for p in o.passes], dtype=np.int32)
            res[f"HtH_{extr}"] = np.stack([p["HtH"] for p in o.passes])
            res[f"Hth_{extr}"] = np.stack([p["Hth"] for p in o.passes])
            res[f"res_sum_{extr}"] = np.array([p["res_sum"] for p in o.passes])
            res[f"selected_{extr}"] = o.selected
        # the inputs are regenerated from the seed at test time; a checksum guards the generator
        np.savez_compressed(os.path.join(OUT, f"{name}.npz"),
                            map_sum=np.float64(pr.map_pts.astype(np.float64).sum()),
                            scan_sum=np.float64(pr.scan.astype(np.float64).sum()),
                            x_prior=pr.x_prior, knn_d2=kd, knn_cnt=kc, knn_pts=kp, **res)
        print("wrote", name, {k: v.shape for k, v in res.items() if k.startswith("x_")})


if __name__ == "__main__":
    main()
