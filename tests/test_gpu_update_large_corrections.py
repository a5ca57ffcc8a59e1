"""The update driven through the exact branches of lie.cuh by large prior errors, against the CPU oracle.

The default priors move rotation by a fraction of a degree, so every pass stays on the series branches and the S2 congruence
is nearly the identity.  Here the prior of the "small" scene carries a roll / pitch error of ~14 degrees (the walls and the
ground pin both angles, so the filter corrects most of it within its passes), a gravity block with variance 1e-2 coupled to
rotation, or an offset_R_L_I error with extrinsic estimation on.  Each case asserts from its own pass logs that a pass's
x [-] x_prop reached its branch: rotation above 0.1 rad (so3_log_exact) or 0.2 rad (A_matrix_exact, cos_sinc_exact of
the boxplus), gravity above 0.05 rad.

Error values (measured with the oracle; the filter's largest x [-] x_prior over the passes before the last):
  rot    rot_err_deg=(10, 10, 0)                                           rotation 0.214 rad
  grav   rot_err_deg=(9, 9, 0), grav_var=1e-2, grav_rot_corr=0.9, grav_deg=2   rotation 0.153, gravity 0.062 rad
  extr   rot_err_deg=(10, 10, 0), offr_deg=3, extrinsic_est_en               rotation 0.114 rad
"""
import numpy as np
import pytest

from fast_lio_b200 import api, synth
from oracle import bind
from refcalls import RefTree

pytestmark = pytest.mark.gpu

CASES = {
    "rot": (dict(rot_err_deg=(10.0, 10.0, 0.0)), 0, dict(rot=0.2)),
    "grav": (dict(rot_err_deg=(9.0, 9.0, 0.0), grav_var=1e-2, grav_rot_corr=0.9, grav_deg=2.0), 0, dict(rot=0.1, grav=0.05)),
    "extr": (dict(rot_err_deg=(10.0, 10.0, 0.0), offr_deg=3.0), 1, dict(rot=0.1)),
}


def problem(problems, case):
    pr = problems("small")
    opts, extr, _ = CASES[case]
    x, P = synth.make_prior(pr.x_true, seed=pr.cfg.seed + 2, **opts)
    return pr, x, P, extr


def reference(problems, case):
    pr, x, P, extr = problem(problems, case)
    return RefTree(f"update_large_{case}", pr.map_pts).update_iterated(pr.scan, x, P, pr.cfg.max_iter, pr.R, pr.limit, extr)


def boxminus(a, b):
    r = np.zeros(23)
    bind.lib().oracle_state_boxminus(np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64), r)
    return r


def run_gpu(problems, case, form):
    pr, x, P, extr = problem(problems, case)
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    solver, fused = {"solver1": (1, -1), "solver0": (0, -1), "split": (1, 0), "device": (1, -1)}[form]
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr),
                  solver=solver, fused=fused)
    if form == "device":
        import torch
        xd = torch.from_numpy(x.copy()).cuda()
        Pd = torch.from_numpy(P.copy()).cuda()
        st = f.update_device(torch.from_numpy(np.ascontiguousarray(pr.scan)).cuda(), xd, Pd, pr.R)
        torch.cuda.synchronize()
        assert int(st[0].item()) == 0
        return xd.cpu().numpy(), Pd.cpu().numpy(), f.pass_logs()
    xo, Po, _ = f.update_iterated_dyn_share_modified(pr.scan, x, P, pr.R)
    return xo, Po, f.pass_logs()


@pytest.mark.parametrize("form", ["solver1", "solver0", "split", "device"])
@pytest.mark.parametrize("case", list(CASES))
def test_large_correction_matches_oracle(problems, case, form):
    o = reference(problems, case)
    pr, x0, P0, _ = problem(problems, case)
    x, P, logs = run_gpu(problems, case, form)
    assert len(logs) == len(o.passes)
    for lg, op in zip(logs, o.passes):
        assert (lg["searched"], lg["effct"], lg["converged"], lg["valid"]) == (op["searched"], op["effct"], op["converged"], op["valid"])
        assert np.allclose(lg["HtH"], op["HtH"], rtol=1e-9, atol=1e-9 * np.abs(op["HtH"]).max())
        assert np.allclose(lg["Hth"], op["Hth"], rtol=1e-9, atol=1e-9 * np.abs(op["Hth"]).max())
        assert np.abs(lg["x_after"] - op["x_after"]).max() < 1e-6
    assert np.abs(x - o.x).max() < 1e-6
    # the normal equations agree to ~n eps (1e-13) relative: different summation orders.  The update carries that through
    # P with at most kappa(P) amplification per pass; 1e-11 kappa(P) leaves a factor 100 for the passes
    scale = np.sqrt(np.outer(np.diag(o.P), np.diag(o.P)))
    assert (np.abs(P - o.P) / scale).max() <= 1e-11 * np.linalg.cond(P0)
    # the pass that followed the largest correction ran its x [-] x_prop on the exact branches
    want = CASES[case][2]
    d = [boxminus(lg["x_after"], x0) for lg in logs[:-1]]
    assert max(np.linalg.norm(v[3:6]) for v in d) > want["rot"]
    if "grav" in want:
        assert max(np.linalg.norm(v[21:23]) for v in d) > want["grav"]


@pytest.mark.parametrize("case", list(CASES))
def test_device_buffer_form_equals_host_form(problems, case):
    xh, Ph, _ = run_gpu(problems, case, "solver1")
    xd, Pd, _ = run_gpu(problems, case, "device")
    assert xh.tobytes() == xd.tobytes() and Ph.tobytes() == Pd.tobytes()
