"""The single-GPU update with one tile per worker block (k_update_wave, chosen wherever two threads per point are) against one
thread per point (FASTLIO_B200_PAIR=1): x, P, the pass logs, Nearest_Points, their counts, point_selected_surf and the number
of queries the BVH walk answered must be byte-equal -- through the host form, the device-buffer form and replays of a captured
graph, whose partial rows carry an epoch kept in device memory rather than the launch nonce the graph was captured with.
The lattice map and the map after deletes and re-inserts are compared the same way by test_gpu_update_pairs.py, whose default
side now runs this kernel."""
import os

import numpy as np
import pytest

from fast_lio_b200 import api
from test_gpu_filter_device import dev, host, same_logs
from test_gpu_update_pairs import assert_same, built

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k", "velodyne_30k_1m"])
@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("search", [0, 1])
def test_wave_equals_single_threads(problems, name, extr, search):
    pr = problems(name)
    out = assert_same(built(pr), pr, pr.scan, extr=extr, search=search)
    assert out["logs"][0][0] == 1 and out["logs"][0][2] > 0 and len(out["logs"]) >= 2


def device_update(f, scan, x0, P0, R):
    x, P = dev(x0), dev(P0)
    st = f.update_device(dev(scan), x, P, R)
    return host(x), host(P), host(st)


def single_thread_update(t, pr, x0, P0):
    os.environ["FASTLIO_B200_PAIR"] = "1"
    try:
        f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)
        x, P, _ = f.update_iterated_dyn_share_modified(pr.scan, x0, P0, pr.R)
        n = len(pr.scan)
        return x, P, f.download_state()[2], f.pass_logs(), f.nearest(n), f.selected(n)
    finally:
        os.environ.pop("FASTLIO_B200_PAIR", None)


@pytest.mark.parametrize("name", ["avia_2k_50k", "velodyne_30k_1m"])
def test_wave_device_form(problems, name):
    pr = problems(name)
    t = built(pr)
    n = len(pr.scan)
    xh, Ph, nh, logs, (ph, ch), sh = single_thread_update(t, pr, pr.x_prior, pr.P_prior)
    f = api.Esekf(t, max_points=n, max_iter=pr.cfg.max_iter, limit=pr.limit)
    xd, Pd, st = device_update(f, pr.scan, pr.x_prior, pr.P_prior, pr.R)
    assert xd.tobytes() == xh.tobytes() and Pd.tobytes() == Ph.tobytes() and list(st) == [0, nh]
    same_logs(f.pass_logs(), logs)
    pd, cd = f.nearest(n)
    assert pd.tobytes() == ph.tobytes() and cd.tobytes() == ch.tobytes() and f.selected(n).tobytes() == sh.tobytes()


def test_wave_graph_replays_from_two_priors(problems):
    """One captured update replayed from two different priors: each replay equals the one-thread update from its prior.  A
    replay passes the nonce it was captured with; rows tagged with it would let the second replay sum the first one's rows."""
    pr = problems("velodyne_30k_1m")
    t = built(pr)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit)
    sd, xs, Ps = dev(pr.scan), dev(pr.x_prior), dev(pr.P_prior)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                  # warm-up outside capture
        f.update_device(sd, xs, Ps, pr.R, status)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        f.update_device(sd, xs, Ps, pr.R, status)
    rng = np.random.default_rng(11)
    outs = []
    for rep in range(2):
        x0 = pr.x_prior.copy()
        x0[:3] += rng.normal(0, 0.05, 3)
        P0 = pr.P_prior * (1.0 + 0.5 * rep)
        xs.copy_(dev(x0)); Ps.copy_(dev(P0))
        g.replay()
        torch.cuda.synchronize()
        xh, Ph, nh, logs, _, _ = single_thread_update(t, pr, x0, P0)
        assert host(xs).tobytes() == xh.tobytes() and host(Ps).tobytes() == Ph.tobytes(), rep
        assert list(host(status)) == [0, nh], rep
        same_logs(f.pass_logs(), logs)
        outs.append(xh.tobytes())
    assert outs[0] != outs[1]
