"""The wave kernels' partial rows (csrc/wave_row.cuh: 32 doubles without extrinsic estimation, 96 with it) against one thread
per point (FASTLIO_B200_PAIR=1, k_update's 96-double rows): byte-equal x, P and pass logs with extrinsic estimation through
back-to-back replays of a captured graph, whose rows are told apart by the epoch alone, and on scans whose last tile is partial."""
import os

import numpy as np
import pytest

from fast_lio_b200 import api
from test_gpu_filter_device import dev, host, same_logs
from test_gpu_update_pairs import assert_same, built

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def one_thread(t, pr, scan, x0, P0, extr):
    os.environ["FASTLIO_B200_PAIR"] = "1"
    try:
        f = api.Esekf(t, max_points=len(scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr))
        x, P, _ = f.update_iterated_dyn_share_modified(scan, x0, P0, pr.R)
        return x, P, f.download_state()[2], f.pass_logs()
    finally:
        os.environ.pop("FASTLIO_B200_PAIR", None)


@pytest.mark.parametrize("name", ["avia_2k_50k", "velodyne_30k_1m"])
@pytest.mark.parametrize("extr", [0, 1])
def test_graph_replays_back_to_back(problems, name, extr):
    """Two replays of one captured update with nothing in between, each from its own prior: each equals the one-thread update."""
    pr = problems(name)
    t = built(pr)
    f = api.Esekf(t, max_points=len(pr.scan), max_iter=pr.cfg.max_iter, limit=pr.limit, extrinsic_est_en=bool(extr))
    sd, xs, Ps = dev(pr.scan), dev(pr.x_prior), dev(pr.P_prior)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        f.update_device(sd, xs, Ps, pr.R, status)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        f.update_device(sd, xs, Ps, pr.R, status)
    rng = np.random.default_rng(23 + extr)
    priors = []
    for rep in range(2):
        x0 = pr.x_prior.copy()
        x0[:3] += rng.normal(0, 0.05, 3)
        priors.append((x0, pr.P_prior * (1.0 + 0.5 * rep)))
    x_in, P_in = [dev(x0) for x0, _ in priors], [dev(P0) for _, P0 in priors]
    outs = []
    for rep in range(2):                             # the second replay follows the first on the stream, no host sync between
        xs.copy_(x_in[rep]); Ps.copy_(P_in[rep])
        g.replay()
        outs.append((xs.clone(), Ps.clone(), status.clone()))
    torch.cuda.synchronize()                         # pass_logs() waits for the filter's stream, not the replays' stream
    logs_last = f.pass_logs()
    for rep, (xd, Pd, sd_) in enumerate(outs):
        xh, Ph, nh, logs = one_thread(t, pr, pr.scan, *priors[rep], extr)
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), rep
        assert list(host(sd_)) == [0, nh], rep
        if rep == 1:
            same_logs(logs_last, logs)
    assert host(outs[0][0]).tobytes() != host(outs[1][0]).tobytes()


@pytest.mark.parametrize("extr", [0, 1])
@pytest.mark.parametrize("n", [256 * 100 + 1, 256 * 117 + 40])
def test_partial_last_tile(problems, extr, n):
    """Scans whose last worker block has 1 and 40 points of its 256."""
    pr = problems("velodyne_30k_1m")
    assert_same(built(pr), pr, pr.scan[:n], extr=extr, search=1)

