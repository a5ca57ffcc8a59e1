"""CPU: the launch plan of the iterated-EKF update (fast_lio_b200/csrc/upd_plan.h), run through a g++-built harness
(tests/kernels/upd_plan_harness.cpp), equals a restatement of the rules each route applied before they were gathered there
(filter.cu / filter.h at commit 6637535; the lines are cited below).  Routes: UpdArgs modes 0-3 over the host-bound scan,
the device count (update_scan_on_stream), neighbour completion and the batch; on H100's capacities and on adversarial ones."""
from __future__ import annotations

import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "kernels", "upd_plan_harness.cpp")

KERNELS = ["U1", "U2", "N1", "N2", "WAVE", "N_WAVE", "BATCH"]      # enum UpdKernel, in order
MODE0, MODE1, MODE2, MODE3, DEVICE_COUNT, NEIGHBOURS, BATCH = range(7)
T = 256                    # UPD_THREADS
WAVE_SMEM = 10496          # sizeof(WavePoint)
FIELDS = ["kernel", "workers", "pair", "grid_x", "slots", "waves", "block", "smem", "pdl"]


def _caps(e0: dict, e1: dict | None = None) -> dict:
    e1 = e0 if e1 is None else e1
    return {k: (e0[k], e1[k]) for k in KERNELS}


# co-resident blocks [kernel] -> (EXTR false, EXTR true)
CAPS = {
    # H100 (132 SMs), as Filter::init measures them: two 256-thread blocks per SM, one 512-thread block (DESIGN §4)
    "h100": _caps(dict(U1=264, U2=132, N1=264, N2=132, WAVE=132, N_WAVE=132, BATCH=264)),
    # the _n and wave forms smaller than the paired host form, and EXTR true differing from EXTR false
    "n_smaller": _caps(dict(U1=264, U2=132, N1=200, N2=100, WAVE=132, N_WAVE=80, BATCH=264),
                       dict(U1=132, U2=132, N1=132, N2=66, WAVE=120, N_WAVE=60, BATCH=132)),
    "wave_smaller": _caps(dict(U1=264, U2=132, N1=264, N2=132, WAVE=40, N_WAVE=20, BATCH=30)),
    # fewer one-thread workers than paired tiles: the paired plan's workers stop short of its tiles
    "one_thread_smaller": _caps(dict(U1=50, U2=132, N1=40, N2=132, WAVE=132, N_WAVE=132, BATCH=7)),
    "ones": _caps({k: 1 for k in KERNELS}),
    # no paired, wave or batch block fits at all (occupancy 0; the one-thread forms count one block per SM)
    "zero": _caps(dict(U1=132, U2=0, N1=132, N2=0, WAVE=0, N_WAVE=0, BATCH=0)),
}
ROWS = [0, 1, 255, 256, 257, 2000, 30000, 131072]
N_HYP = [0, 1, 2, 29, 1000]


def _rows(caps: dict) -> list[int]:
    """ROWS plus the rows on either side of every tile count next to a capacity (where workers, pairing or the wave flip)."""
    out = set(ROWS)
    for c in {v for pair in caps.values() for v in pair}:
        for t in (c - 2, c - 1, c, c + 1):
            out.update(r for r in (T * t - 1, T * t, T * t + 1) if r >= 0)
    return sorted(out)


# ------------------------------------------------------------------------------------------------ the rules at 6637535
def _tiles(nq):
    return (nq + T - 1) // T


def _upd_pair(caps, e, nq, one_thread):
    """Filter::upd_pair, filter.cu:1321-1325 (FASTLIO_B200_PAIR=1 -> one_thread)."""
    if one_thread:
        return 1
    return 2 if 1 <= _tiles(nq) <= caps["U2"][e] - 1 else 1


def _plan(kernel, workers, pair, slots=1, waves=1, pdl=True):
    smem = WAVE_SMEM if kernel in ("WAVE", "N_WAVE") else 0
    return dict(kernel=KERNELS.index(kernel), workers=workers, pair=pair, grid_x=workers + 1, slots=slots, waves=waves,
                block=pair * T, smem=smem, pdl=int(pdl))


def reference_plan(caps, route, nq, e, one_thread, n_hyp):
    """The launch each route made; None where batch_plan refused (FL_ERR_CAPACITY)."""
    cap = {k: v[e] for k, v in caps.items()}
    if route <= MODE3:
        # Filter::launch_update, filter.cu:1298-1316 (workers 1302-1306, the wave 1308-1311), Filter::use_wave, filter.h:199,
        # Filter::launch_upd, filter.cu:1326-1332 (block pair * UPD_THREADS, grid workers + 1, PDL as the filter has it)
        workers = max(0, 0 if route == MODE3 else min(cap["U1"] - 1, _tiles(nq)))
        pair = _upd_pair(caps, e, nq, one_thread)
        if route == MODE0 and pair == 2 and workers + 1 <= cap["WAVE"]:
            return _plan("WAVE", workers, 2)
        return _plan(f"U{pair}", workers, pair)
    if route == NEIGHBOURS:
        # Filter::complete_neighbours, filter.cu:1232-1235: launch_upd(workers, false, a, upd_pair(nq))
        workers = max(1, min(cap["U1"] - 1, _tiles(nq)))
        pair = _upd_pair(caps, e, nq, one_thread)
        return _plan(f"U{pair}", workers, pair, pdl=False)
    if route == DEVICE_COUNT:
        # Filter::update_scan_on_stream, filter.cu:1521-1534
        pair = 2 if _upd_pair(caps, e, nq, one_thread) == 2 and _tiles(nq) <= cap["N2"] - 1 else 1
        workers = max(0, min(cap["N1"] - 1, _tiles(nq)))
        if pair == 2 and workers + 1 <= cap["N_WAVE"]:
            return _plan("N_WAVE", workers, pair)
        return _plan(f"N{pair}", workers, pair)
    # Filter::batch_plan, filter.cu:1544-1557; the launch, filter.cu:1638-1640 (grid (workers + 1, hypotheses), UPD_THREADS)
    w = max(0, min(cap["U1"] - 1, _tiles(nq)))
    if w + 1 > cap["BATCH"]:
        return None
    s = cap["BATCH"] // (w + 1)
    return _plan("BATCH", w, 1, slots=s, waves=(n_hyp + s - 1) // s)


# ------------------------------------------------------------------------------------------------ harness
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("upd_plan") / "libupd_plan.so")
    res = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC", SRC, "-o", out],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    lib = C.CDLL(out)
    assert lib.up_kernel_count() == len(KERNELS)
    i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
    lib.up_plan.argtypes = [i32p, C.c_int, C.c_int, C.c_int, i32p, i32p]

    def plan(caps, cases):
        blocks = np.array([caps[k] for k in KERNELS], dtype=np.int32)
        inp = np.ascontiguousarray(np.array(cases, dtype=np.int32).reshape(-1, 5))
        out = np.zeros((len(inp), len(FIELDS)), dtype=np.int32)
        lib.up_plan(blocks, T, WAVE_SMEM, len(inp), inp, out)
        return [dict(zip(FIELDS, map(int, row))) for row in out]
    return plan


def _cases(caps):
    for route, nq, e, one_thread in itertools.product(range(7), _rows(caps), (0, 1), (0, 1)):
        for n_hyp in (N_HYP if route == BATCH else [0]):
            yield (route, nq, e, one_thread, n_hyp)


@pytest.mark.parametrize("name", sorted(CAPS))
def test_every_route_plans_what_it_launched_before(planner, name):
    caps = CAPS[name]
    cases = list(_cases(caps))
    got = planner(caps, cases)
    seen = set()
    for case, g in zip(cases, got):
        want = reference_plan(caps, *case)
        if want is None:
            assert g["slots"] == 0 and g["waves"] == 0, (case, g)
            continue
        assert g == want, (case, g, want)
        seen.add(KERNELS[g["kernel"]])
    # the grid reaches every kernel the capacities allow.  Where k_update_n_wave's grid is as large as k_update_n<EXTR, 2>'s,
    # as on H100, every paired device-count launch runs the wave form.
    reachable = {"h100": set(KERNELS) - {"N2"}, "one_thread_smaller": set(KERNELS) - {"N2"}, "zero": {"U1", "N1"},
                 "ones": {"U1", "N1", "BATCH"}}
    assert seen == reachable.get(name, set(KERNELS)), seen


def test_h100_plans(planner):
    """The grids DESIGN §4 and §6b quote for H100: avia_2k (2 000 points, 8 tiles) and config 2 (30 000 points, 118 tiles)
    pair and run the wave kernels in mode 0, config 3 (131 072 points, 512 tiles) keeps one thread per point, and a batch wave
    holds 29 hypotheses at 2 000 points and 2 at config 2.  The three routes that differ from mode 0 differ as before: neighbour
    completion has no PDL and no wave kernel, mode 3 is one block of the pair choice's size, and the device count pairs only
    while its own paired grid holds the tiles."""
    caps = CAPS["h100"]

    def one(route, nq, one_thread=0, n_hyp=0, caps=caps):
        return planner(caps, [(route, nq, 0, one_thread, n_hyp)])[0]

    p = one(MODE0, 2000)
    assert (KERNELS[p["kernel"]], p["workers"], p["block"], p["smem"], p["pdl"]) == ("WAVE", 8, 512, WAVE_SMEM, 1)
    assert KERNELS[one(MODE0, 30000)["kernel"]] == "WAVE" and one(MODE0, 30000)["grid_x"] == 119
    assert KERNELS[one(DEVICE_COUNT, 30000)["kernel"]] == "N_WAVE"
    assert KERNELS[one(MODE0, 2000, one_thread=1)["kernel"]] == "U1"
    p = one(MODE0, 131072)
    assert (KERNELS[p["kernel"]], p["workers"], p["block"]) == ("U1", 263, 256)
    p = one(MODE3, 2000)
    assert (KERNELS[p["kernel"]], p["grid_x"], p["block"]) == ("U2", 1, 512)
    p = one(NEIGHBOURS, 2000)
    assert (KERNELS[p["kernel"]], p["workers"], p["pdl"]) == ("U2", 8, 0)
    assert one(NEIGHBOURS, 0)["workers"] == 1
    assert (one(BATCH, 2000, n_hyp=256)["slots"], one(BATCH, 2000, n_hyp=256)["waves"]) == (29, 9)
    assert one(BATCH, 30000, n_hyp=5)["slots"] == 2
    # 100 tiles: the host form pairs, the device count against an _n paired grid of 100 blocks does not
    n_small = _caps(dict(U1=264, U2=132, N1=264, N2=100, WAVE=132, N_WAVE=100, BATCH=264))
    assert KERNELS[one(MODE0, 100 * T, caps=n_small)["kernel"]] == "WAVE"
    assert KERNELS[one(DEVICE_COUNT, 100 * T, caps=n_small)["kernel"]] == "N1"
