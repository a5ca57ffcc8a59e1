"""CPU: the wave kernels' partial row (csrc/wave_row.cuh).  Without extrinsic estimation the row carries only the 29 sums
warp_accumulate writes -- H^T H with a <= b < 6, H^T h[0..5], effct, sum |res| -- and the index map must send each of them to
exactly one slot, in warp_accumulate's order, and no other entry anywhere; with it the row is the 96 sums as they are.  Also the
footprint of k_update_wave: 128 registers and one 512-thread block per SM, no more stack or spills than before the compact row."""
import os
import subprocess

import pytest

from fast_lio_b200 import build
from test_device_queries_build import spills
from test_frontend_device_build import frames
from test_map_async_build import cubin

PROBE = r"""
#define __host__
#define __device__
#include <cstdio>
#include "wave_row.cuh"
int main() {
    for (int s = 0; s < fl::WaveRow<false>::LIVE; s++) std::printf("e0 %d %d\n", s, fl::wave_entry<false>(s));
    for (int s = 0; s < fl::WaveRow<true>::LIVE; s++) std::printf("e1 %d %d\n", s, fl::wave_entry<true>(s));
    for (int o = 0; o < 96; o++) std::printf("s0 %d %d\ns1 %d %d\n", o, fl::wave_slot<false>(o), o, fl::wave_slot<true>(o));
    std::printf("w %d %d %d %d\n", fl::WaveRow<false>::W, fl::WaveRow<false>::LIVE, fl::WaveRow<true>::W, fl::WaveRow<true>::LIVE);
}
"""


def tri12(a, b):
    return a * 12 - a * (a - 1) // 2 + (b - a)


@pytest.fixture(scope="module")
def wave_map(tmp_path_factory):
    d = tmp_path_factory.mktemp("wave_row")
    src, exe = d / "probe.cpp", d / "probe"
    src.write_text(PROBE)
    subprocess.run(["g++", "-std=c++17", "-I", build.CSRC, str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    out = {"e0": {}, "e1": {}, "s0": {}, "s1": {}}
    for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        f = line.split()
        if f[0] == "w":
            out["w"] = tuple(int(v) for v in f[1:])
        else:
            out[f[0]][int(f[1])] = int(f[2])
    return out


def test_compact_row_carries_each_live_sum_once(wave_map):
    # warp_accumulate<false>'s outputs, in its order: the pairs (a <= b < 6) row-major, H^T h, effct, sum |res|
    live = [tri12(a, b) for a in range(6) for b in range(a, 6)] + [78 + a for a in range(6)] + [90, 91]
    assert len(live) == 29
    assert wave_map["w"] == (32, 29, 96, 96)
    assert [wave_map["e0"][s] for s in range(29)] == live
    for o in range(96):
        assert wave_map["s0"][o] == (live.index(o) if o in live else -1), o
    # the pads 29..31 carry nothing; the 67 dead entries have no slot
    assert sum(v < 0 for v in wave_map["s0"].values()) == 96 - 29


def test_wide_row_is_the_partial_row(wave_map):
    assert [wave_map["e1"][s] for s in range(96)] == list(range(96))
    assert [wave_map["s1"][o] for o in range(96)] == list(range(96))


@pytest.fixture(scope="module")
def filter_log(tmp_path_factory):
    return cubin("filter.cu", tmp_path_factory)[0]


@pytest.mark.parametrize("kernel, stack, spilled", [
    ("_ZN2fl13k_update_waveILb0EEEvNS_7UpdArgsEPy", 800, 384),
    ("_ZN2fl13k_update_waveILb1EEEvNS_7UpdArgsEPy", 848, 564),
])
def test_wave_kernel_footprint(filter_log, kernel, stack, spilled):
    """One 512-thread block per SM at the 128-register cap; stack and spill bytes no larger than the 96-double row's (nvcc 12.9:
    800 / 848 bytes of stack and 384 / 564 bytes spilled for EXTR false / true)."""
    st, regs, _ = frames(filter_log)[kernel]
    assert regs <= 128, regs
    assert st <= stack, st
    assert spills(filter_log)[kernel] <= spilled, spills(filter_log)[kernel]
