"""The reference's own Preprocess::process (oracle/_ref/libpreprocess_ref.so: src/preprocess.cpp compiled unmodified) against
tests/preprocess_rules.py, bit for bit, on the four LiDAR types with feature extraction off.  Where oracle/_ref is absent the
reference's answers are replayed from tests/golden/ref/preprocess_oracle.npz (digests of its pl_surf)."""
import numpy as np
import pytest

import preprocess_rules as R
from fast_lio_b200 import api, synth
from refcalls import digest
from refpreprocess import RefPreprocess

CFG = {R.AVIA: dict(n_scans=6, scan_rate=10, time_unit=R.NS), R.VELO16: dict(n_scans=32, scan_rate=10, time_unit=R.US),
       R.OUST64: dict(n_scans=64, scan_rate=10, time_unit=R.NS), R.MARSIM: dict(n_scans=1, scan_rate=10, time_unit=R.US)}


@pytest.fixture(scope="module")
def ref():
    return RefPreprocess("preprocess_oracle")


def small_frame(t, blind, times=True):
    if t == R.AVIA:
        return synth.raw_frame("avia", seed=11, blind=blind, n=3000)
    if t == R.VELO16:
        return synth.raw_frame("velodyne", seed=12, blind=blind, rings=16, cols=120, yaw0_deg=-171.0, times=times)
    if t == R.OUST64:
        return synth.raw_frame("ouster", seed=13, blind=blind, rings=16, cols=128)
    return synth.raw_frame("marsim", seed=14, blind=blind, n=2000)


def check(ref, raw, t, pfn, blind, offsets=None, **over):
    cfg = dict(CFG[t], **over)
    offsets = api.layout_offsets(raw.dtype, t) if offsets is None else offsets
    want = ref.process(raw, offsets, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, blind)
    xyzi, ms = R.process(raw, offsets, t, cfg["n_scans"], cfg["scan_rate"], cfg["time_unit"], pfn, blind)
    if "xyzi" in want:
        assert len(want["ms_full"]) == len(ms), (len(want["ms_full"]), len(ms))
        np.testing.assert_array_equal(want["xyzi"].view(np.uint32), xyzi.view(np.uint32))
        np.testing.assert_array_equal(want["ms_full"].view(np.uint32), ms.view(np.uint32))
    assert want["count"] == len(ms)
    assert want["xyzi_digest"] == digest(xyzi) and want["ms_digest"] == digest(ms)
    return xyzi, ms


@pytest.mark.parametrize("blind", [0.5, 2.0])
@pytest.mark.parametrize("pfn", [1, 2, 3, 4])
@pytest.mark.parametrize("t", [R.AVIA, R.VELO16, R.OUST64, R.MARSIM])
def test_frames(ref, t, pfn, blind):
    raw = small_frame(t, blind)
    xyzi, ms = check(ref, raw, t, pfn, blind)
    r2 = (xyzi[:, 0] * xyzi[:, 0] + xyzi[:, 1] * xyzi[:, 1] + xyzi[:, 2] * xyzi[:, 2]).astype(np.float64)
    on_blind = np.isclose(r2, blind * blind, rtol=0, atol=0)
    if t in (R.OUST64, R.MARSIM) and (t == R.MARSIM or pfn == 1):
        assert on_blind.any(), "a row exactly at blind^2 is kept by Ouster and MARSIM"
    if t in (R.AVIA, R.VELO16):
        assert not on_blind.any(), "a row exactly at blind^2 is dropped by Avia and Velodyne"
    if t == R.MARSIM:
        assert len(ms) == len(check(ref, raw, t, 1, blind)[1]), "MARSIM ignores point_filter_num"
    if t == R.OUST64:
        assert (raw["t"] > 2 ** 24).any()


@pytest.mark.parametrize("pfn", [1, 3])
def test_velodyne_yaw_path(ref, pfn):
    """No point times: the offset time comes from the yaw per ring; each ring's first row is never output, and the sweep
    crosses +-180 deg."""
    raw = small_frame(R.VELO16, 0.5, times=False)
    xyzi, ms = check(ref, raw, R.VELO16, pfn, 0.5)
    firsts = {int(r): i for i, r in reversed(list(enumerate(raw["ring"])))}
    out = {tuple(p) for p in xyzi[:, :3].tolist()}
    assert not any((raw["x"][i], raw["y"][i], raw["z"][i]) in out for i in firsts.values())
    yaw = np.degrees(np.arctan2(raw["y"], raw["x"]))
    assert yaw.min() < -170 and yaw.max() > 170
    assert ms.max() > 0 and (ms >= 0).all()


def test_velodyne_missing_time_field(ref):
    """A cloud without a `time` field reads time 0 (as PCL's fromROSMsg leaves it): the yaw path."""
    raw = small_frame(R.VELO16, 0.5, times=True)
    off = api.layout_offsets(raw.dtype, R.VELO16)
    off[4] = -1
    xyzi, ms = check(ref, raw, R.VELO16, 1, 0.5, offsets=off)
    assert len(ms) < len(raw) - 16 + 1


def test_ouster_missing_time_field(ref):
    raw = small_frame(R.OUST64, 0.5)
    off = api.layout_offsets(raw.dtype, R.OUST64)
    off[4] = -1
    xyzi, ms = check(ref, raw, R.OUST64, 2, 0.5, offsets=off)
    assert (ms == 0).all()


@pytest.mark.parametrize("t", [R.AVIA, R.VELO16, R.OUST64, R.MARSIM])
@pytest.mark.parametrize("n", [0, 1, 2])
def test_tiny_frames(ref, t, n):
    raw = small_frame(t, 0.5)[5:5 + n]
    check(ref, raw, t, 1, 0.5)


def _avia_rows(pts, tags=None):
    a = np.zeros(len(pts), api.CUSTOM_POINT)
    p = np.asarray(pts, np.float32)
    a["x"], a["y"], a["z"] = p[:, 0], p[:, 1], p[:, 2]
    a["offset_time"] = np.arange(len(pts)) * 1000
    a["reflectivity"] = np.arange(len(pts))
    a["tag"] = 0x10 if tags is None else tags
    return a


def test_avia_duplicates_and_row0(ref):
    """Row 0 is never output.  With pfn 1 a row equal to the previous (selected) row is dropped; with pfn 2 the previous row
    was not selected, so the comparison is with the origin and equal consecutive rows are kept.  Two rows 0.5 m apart in x
    are different points: abs() is the float overload (abs(int) would truncate 0.5 to 0).  blind 0 lets points next to the
    origin through the range test."""
    pts = [[9, 9, 9], [5, 1, 1], [5, 1, 1], [5, 1, 1], [5, 1, 1], [10.0, 3, 4], [10.5, 3, 4], [5e-8, 0, 0], [5e-8, 0, 0],
           [0, 0, 0], [2e-7, 0, 0], [7, 7, 7]]
    raw = _avia_rows(pts)
    check(ref, raw, R.AVIA, 1, 0.0)
    rows1 = R.avia(R.decode(raw, api.layout_offsets(raw.dtype, R.AVIA), R.AVIA), 6, 1, 0.0)[0]
    assert 0 not in rows1 and 5 in rows1 and 6 in rows1 and 2 not in rows1
    rows2 = R.avia(R.decode(raw, api.layout_offsets(raw.dtype, R.AVIA), R.AVIA), 6, 2, 0.0)[0]
    check(ref, raw, R.AVIA, 2, 0.0)
    assert 2 in rows2 and 4 in rows2 and 8 not in rows2          # rows 2, 4: vs the origin; row 8 (5e-8 m) is the origin's duplicate
    for pfn in (3, 4):
        check(ref, raw, R.AVIA, pfn, 0.0)
    tags = np.array([0x10, 0x20, 0x30, 0x00, 0x10, 0x10, 0x12, 0x01, 0x10, 0x10, 0x10, 0x10], np.uint8)
    raw_t = _avia_rows(pts, tags)
    raw_t["line"][3] = 6
    for pfn in (1, 2):
        check(ref, raw_t, R.AVIA, pfn, 0.0)


# ------------------------------------------------------------------------------------------- the scan form of the recurrence
def _scan_case(rng, n, rings, pool):
    keys = np.sort(rng.integers(0, rings, n))
    lo = rng.choice(pool, n).astype(np.float32)
    hi = (lo.astype(np.float64) + 360.0 / 3.61).astype(np.float32)
    return keys, lo, hi


@pytest.mark.parametrize("seed", range(6))
def test_triple_scan_equals_sequential_loop(seed):
    """The segmented scan of (t, a, b) maps equals the reference's sequential loop bit for bit, on ties lo == c_prev, NaN,
    +-0, lo at the period, repeated values and many rings."""
    rng = np.random.default_rng(seed)
    period = np.float32(360.0 / 3.61)
    pool = np.array([0.0, -0.0, np.nan, period, np.nextafter(period, np.float32(0)), np.nextafter(period, np.float32(200)),
                     1.0, 1.0, 50.0, 99.0, 2 * period, -1.0, np.inf, -np.inf, 1e-30], np.float32)
    for n, rings in ((1, 1), (2, 1), (17, 3), (300, 1), (1000, 64), (4096, 128)):
        if seed % 2:
            keys, lo, hi = _scan_case(rng, n, rings, pool)
        else:
            # mostly realistic times, with a fifth of the rows from the adversarial pool
            keys, _, _ = _scan_case(rng, n, rings, pool)
            lo = rng.uniform(0, 110, n).astype(np.float32)
            m = rng.random(n) < 0.2
            lo[m] = rng.choice(pool, m.sum())
            hi = (lo.astype(np.float64) + 360.0 / 3.61).astype(np.float32)
        want = R.sequential(keys, lo, hi)
        got = R.scan_by_key(keys, lo, lo, hi)
        np.testing.assert_array_equal(want.view(np.uint32), got.view(np.uint32))
        # ties: a row equal to its predecessor's result keeps lo (the comparison is strict)
        tie = np.concatenate([[False], (lo[1:] == want[:-1]) & (keys[1:] == keys[:-1])])
        assert (want[tie].view(np.uint32) == lo[tie].view(np.uint32)).all()
