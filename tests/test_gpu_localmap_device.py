"""Device forms of lasermap_fov_segment and Delete_Point_Boxes (fl_localmap_segment_device, fl_map_delete_boxes_async): the
cube slid from the state on the device and the delete on the caller's stream equal the host forms and the reference's
ikd-Tree, and one CUDA graph replays the whole per-scan chain of laserMapping.cpp."""
import os
import struct
import subprocess

import numpy as np
import pytest

from fast_lio_b200 import api, build, synth
from refcalls import RefTree
from semantics import sort_rows

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FL_OK, FL_ERR_ARG, FL_ERR_STATE, FL_ERR_CAPACITY = 0, -2, -4, -5


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def pos_lid(x):
    """state.pos + state.rot * state.offset_T_L_I (laserMapping.cpp:890) in the order of Eigen's _transformVector."""
    q, v = x[3:6], x[11:14]
    uv = cross(q, v)
    uv = uv + uv
    return x[0:3] + ((v + uv * x[6]) + cross(q, uv))


def state_at(pr, pos, rng):
    """The problem's state with the position moved and the attitude and extrinsic turned, so that pos_lid != pos."""
    x = pr.x_prior.copy()
    x[0:3] = pos
    x[3:7] = synth.quat_mul(x[3:7], synth.quat_exp(rng.normal(0, 0.3, 3)))
    x[11:14] = [0.3, -0.2, 0.15]
    return x


def twins(pr):
    trees = [api.KdTree(0, 0.5) for _ in range(2)]
    for t in trees:
        t.Build(pr.map_pts)
    return trees


def same_map(a, b, queries, size=True):
    """size = False: the maps may have re-packed at different times (size() counts lazily deleted points until a re-pack)."""
    assert a.validnum() == b.validnum() and (not size or a.size() == b.size())
    assert a.tree_range().tobytes() == b.tree_range().tobytes()
    assert sort_rows(a.flatten()).tobytes() == sort_rows(b.flatten()).tobytes()
    for x, y in zip(a.Nearest_Search_K(queries, 5, 2.0), b.Nearest_Search_K(queries, 5, 2.0)):
        assert x.tobytes() == y.tobytes()


def walk(seed, n, step, start):
    rng = np.random.default_rng(seed)
    drift = rng.normal(0, 1, 3)
    drift[2] *= 0.2
    drift /= np.linalg.norm(drift)
    pos = np.array(start, dtype=np.float64)
    for _ in range(n):
        pos = pos + step * (drift + 0.5 * rng.normal(0, 1, 3))
        yield pos.copy()


@pytest.mark.parametrize("cube_len, det_range", [(40.0, 8.0), (24.0, 4.0)])
def test_twin_maps_over_a_walk(problems, cube_len, det_range):
    """segment_device on one map, the host form with pos_lid restated in numpy on the other, the reference's ikd-Tree on a
    third: cub_needrm, kdtree_delete_counter and, after fl_map_maintain, the maps."""
    pr = problems("small")
    th, td = twins(pr)
    lh, ld = api.LocalMap(cube_len, det_range), api.LocalMap(cube_len, det_range)
    rt = RefTree(f"localmap_device_walk_{int(cube_len)}", pr.map_pts)
    rng = np.random.default_rng(5)
    q = np.ascontiguousarray(pr.map_pts[::37])
    out3 = torch.zeros(3, dtype=torch.int32, device="cuda")
    boxes = torch.zeros((3, 6), dtype=torch.float32, device="cuda")
    slides = total = 0
    for pos in walk(9, 30, cube_len / 25.0, pr.x_prior[:3]):
        x = state_at(pr, pos, rng)
        ld.segment_device(td, dev(x), out3, boxes)
        b_h, n_h = lh.segment(pos_lid(x), th)
        o = host(out3)
        assert o[0] == len(b_h) and o[1] == n_h and o[2] in (FL_OK, 1), (o, len(b_h), n_h)
        assert host(boxes)[:len(b_h)].tobytes() == b_h.tobytes()
        if len(b_h):
            assert n_h == rt.delete_boxes(b_h)
            slides += 1
        total += n_h
        td.maintain()
        assert ld.box().tobytes() == lh.box().tobytes()
        same_map(th, td, q)
    assert td.validnum() == rt.validnum()
    assert slides >= 3 and total > 0


def test_first_call_empty_scan_and_far_pose(problems):
    """The first call only places the cube; a zero in n_scan changes nothing and places nothing; a pose far from every face
    deletes nothing (the deleted count read back is 0)."""
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    n0 = t.validnum()
    lm, ref = api.LocalMap(40.0, 8.0), api.LocalMap(40.0, 8.0)
    rng = np.random.default_rng(1)
    x = state_at(pr, pr.x_prior[:3], rng)
    zero = dev(np.array([0], np.int32))
    o = host(lm.segment_device(t, dev(x), n_scan=zero))
    assert o.tolist() == [0, 0, FL_OK]
    with pytest.raises(api.FastLioError):
        lm.box()                                                   # still not placed
    o = host(lm.segment_device(t, dev(x), n_scan=dev(np.array([5], np.int32))))
    assert o.tolist() == [0, 0, FL_OK]
    ref.segment(pos_lid(x))
    assert lm.box().tobytes() == ref.box().tobytes()
    near = x.copy()
    near[0] += 15.0                                                # within 1.5 * det_range of the +x face
    o = host(lm.segment_device(t, dev(near), n_scan=zero))
    assert o.tolist() == [0, 0, FL_OK] and lm.box().tobytes() == ref.box().tobytes() and t.validnum() == n0
    far = x.copy()
    far[0] += 2.0
    o = host(lm.segment_device(t, dev(far)))
    assert o.tolist() == [0, 0, FL_OK] and t.validnum() == n0
    assert len(ref.segment(pos_lid(far))[0]) == 0 and lm.box().tobytes() == ref.box().tobytes()
    o = host(lm.segment_device(t, dev(near)))                      # and now it slides
    b, _ = ref.segment(pos_lid(near))
    assert o[0] == len(b) == 1 and o[1] > 0 and t.validnum() == n0 - o[1]


def cluster(centre, n, half, seed):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), np.float32)
    p[:, :3] = np.asarray(centre, np.float32) + rng.uniform(-half, half, (n, 3)).astype(np.float32)
    p[:, 3] = rng.uniform(0, 100, n).astype(np.float32)
    return p


def test_delete_boxes_async_reads_the_device_leaf_count(problems):
    """fl_map_delete_boxes_async against the host form and the reference: one box, three boxes, nb = 0, nb above nb_max
    (clamped), and a box over points that add_points_async put into overflow leaves since the map last settled, which the
    host's mirror of the used leaves does not count."""
    pr = problems("small")
    th, td = twins(pr)
    rt = RefTree("localmap_device_delete_async", pr.map_pts)
    c = pr.map_pts[:, :3].mean(0)
    q = np.ascontiguousarray(pr.map_pts[::41])
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    B = lambda lo, hi: np.array([*lo, *hi], np.float32)      # noqa: E731
    cases = [
        ([B(c - 2, c + 2)], 1, 1),
        ([B(c + [3, 3, -5], c + [6, 7, 5]), B(c - [8, 8, 5], c - [5, 4, -5]), B(c + [-1, 5, -5], c + [1, 9, 5])], 3, 3),
        ([B(c - 30, c + 30)], 0, 1),                                     # nb = 0: nothing
        ([B(c + [-9, -9, -5], c + [-7, 9, 5]), B(c + [7, -9, -5], c + [9, 9, 5]), B(c - 30, c + 30)], 5, 2),   # clamped to 2
    ]
    for boxes, nb, nb_max in cases:
        boxes = np.array(boxes, np.float32)
        td.delete_boxes_async(dev(boxes), dev(np.array([nb], np.int32)), nb_max, status)
        want = boxes[:min(nb, nb_max)]
        n_h = th.Delete_Point_Boxes(want) if len(want) else 0
        if len(want):
            assert n_h == rt.delete_boxes(want)
        assert host(status).tolist() == [FL_OK, n_h]
    # a dense cluster overflows its leaves (fewer than the chains that would make a re-pack due); no settle between the inserts
    # and the delete
    pts = cluster(c + [12.0, 0.0, 0.0], 1_000, 0.4, seed=3)
    n_d = dev(np.array([len(pts)], np.int32))
    st_add = td.add_points_async(dev(pts), n_d, len(pts), False)
    th.Add_Points(pts, False)
    rt.add(pts, False)
    box = np.array([B(c + [11.0, -1.0, -1.0], c + [13.0, 1.0, 1.0])], np.float32)
    td.delete_boxes_async(dev(box), dev(np.array([1], np.int32)), 1, status)
    n_h = th.Delete_Point_Boxes(box)
    assert host(st_add)[0] in (FL_OK, 1)                          # 1: the crowded cells want a re-list, which keeps the slots
    assert n_h >= len(pts) and n_h == rt.delete_boxes(box)
    assert host(status)[1] == n_h, (host(status), n_h)
    # the host form re-packed the chained leaves right after its insert, the device form at fl_map_maintain after the delete
    td.maintain()
    same_map(th, td, q, size=False)
    assert td.validnum() == rt.validnum()


def test_deferred_repack(problems):
    """A delete that leaves more lazily deleted points than valid ones (and > 1024) reports 1; after fl_map_maintain the map is
    the one the host form re-packed at once."""
    pr = problems("small")
    th, td = twins(pr)
    lo, hi = pr.map_pts[:, :3].min(0), pr.map_pts[:, :3].max(0)
    mid = (lo + hi) / 2
    box = np.array([[*(lo - 1), mid[0] + 0.3 * (hi[0] - mid[0]), hi[1] + 1, hi[2] + 1]], np.float32)
    status = td.delete_boxes_async(dev(box), dev(np.array([1], np.int32)), 1)
    n_h = th.Delete_Point_Boxes(box)
    s = host(status)
    assert s[1] == n_h and n_h > max(1024, th.validnum()), (s, n_h, th.validnum())
    assert s[0] == 1
    td.maintain()
    same_map(th, td, np.ascontiguousarray(pr.map_pts[::29]))


def test_removed_points_record(problems):
    """With the record started, acquire_removed after device deletes returns the point set of the host deletes.  In a captured
    graph replayed until the record is full, a call is refused: map, cube and k-NN answers unchanged; after fl_map_maintain the
    next replay goes through, and the record holds every point deleted."""
    pr = problems("small")
    th, td = twins(pr)
    for t in (th, td):
        assert len(t.acquire_removed_points()) == 0                   # starts the record
    lh, ld = api.LocalMap(40.0, 8.0), api.LocalMap(40.0, 8.0)
    rng = np.random.default_rng(2)
    for pos in list(walk(3, 12, 3.0, pr.x_prior[:3])):
        x = state_at(pr, pos, rng)
        ld.segment_device(td, dev(x))
        lh.segment(pos_lid(x), th)
    rh, rd = th.acquire_removed_points(), td.acquire_removed_points()
    assert len(rh) > 0 and sort_rows(rh).tobytes() == sort_rows(rd).tobytes()

    # Two graphs, replayed in turn: an Add_Points of a fresh cluster in the cube's low slab (the record's room shrinks by the
    # inserted points; statuses of 1 are left owed, since fl_map_maintain would grow the record), then the segment, which slides
    # +x over the cluster.  The first (uncaptured) calls come before the record starts, so fl_map_maintain sizes it first.
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    lm = api.LocalMap(40.0, 8.0)
    x = state_at(pr, pr.x_prior[:3], rng)
    xd = dev(x)
    out3 = torch.zeros(3, dtype=torch.int32, device="cuda")
    n_c = 1_500
    pts = torch.zeros((n_c, 4), dtype=torch.float32, device="cuda")
    n_d = dev(np.array([n_c], np.int32))
    st_add = torch.zeros(2, dtype=torch.int32, device="cuda")
    q = np.ascontiguousarray(pr.map_pts[::31])

    def fill(k):
        box = lm.box()
        pts.copy_(dev(cluster([box[0] + 3.0, (box[1] + box[4]) / 2, (box[2] + box[5]) / 2], n_c, 2.5, seed=k)))
        x[0] = box[3] - 11.0                                         # within 1.5 * det_range of the +x face only
        xd.copy_(dev(x))
        torch.cuda.synchronize()

    lm.segment_device(t, xd, out3)                                   # outside capture: places the cube
    fill(100)
    t.add_points_async(pts, n_d, n_c, False, st_add)                 # outside capture: the map's scratch for n_c points
    t.acquire_removed_points()                                        # starts the record, not sized yet
    L = api.load()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                                        # a record that might be short: nothing captured
        rc = L.fl_localmap_segment_device(lm.h, t.h, xd.data_ptr(), None, None, out3.data_ptr(), t._stream())
    assert rc == FL_ERR_CAPACITY
    assert t.maintain()                                              # sizes the record: graphs captured before are stale

    def capture():
        ga, gs = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(ga):
            t.add_points_async(pts, n_d, n_c, False, st_add)
        with torch.cuda.graph(gs):
            lm.segment_device(t, xd, out3)
        return ga, gs

    ga, gs = capture()
    deleted, refused = 0, False
    for k in range(16):
        fill(k)
        ga.replay()
        assert host(st_add).tolist() in ([FL_OK, 0], [1, 0]), host(st_add)
        before = (t.validnum(), lm.box().tobytes(), [a.tobytes() for a in t.Nearest_Search_K(q, 5, 5.0)])
        gs.replay()
        o = host(out3)
        if o[2] == FL_ERR_CAPACITY:
            refused = True
            assert o[1] == 0
            assert (t.validnum(), lm.box().tobytes(), [a.tobytes() for a in t.Nearest_Search_K(q, 5, 5.0)]) == before
            assert t.maintain()                                      # grows the record, which moves
            ga, gs = capture()
            gs.replay()
            o = host(out3)
            assert o[2] in (FL_OK, 1) and o[0] == 1 and o[1] >= n_c, o
            deleted += int(o[1])
            break
        assert o[2] in (FL_OK, 1) and o[0] == 1 and o[1] >= n_c, o
        deleted += int(o[1])
    assert refused
    assert len(t.acquire_removed_points(cap=1 << 22)) == deleted


def stream_of_raw_scans(pr, n_scans, n_max):
    rng = np.random.default_rng(11)
    out = []
    for step in range(n_scans):
        n = int(rng.integers(n_max // 3, n_max + 1))
        hz = float(rng.choice([100.0, 200.0, 250.0, 400.0]))
        out.append(synth.make_raw_scan(pr.scene, n, synth.true_state(pr.cfg.lidar, step), seed=300 + step, imu_hz=hz))
    return out


CUBE, DET = 3.0, 0.5            # with the predicted state 0.25 m further each scan, the cube slides every 3 scans
PREDICT_DX = 0.25


def test_one_graph_for_the_whole_chain(problems):
    """segment -> upload -> undistort -> down-sample -> update -> map_incremental captured once with n_max (again only after a
    maintenance that moved the map), replayed over 32 raw scans of different sizes: the host-form chain on a twin map gives the
    same cub_needrm, deletes, x, P and, at the end, map.  Between scans the host stands in for esekf::predict by moving the
    updated state 0.25 m along x, and copies the predicted state into the captured x."""
    pr = problems("small")
    n_max, leaf = 9_000, 0.5
    scans = stream_of_raw_scans(pr, 32, n_max)
    n_pose_max = max(len(r.imu_pose) for r in scans)
    th, td = twins(pr)
    fh, fd = (api.Esekf(t, max_points=n_max, max_iter=3) for t in (th, td))
    sh, sd = api.Scan(th), api.Scan(td)
    lh, ld = api.LocalMap(CUBE, DET), api.LocalMap(CUBE, DET)
    sd.reserve(n_max, n_pose_max)
    xyzi = torch.zeros((n_max, 4), dtype=torch.float32, device="cuda")
    tms = torch.zeros(n_max, dtype=torch.float32, device="cuda")
    n_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    poses = torch.zeros((n_pose_max, 22), dtype=torch.float64, device="cuda")
    np_d = torch.zeros(1, dtype=torch.int32, device="cuda")
    xend = torch.zeros(26, dtype=torch.float64, device="cuda")
    xh, Ph = pr.x_prior.copy(), pr.P_prior.copy()
    xd, Pd = dev(xh), dev(Ph)
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    out4 = torch.zeros(4, dtype=torch.int32, device="cuda")
    seg3 = torch.zeros(3, dtype=torch.int32, device="cuda")
    boxes = torch.zeros((3, 6), dtype=torch.float32, device="cuda")

    def fill(r):
        xyzi[:len(r.xyzi)] = dev(r.xyzi); tms[:len(r.xyzi)] = dev(r.offset_ms); n_d.fill_(len(r.xyzi))
        poses[:len(r.imu_pose)] = dev(r.imu_pose); np_d.fill_(len(r.imu_pose)); xend.copy_(dev(r.x_end))

    def chain():
        ld.segment_device(td, xd, seg3, boxes, n_d)
        sd.upload_device(xyzi, tms, n_d, n_max)
        sd.undistort_device(poses, np_d, xend)
        sd.voxel_downsample_device(leaf)
        sd.update_device(fd, xd, Pd, pr.R, status)
        fd.map_incremental_device(0.5, True, out4)

    side = torch.cuda.Stream()
    g, slides, replays = None, 0, 0
    for step, r in enumerate(scans):
        b_h, n_h = lh.segment(pos_lid(xh), th)
        sh.upload(r.xyzi, r.offset_ms); sh.undistort(r.imu_pose, r.x_end); sh.voxel_downsample(leaf)
        xh, Ph, _ = sh.update(fh, xh, Ph, pr.R)
        o3 = fh.map_incremental(0.5, True)
        fill(r)
        torch.cuda.synchronize()
        if step == 0:                                        # outside capture once: the cube and the map's scratch
            with torch.cuda.stream(side):
                chain()
            torch.cuda.synchronize()
        else:
            if g is None:
                td.maintain()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    chain()
            g.replay()
            replays += 1
        s3, o = host(seg3), host(out4)
        assert s3[0] == len(b_h) and s3[1] == n_h and s3[2] in (FL_OK, 1), (step, s3, len(b_h), n_h)
        assert host(boxes)[:len(b_h)].tobytes() == b_h.tobytes(), step
        slides += len(b_h) > 0
        assert host(status)[0] == FL_OK, step
        assert tuple(int(v) for v in o[:3]) == o3 and o[3] in (FL_OK, 1), (step, o)
        assert host(xd).tobytes() == xh.tobytes() and host(Pd).tobytes() == Ph.tobytes(), step
        if (o[3] == 1 or s3[2] == 1) and td.maintain():
            g = None
        xh = xh.copy()
        xh[0] += PREDICT_DX
        xd.copy_(dev(xh))
    assert slides >= 3 and replays >= 30
    td.maintain()
    same_map(th, td, scans[-1].xyzi[::5].copy())
    assert ld.box().tobytes() == lh.box().tobytes()


def test_refusals_enqueue_nothing(problems):
    pr = problems("small")
    L = api.load()
    th, td = twins(pr)
    n0 = td.validnum()
    stream = td._stream()
    x = dev(pr.x_prior)
    out3 = dev(np.array([77, 77, 77], np.int32))
    lm = api.LocalMap(40.0, 8.0)
    # the first call on a capturing stream: nothing captured
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        rc = L.fl_localmap_segment_device(lm.h, td.h, x.data_ptr(), None, None, out3.data_ptr(), td._stream())
    assert rc == FL_ERR_STATE
    h_x = np.ascontiguousarray(pr.x_prior)
    assert L.fl_localmap_segment_device(lm.h, td.h, h_x.ctypes.data, None, None, out3.data_ptr(), stream) == FL_ERR_ARG   # host
    assert L.fl_localmap_segment_device(lm.h, td.h, x.data_ptr() + 4, None, None, out3.data_ptr(), stream) == FL_ERR_ARG  # misaligned
    assert L.fl_localmap_segment_device(lm.h, td.h, x.data_ptr(), None, None, None, stream) == FL_ERR_ARG                 # null out3
    assert L.fl_localmap_segment_device(lm.h, None, x.data_ptr(), None, None, out3.data_ptr(), stream) == FL_ERR_ARG      # null map
    lm.segment_device(td, x)
    assert L.fl_localmap_segment_device(lm.h, th.h, x.data_ptr(), None, None, out3.data_ptr(), stream) == FL_ERR_ARG      # second map
    boxes = dev(np.array([[-1e4, -1e4, -1e4, 1e4, 1e4, 1e4]], np.float32))
    nb = dev(np.array([1], np.int32))
    st = dev(np.array([77, 77], np.int32))
    h_nb = np.array([1], np.int32)
    assert L.fl_map_delete_boxes_async(td.h, boxes.data_ptr(), h_nb.ctypes.data, 1, st.data_ptr(), stream) == FL_ERR_ARG
    assert L.fl_map_delete_boxes_async(td.h, boxes.data_ptr() + 2, nb.data_ptr(), 1, st.data_ptr(), stream) == FL_ERR_ARG
    assert L.fl_map_delete_boxes_async(td.h, boxes.data_ptr(), nb.data_ptr(), 1, None, stream) == FL_ERR_ARG
    assert L.fl_map_delete_boxes_async(td.h, boxes.data_ptr(), nb.data_ptr(), -1, st.data_ptr(), stream) == FL_ERR_ARG
    assert L.fl_map_delete_boxes_async(td.h, None, nb.data_ptr(), 1, st.data_ptr(), stream) == FL_ERR_ARG
    assert host(st).tolist() == [77, 77] and host(out3).tolist() == [77, 77, 77]
    assert td.validnum() == n0


def test_ordering_against_other_streams(problems):
    """A device query in flight on another stream sees the map before the delete; the state written on a sleeping caller
    stream is read after it."""
    pr = problems("small")
    t = api.KdTree(0, 0.5)
    t.Build(pr.map_pts)
    q = np.ascontiguousarray(pr.map_pts[::13])
    want = t.Nearest_Search_K(q, 5, 3.0)
    lm, ref = api.LocalMap(40.0, 8.0), api.LocalMap(40.0, 8.0)
    rng = np.random.default_rng(4)
    x0 = state_at(pr, pr.x_prior[:3], rng)
    lm.segment_device(t, dev(x0))
    ref.segment(pos_lid(x0))
    near = x0.copy()
    near[0] += 15.0
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    qd = dev(q)
    xs = torch.zeros(26, dtype=torch.float64, device="cuda")
    src = dev(near)
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(50_000_000)
        got = t.nearest_search_device(qd, 5, 3.0)
    with torch.cuda.stream(b):
        torch.cuda._sleep(50_000_000)
        xs.copy_(src)
        out3 = lm.segment_device(t, xs)
    torch.cuda.synchronize()
    assert all(g.cpu().numpy().tobytes() == w.tobytes() for g, w in zip(got, want))
    bx, _ = ref.segment(pos_lid(near))
    o = host(out3)
    assert o[0] == len(bx) == 1 and o[1] > 0
    assert lm.box().tobytes() == ref.box().tobytes()


def test_delete_boxes_async_ordering(problems):
    """fl_map_delete_boxes_async: a device query in flight on another stream sees the map before the delete, and the boxes,
    their count and (for nb_max = 0) the status written on a sleeping caller stream are read or overwritten after it."""
    pr = problems("small")
    th, td = twins(pr)
    q = np.ascontiguousarray(pr.map_pts[::13])
    want = td.Nearest_Search_K(q, 5, 3.0)
    c = pr.map_pts[:, :3].mean(0)
    box = np.array([[*(c - 6), *(c + 6)]], np.float32)
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    qd, src_b, src_n = dev(q), dev(box), dev(np.array([1], np.int32))
    boxes = torch.zeros((1, 6), dtype=torch.float32, device="cuda")
    nb = torch.zeros(1, dtype=torch.int32, device="cuda")
    status = torch.full((2,), 77, dtype=torch.int32, device="cuda")
    status0 = torch.full((2,), 77, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(50_000_000)
        got = td.nearest_search_device(qd, 5, 3.0)
    with torch.cuda.stream(b):
        torch.cuda._sleep(50_000_000)
        boxes.copy_(src_b); nb.copy_(src_n)
        td.delete_boxes_async(boxes, nb, 1, status)
        torch.cuda._sleep(20_000_000)
        status0.fill_(5)
        td.delete_boxes_async(boxes, nb, 0, status0)                 # nb_max = 0: (FL_OK, 0), after the fill
    torch.cuda.synchronize()
    assert all(g.cpu().numpy().tobytes() == w.tobytes() for g, w in zip(got, want))
    n_h = th.Delete_Point_Boxes(box)
    assert n_h > 0 and host(status).tolist() == [FL_OK, n_h]
    assert host(status0).tolist() == [FL_OK, 0]
    td.maintain()
    same_map(th, td, q)


def test_plain_c_program_with_one_graph(problems, tmp_path):
    """tests/facade/localmap_device.cu: the C ABI alone captures the six calls once and replays them over raw scans against the
    host forms."""
    pr = problems("small")
    n_max, leaf = 6_000, 0.5
    scans = stream_of_raw_scans(pr, 20, n_max)
    n_pose_max = max(len(r.imu_pose) for r in scans)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as fo:
        fo.write(struct.pack("5i", len(pr.map_pts), len(scans), n_max, n_pose_max, 3))
        fo.write(struct.pack("d", pr.R)); fo.write(struct.pack("f", leaf))
        fo.write(struct.pack("d", CUBE)); fo.write(struct.pack("f", DET)); fo.write(struct.pack("d", PREDICT_DX))
        fo.write(np.ascontiguousarray(pr.map_pts, np.float32).tobytes())
        fo.write(pr.x_prior.astype(np.float64).tobytes()); fo.write(pr.P_prior.astype(np.float64).tobytes())
        for r in scans:
            fo.write(struct.pack("2i", len(r.xyzi), len(r.imu_pose)))
            fo.write(r.xyzi.tobytes()); fo.write(r.offset_ms.tobytes())
            fo.write(r.imu_pose.astype(np.float64).tobytes()); fo.write(r.x_end.astype(np.float64).tobytes())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "localmap_device"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++14", "-I", os.path.join(root, "include"),
           os.path.join(root, "tests", "facade", "localmap_device.cu"), "-o", str(exe), build.LIB,
           "-Xlinker", "-rpath," + os.path.dirname(build.LIB), "-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    res = subprocess.run([str(exe), str(inp)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "all equal" in res.stdout, res.stdout + res.stderr
