"""CPU: the reference's KD_TREE::Box_Search / Radius_Search (live, or replayed from tests/golden/ref) against the numpy
statement of their per-point rules (range_rules.py) -- the contract the device map's range search is held to."""
import numpy as np
import pytest

import range_rules as rr
from refcalls import rows_digest
from refrange import RangeRefTree
from semantics import sort_rows


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_box_search_is_the_half_open_rule(problems, name):
    pr = problems(name)
    boxes, _ = rr.make_queries(pr.map_pts, np.random.default_rng(5), 1000)
    r = RangeRefTree(f"range_box_{name}", pr.map_pts)
    cnt, dig = r.box_search(boxes)
    want = rr.box_sets(boxes, pr.map_pts)
    assert [len(w) for w in want] == list(cnt)
    assert [rows_digest(w) for w in want] == dig
    assert sum(len(w) for w in want[len(want) // 2:]) > 0            # the planted half finds points on its faces


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_radius_search_is_the_literal_rule_up_to_the_band(problems, name):
    pr = problems(name)
    _, spheres = rr.make_queries(pr.map_pts, np.random.default_rng(6), 1000)
    r = RangeRefTree(f"range_radius_{name}", pr.map_pts)
    got = r.radius_search(spheres, pr.map_pts)        # checks literal <= reference <= literal + band, query by query
    lit, band = rr.radius_sets(spheres, pr.map_pts)
    in_band = sum(len(b) for b in band)
    taken = sum(len(g) - len(l) for g, l in zip(got, lit))
    print(f"{name}: {in_band} (query, point) pairs in the band, the reference returned {taken} of them")
    assert in_band > 0                                             # the planted radii reach the band
    for g, l in zip(got, lit):
        assert rr.members(l, g).all()


def test_degenerate_queries_find_nothing():
    rng = np.random.default_rng(8)
    pts = rng.uniform(-5, 5, (3000, 4)).astype(np.float32)
    r = RangeRefTree("range_degenerate", pts)
    boxes = np.array([[np.nan, -5, -5, 5, 5, 5], [-5, -5, -5, 5, np.nan, 5], [1, -5, -5, -1, 5, 5], [0, 0, 0, 0, 0, 0],
                      [-5, -5, -5, 5, 5, 5]], dtype=np.float32)
    cnt, _ = r.box_search(boxes)
    assert list(cnt[:4]) == [0, 0, 0, 0] and cnt[4] == len(pts)
    spheres = np.array([[0, 0, 0, -1], [np.nan, 0, 0, 3], [0, 0, 0, np.nan], [0, 0, 0, 3]], dtype=np.float32)
    got = r.radius_search(spheres, pts)
    assert [len(g) for g in got[:3]] == [0, 0, 0] and len(got[3]) > 0
    empty = RangeRefTree("range_unbuilt", np.zeros((0, 4), np.float32))
    assert list(empty.box_search(boxes)[0]) == [0] * 5
    assert [len(g) for g in empty.radius_search(spheres, np.zeros((0, 4), np.float32))] == [0] * 4


def test_points_on_the_sphere_and_on_the_faces():
    """d2 == r * r exactly (axis offsets of 0.5 m from a centre on the float grid) is inside; min is in, max is out."""
    c = np.array([1.0, 2.0, 3.0], dtype=np.float32)
    pts = np.array([[*(c + [0.5, 0, 0]), 1], [*(c - [0, 0.5, 0]), 2], [*(c + [0, 0, 0.5]), 3], [*(c + [0.5, 0.5, 0]), 4],
                    [*c, 5]], dtype=np.float32)
    r = RangeRefTree("range_exact_boundary", pts)
    got = r.radius_search(np.array([[*c, 0.5]], dtype=np.float32), pts)[0]
    assert np.array_equal(got, sort_rows(pts[[0, 1, 2, 4]]))
    cnt, dig = r.box_search(np.array([[1.0, 2.0, 3.0, 1.5, 2.5, 4.0]], dtype=np.float32))
    assert cnt[0] == 2 and dig[0] == rows_digest(pts[[2, 4]])        # x == 1.5 and y == 2.5 lie on max faces, y == 1.5 below min
