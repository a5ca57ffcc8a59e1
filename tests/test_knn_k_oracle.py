"""CPU: the reference's KD_TREE::Nearest_Search(point, k, .., max_dist) (live, or replayed from tests/golden/ref) against the
numpy statement of its contract (knn_rules.py) -- the contract the device map's fl_map_nearest_search is held to."""
import numpy as np
import pytest

import knn_rules
from refcalls import digest, row_digests
from refknn import GATED_KS, KS, MAX_DISTS, KnnRefTree, gated_queries, mutation_run, world_queries


def check(ref, rule):
    """The reference's (row digests, d2 digest, counts) equal the rule's: counts and distances on every row, the neighbour
    rows on decided rows.  Returns how many rows are decided."""
    rows, d, c = ref
    p, rd, rc, decided = rule
    assert np.array_equal(c, rc)
    assert d == digest(rd)
    assert np.array_equal(rows[decided], row_digests(p)[decided])
    return int(decided.sum())


@pytest.mark.parametrize("name", ["tiny", "small", "avia_2k_50k"])
def test_reference_is_the_rule_on_scan_queries(problems, name):
    pr = problems(name)
    q = world_queries(pr)
    r = KnnRefTree(f"knnk_{name}", pr.map_pts)
    for k in KS:
        n = check(r.nearest_search(q, k), knn_rules.nearest(q, pr.map_pts, k))
        assert n >= len(q) // 2


def test_reference_applies_max_dist_as_the_rule(problems):
    pr = problems("small")
    q = gated_queries(pr)
    r = KnnRefTree("knnk_maxdist_small", pr.map_pts)
    for md in MAX_DISTS:
        for k in GATED_KS:
            rule = knn_rules.nearest(q, pr.map_pts, k, md)
            check(r.nearest_search(q, k, md), rule)
            if np.isnan(md):
                assert (rule[2] == 0).all()
            if md == 0:
                assert 0 < rule[2].sum() <= len(q)                   # only coincident points


def test_reference_after_map_mutation_is_the_rule(problems):
    for live, q, answers in mutation_run(problems("tiny")):
        for (k, md), ref in answers.items():
            check(ref, knn_rules.nearest(q, live, k, md))
