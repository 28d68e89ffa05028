"""CPU checks of filtered search (InlineFilterSearch, diskann/src/graph/search/inline_filter_search.rs).

The oracle (oracle/filtered_search.cpp) reproduces the reference's 12 inline baselines, passes the reference's
compute_adaptive_l unit cases and equals an independent Python restatement (tests/filtered_oracle.py) on random and edge
graphs at every selectivity, both modes and every adaptive-L region.  With a filter that accepts every id and no adaptive
L its traversal is the k-NN traversal.  The C entry points refuse a NULL index before any device work."""
import json
import os

import numpy as np
import pytest

import filtered_oracle as F
import oracle_lib as O
from test_oracle_golden import grid
from test_traversal_edges import clustered, grid as tie_grid, malformed_case, many_starts, non_finite

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIVE = ("ids", "dists", "counts", "cmps", "hops")
EMPTY = 0xFFFFFFFF


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


# ---------------------------------------------------------------- the reference's graphs, restated

def provider_graph(start_id, start_pos, start_nbrs, points, max_degree):
    """test_provider::Provider::new_from over 1-D points: the data ids are renumbered 0.. in id order and the start
    point becomes the last id, as the index keeps start points after the data.  Returns (vecs, adj, n, to_ref)."""
    ref_ids = sorted(p[0] for p in points)
    to_new = {r: i for i, r in enumerate(ref_ids)}
    n = len(ref_ids)
    to_new[start_id] = n
    vecs = np.zeros((n + 1, 1), np.float32)
    adj = np.zeros((n + 1, max_degree + 1), np.uint32)
    for rid, pos, nbrs in list(points) + [(start_id, [start_pos], start_nbrs)]:
        u = to_new[rid]
        vecs[u] = pos
        adj[u, 0] = len(nbrs)
        adj[u, 1:1 + len(nbrs)] = [to_new[v] for v in nbrs]
    to_ref = np.array(ref_ids + [start_id], np.uint32)
    return vecs, adj, n, to_ref


def three_level():
    """build_three_level_labeled_provider (inline.rs): start 0 at 0.0, ids 1-2 at 0.0, 3-6 at 1.0, 7-14 at 2.0"""
    pts = [(1, [0.0], [0, 3, 4]), (2, [0.0], [0, 5, 6])]
    pts += [(3 + i, [1.0], [1 + i // 2, 7 + 2 * i, 8 + 2 * i]) for i in range(4)]
    pts += [(7 + i, [2.0], [3 + i // 2]) for i in range(8)]
    return provider_graph(0, 0.0, [1, 2], pts, 3)


def reaches_matches():
    """inline_search_reaches_matches_through_non_matching_nodes: build_1d_index (multihop.rs), start 10 at 5.0"""
    pts = [(0, [0.0], [1, 10]), (1, [1.0], [0, 2, 10]), (2, [2.0], [1, 3]), (3, [3.0], [0, 4, 10]), (4, [4.0], [3, 2])]
    return provider_graph(10, 5.0, [0, 1, 3], pts, 4)


def golden_case(c):
    """(vecs, adj, n, to_ref, labels): each case's predicate is a function of the id, so it is one label bit"""
    if c["graph"] == "grid_1d":
        vecs, adj, n = grid(1, 100)
        to_ref = np.arange(n + 1, dtype=np.uint32)
    else:
        vecs, adj, n, to_ref = three_level() if c["graph"] == "three_level" else reaches_matches()
    accept = (to_ref % 2 == 0) if c["accept"] == "even" else np.isin(to_ref, c["accept"])
    return vecs, adj, n, to_ref, accept.astype(np.uint64)


def golden():
    return json.load(open(os.path.join(GOLDEN, "inline_search.json")))["cases"]


@pytest.mark.parametrize("flavour", [O.SIMD, O.AVX2])
def test_the_reference_baselines(flavour):
    """ids (in the reference's order), distances, result_count, comparisons and hops of all 12 baselines"""
    cases = golden()
    assert len(cases) == 12
    for c in cases:
        vecs, adj, n, to_ref, labels = golden_case(c)
        idx = O.Index(vecs, adj, n, 1, O.L2)
        q = np.array([c["query"]], np.float32)
        adaptive = tuple(c["adaptive_l"]) if c["adaptive_l"] else None
        ids, dists, counts, cmps, hops = F.search_batch(idx, q, c["k"], c["l"], labels, 1, adaptive_l=adaptive, flavour=flavour)
        cnt = int(counts[0])
        assert cnt == c["result_count"], c["case"]
        assert to_ref[ids[0, :cnt]].tolist() == c["result_ids"], c["case"]
        assert dists[0, :cnt].tolist() == c["result_distances"], c["case"]
        assert (cmps[0], hops[0]) == (c["comparisons"], c["hops"]), c["case"]
        # the Python restatement agrees
        same(F.py_batch(vecs, adj, n, 1, O.L2, q, c["k"], c["l"], labels, 1, adaptive_l=adaptive), (ids, dists, counts, cmps, hops),
             c["case"])


def test_compute_adaptive_l_reference_cases():
    """test_compute_adaptive_l_{piecewise_regions, zero_samples_or_matches, respects_max_multiplier}"""
    for f in (F.compute_adaptive_l, F.py_adaptive_l):
        assert [f(100, 1000, m, 16.0) for m in (500, 900, 100, 499, 10, 1)] == [100, 100, 200, 200, 400, 800]
        assert f(100, 1000, 0, 16.0) == 1600 and f(100, 0, 0, 16.0) == 1600
        assert f(100, 1000, 1, 4.0) == 400 and f(100, 1000, 10, 1.5) == 150


def test_compute_adaptive_l_equals_the_restatement_everywhere():
    rng = np.random.default_rng(3)
    for _ in range(3000):
        L = int(rng.integers(1, 300))
        v = int(rng.integers(1, 5000))
        m = int(rng.integers(0, v + 1)) if rng.random() < 0.5 else int(rng.integers(0, max(1, v // 20)))
        s = float(rng.choice([1.0, 1.5, 2.0, 3.7, 8.0, 16.0]))
        assert F.compute_adaptive_l(L, v, m, s) == F.py_adaptive_l(L, v, m, s), (L, v, m, s)


# ---------------------------------------------------------------- random and edge graphs

SELECTIVITY = (1.0, 0.5, 0.1, 0.01, 0.0)


def random_labels(rng, total, selectivity, bits=8):
    """labels whose bit b is set with probability `selectivity` for bit 0 and 0.5 for the others"""
    labels = (rng.random((total, bits)) < 0.5).astype(np.uint64)
    labels[:, 0] = rng.random(total) < selectivity
    return (labels << np.arange(bits, dtype=np.uint64)).sum(1).astype(np.uint64)


def built(n, d, n_start, seed, metric=O.L2, dt=np.float32):
    rng = np.random.default_rng(seed)
    base = clustered(rng, n, d)
    vecs = np.concatenate([base, base[rng.integers(0, n, n_start)] + np.float32(0.01)]).astype(dt)
    adj = O.build_graph(vecs, n, n_start, metric, 16, 20, 30)
    queries = (base[rng.integers(0, n, 6)] + np.float32(0.1) * rng.normal(size=(6, d)).astype(np.float32)).astype(dt)
    return vecs, adj, queries, rng


@pytest.mark.parametrize("beam", [1, 2, 4])
def test_oracle_equals_restatement_on_random_graphs(beam):
    n, n_start = 400, 2
    vecs, adj, queries, rng = built(n, 12, n_start, 10 + beam)
    idx = O.Index(vecs, adj, n, n_start, O.L2)
    for sel in SELECTIVITY:
        labels = random_labels(rng, n + n_start, sel)
        for match_all, masks in ((False, np.uint64(1)), (True, np.uint64(1)), (False, np.uint64(0b110)), (True, np.uint64(0b101)),
                                 (True, np.uint64(0))):
            for adaptive in (None, (1, 1.0), (40, 2.0), (60, 8.0), (30, 3.5)):
                args = (queries, 10, 20, labels, masks)
                got = F.search_batch(idx, *args, match_all=match_all, adaptive_l=adaptive, beam=beam)
                want = F.py_batch(vecs, adj, n, n_start, O.L2, *args, match_all=match_all, adaptive_l=adaptive, beam=beam)
                same(got, want, (sel, match_all, int(masks), adaptive))


def test_every_adaptive_region_is_reached():
    """the sample lands in each multiplier region and the grown list changes the results somewhere"""
    n = 600
    vecs, adj, queries, rng = built(n, 8, 1, 5)
    idx = O.Index(vecs, adj, n, 1, O.L2)
    changed = 0
    for sel in (0.9, 0.3, 0.05, 0.005, 0.0):
        labels = random_labels(rng, n + 1, sel)
        fixed = F.search_batch(idx, queries, 10, 12, labels, 1)
        grown = F.search_batch(idx, queries, 10, 12, labels, 1, adaptive_l=(30, 16.0))
        same(grown, F.py_batch(vecs, adj, n, 1, O.L2, queries, 10, 12, labels, 1, adaptive_l=(30, 16.0)), sel)
        changed += int((grown[4] != fixed[4]).any())
    assert changed >= 3


def test_reconfigure_can_shorten_the_list():
    """with many start points a grown L below L + #start cuts the list: fewer hops than without adaptive L"""
    case = many_starts(300, 8, 40, 6, 2)
    labels = np.zeros(case.total, np.uint64)
    labels[::3] = 1
    fixed = F.search_batch(case.oracle, case.queries, 5, 10, labels, 1)
    cut = F.search_batch(case.oracle, case.queries, 5, 10, labels, 1, adaptive_l=(1, 2.0))
    same(cut, F.py_batch(case.vecs, case.adj, case.n, case.n_start, O.L2, case.queries, 5, 10, labels, 1, adaptive_l=(1, 2.0)), "cut")
    assert (cut[4] < fixed[4]).any()


def test_start_points_accepted_and_rejected():
    case = many_starts(300, 8, 70, 6, 4)
    for start_label in (0, 1):
        labels = np.zeros(case.total, np.uint64)
        labels[:case.n:2] = 1
        labels[case.n:] = start_label
        for adaptive in (None, (5, 4.0)):
            got = F.search_batch(case.oracle, case.queries, 10, 30, labels, 1, adaptive_l=adaptive, beam=2)
            same(got, F.py_batch(case.vecs, case.adj, case.n, case.n_start, O.L2, case.queries, 10, 30, labels, 1, adaptive_l=adaptive, beam=2),
                 (start_label, adaptive))
            assert (got[0][got[0] != EMPTY] < case.n).all()


def test_edge_graphs():
    rng = np.random.default_rng(8)
    cases = [malformed_case(300, 8, 3, 24, 6, 1), tie_grid(300, 6, 2, 6, 2), non_finite(200, 8, np.float32, O.L2, 6, 3)[0],
             non_finite(200, 8, np.float32, O.INNER_PRODUCT, 6, 4)[0]]
    for c in cases:
        labels = random_labels(rng, c.total, 0.4)
        for adaptive in (None, (20, 4.0)):
            got = F.search_batch(c.oracle, c.queries, 10, 25, labels, 1, adaptive_l=adaptive)
            same(got, F.py_batch(c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries, 10, 25, labels, 1, adaptive_l=adaptive), adaptive)


def test_deleted_ids_are_matched_but_not_returned():
    n = 300
    vecs, adj, queries, rng = built(n, 8, 1, 9)
    idx = O.Index(vecs, adj, n, 1, O.L2)
    labels = random_labels(rng, n + 1, 0.5)
    deleted = rng.random(n + 1) < 0.3
    got = F.search_batch(idx, queries, 10, 30, labels, 1, deleted=deleted)
    same(got, F.py_batch(vecs, adj, n, 1, O.L2, queries, 10, 30, labels, 1, deleted=deleted), "deleted")
    assert not deleted[got[0][got[0] != EMPTY]].any()


@pytest.mark.parametrize("dt,metric", [(np.float32, O.COSINE), (np.float16, O.INNER_PRODUCT), (np.int8, O.L2), (np.uint8, O.COSINE)])
def test_row_types(dt, metric):
    rng = np.random.default_rng(6)
    n = 300
    base = clustered(rng, n, 16)
    if dt in (np.int8, np.uint8):
        base = np.clip(base * 30 + (0 if dt == np.int8 else 100), -128 if dt == np.int8 else 0, 127 if dt == np.int8 else 255)
    vecs = np.concatenate([base, base[:1]]).astype(dt)
    adj = O.build_graph(vecs, n, 1, metric, 16, 20, 30)
    queries = vecs[rng.integers(0, n, 5)]
    labels = random_labels(rng, n + 1, 0.2)
    idx = O.Index(vecs, adj, n, 1, metric)
    got = F.search_batch(idx, queries, 10, 20, labels, 1, adaptive_l=(20, 8.0))
    same(got, F.py_batch(vecs, adj, n, 1, metric, queries, 10, 20, labels, 1, adaptive_l=(20, 8.0)), (dt, metric))


def test_accept_all_is_the_knn_traversal():
    """labels that every query accepts, no adaptive L: the k-NN traversal's hops, its cmps less the start points (which
    the filtered search does not count, inline_filter_search.rs:199-209), and its ids up to exact ties"""
    for n_start, seed in ((1, 1), (5, 2)):
        n = 500
        vecs, adj, queries, rng = built(n, 12, n_start, seed)
        idx = O.Index(vecs, adj, n, n_start, O.L2)
        for beam in (1, 3):
            for match_all, mask, labels in ((False, 1, np.ones(n + n_start, np.uint64)), (True, 0, random_labels(rng, n + n_start, 0.5))):
                got = F.search_batch(idx, queries, 10, 20, labels, mask, match_all=match_all, beam=beam)
                want = idx.search_batch(queries, 10, 20, beam=beam)
                assert np.array_equal(got[4], want[4]) and np.array_equal(got[3], want[3] - n_start)
                assert np.array_equal(got[2], want[2]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
                for q in range(queries.shape[0]):
                    for d in np.unique(want[1][q]):
                        assert set(got[0][q][got[1][q] == d]) == set(want[0][q][want[1][q] == d])


# ---------------------------------------------------------------- the C entry points without a device

def test_entry_points_refuse_a_null_index_before_any_device_work():
    import diskann_b200 as dab
    L = dab.lib()
    before = L.dab_launch_count()
    masks = np.ones(4, np.uint64)
    assert L.dab_upload_labels(None, O.ptr(masks), 0, 4) == 1
    assert b"NULL" in L.dab_last_error()
    for fn in (L.dab_search_batch_filtered, L.dab_search_batch_filtered_device):
        assert fn(None, None, 0, 10, 20, 1, O.ptr(masks), 0, 0, 1.0, None, None, None, None, None) == 1
        assert b"idx is NULL" in L.dab_last_error()
        assert fn(None, None, 4, 10, 20, 1, O.ptr(masks), 1, 100, 0.5, None, None, None, None, None) == 1
    assert L.dab_launch_count() == before


def test_python_refuses_a_zero_sample_count():
    import diskann_b200 as dab
    with pytest.raises(ValueError, match="sample count"):
        dab.GpuIndex._adaptive((0, 2.0))
    assert dab.GpuIndex._adaptive(None) == (0, 1.0)
