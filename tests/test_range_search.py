"""The range search oracle (oracle/range_search.cpp) against the reference: its five range-search baselines
(tests/golden/range_search.json) under both oracle flavours, an independent Python restatement of Range::search and
range_search_internal (diskann/src/graph/search/range_search.rs:255-469) over random graphs and the edge graphs of
test_traversal_edges.py with every argument the reference accepts, and the reference's argument validation tests
(range_search.rs:515-550).  CPU only: the device is compared with this oracle in test_range_search_gpu.py."""
import json
import os

import numpy as np
import pytest

import oracle_lib as O
import range_oracle as R
from test_gpu_parity import make_index
from test_oracle_golden import grid as lattice
from test_traversal_edges import grid, malformed_case, many_starts, non_finite

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "range_search.json")
F32 = np.float32


def py_range(vecs, adj, n_points, n_start, metric, query, L, radius, beam=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
             max_returned=None, deleted=None):
    """Range::search restated: (ids, dists, cmps, hops, second_round) of one query, with the oracle's distances"""
    total = n_points + n_start
    q = np.ascontiguousarray(query.astype(F32) if vecs.dtype == np.float16 else query)  # f16 queries are widened
    dist = lambda ids: O.distance_rows(q, vecs[np.asarray(ids, np.int64)], metric, O.AVX2) if len(ids) else np.empty(0, F32)
    neighbours = lambda i: [int(x) for x in adj[i, 1:1 + adj[i, 0]]]

    def expand(nodes, visited):  # expand_beam: every neighbour enters the visited set before the bounds check
        out = []
        for node in nodes:
            for j in neighbours(node):
                if j in visited:
                    continue
                visited.add(j)
                if j < total:
                    out.append(j)
        return out

    # phase 1: search_internal over a NeighborPriorityQueue of L + #start entries
    cap, ids, ds, done, cursor = L + n_start, [], [], [], 0

    def insert(i, d):
        nonlocal cursor
        if np.isnan(d) or (len(ids) == cap and ds[-1] < d):
            return
        at = next((j for j, x in enumerate(ds) if x >= d), len(ds))
        if len(ids) == cap:
            del ids[-1], ds[-1], done[-1]
        ids.insert(at, i), ds.insert(at, d), done.insert(at, False)
        cursor = min(cursor, at)

    visited = set(range(n_points, total))
    for i, d in zip(range(n_points, total), dist(list(range(n_points, total)))):
        insert(i, d)
    cmps, hops = n_start, 0
    while cursor < len(ids):
        nodes = []
        while len(nodes) < beam and cursor < len(ids):
            done[cursor] = True
            nodes.append(ids[cursor])
            while cursor < len(ids) and done[cursor]:
                cursor += 1
        new = expand(nodes, visited)
        for i, d in zip(new, dist(new)):
            insert(i, d)
        cmps += len(new)
        hops += len(nodes)
    # in_range, the second round, the output
    in_range = [(i, d) for i, d in zip(ids[:L], ds[:L]) if d <= radius]
    limit = max_returned or (1 << 63)
    second = len(in_range) >= int(F32(L) * F32(initial_slack)) and len(in_range) < limit
    if second:
        visited, front, hops2 = {i for i, _ in in_range}, 0, 0
        with np.errstate(invalid="ignore"):
            bound = F32(radius) * F32(range_slack)  # 0 * inf: NaN, which admits nothing
        while front < len(in_range) and len(in_range) < limit:
            nodes = [i for i, _ in in_range[front:front + beam]]
            front += len(nodes)
            new = expand(nodes, visited)
            for i, d in zip(new, dist(new)):
                if d <= bound and len(in_range) < limit:
                    in_range.append((i, d))
            hops2 += len(nodes)
        hops = hops + (hops + hops2)
    out = [(i, d) for i, d in in_range if i < n_points and not (deleted is not None and deleted[i])
           and not (inner_radius is not None and d <= inner_radius) and d <= radius]
    return [i for i, _ in out], np.array([d for _, d in out], F32), cmps, hops, second


def compare(vecs, adj, n, n_start, metric, queries, runs, deleted=None):
    oidx = O.Index(vecs, adj, n, n_start, metric)
    second = 0
    for L, beam, radius, kw in runs:
        off, ids, dists, cmps, hops, sec = R.range_search(oidx, queries, L, radius, beam=beam, deleted=deleted, **kw)
        for q in range(queries.shape[0]):
            w_ids, w_d, w_c, w_h, w_s = py_range(vecs, adj, n, n_start, metric, queries[q], L, radius, beam, deleted=deleted, **kw)
            a, b = int(off[q]), int(off[q + 1])
            what = (L, beam, radius, kw, q)
            assert ids[a:b].tolist() == w_ids, what
            assert np.array_equal(dists[a:b].view(np.uint32), w_d.view(np.uint32)), what
            assert (int(cmps[q]), int(hops[q]), bool(sec[q])) == (w_c, w_h, w_s), what
        second += int(sec.sum())
    return second


def radii(vecs, adj, n, n_start, metric, queries, L):
    want = O.Index(vecs, adj, n, n_start, metric).search_batch(queries, 3 * L, 3 * L)[1]
    return [float(np.median(want[:, i])) for i in (1, L // 2, L - 1, 3 * L - 1)]


@pytest.mark.parametrize("flavour", [O.AVX2, O.SCALAR])
def test_the_reference_baselines(flavour):
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) == 5
    for c in cases:
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        off, ids, dists, cmps, hops, second = R.range_search(O.Index(data, adj, n, 1, O.L2), np.array([c["query"]], F32), c["starting_l"],
                                                             c["radius"], inner_radius=c["inner_radius"], max_returned=c["max_returned"],
                                                             flavour=flavour)
        assert int(off[1]) == c["result_count"], c["case"]
        assert (int(cmps[0]), int(hops[0]), bool(second[0])) == (c["comparisons"], c["hops"], c["range_search_second_round"]), c["case"]
        if isinstance(c["results"], list):
            assert [[int(i), float(d)] for i, d in zip(ids, dists)] == c["results"], c["case"]
        assert len(set(ids.tolist())) == len(ids), c["case"]


def test_hops_count_the_first_phase_twice():
    """max_results_respected_and_second_round_triggered: 12 hops = 5 (phase 1) + (5 + 2)"""
    c = next(c for c in json.load(open(GOLDEN))["cases"] if c["case"] == "max_results_respected_and_second_round_triggered")
    data, adj, n = lattice(c["grid_dims"], c["grid_size"])
    oidx = O.Index(data, adj, n, 1, O.L2)
    q = np.array([c["query"]], F32)
    assert oidx.search_batch(q, 4, c["starting_l"])[4][0] == 5
    assert R.range_search(oidx, q, c["starting_l"], c["radius"], max_returned=5)[4][0] == 12


@pytest.mark.parametrize("beam", [1, 4, 64])
def test_random_graphs(beam):
    rng = np.random.default_rng(beam)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 600, 16, 12, 24)
    queries = (vecs[rng.integers(0, 600, 12)] + 0.1 * rng.normal(size=(12, 16))).astype(F32)
    runs = [(L, beam, r, {}) for L in (1, 8, 30) for r in radii(vecs, adj, 600, 1, O.L2, queries, max(L, 2))]
    assert compare(vecs, adj, 600, 1, O.L2, queries, runs) > 0


@pytest.mark.parametrize("dt,metric", [(np.float16, O.INNER_PRODUCT), (np.int8, O.COSINE), (np.uint8, O.L2)])
def test_row_types(dt, metric):
    rng = np.random.default_rng(17)
    vecs, adj, maxdeg = make_index(rng, dt, metric, 500, 24, 12, 24)
    queries = vecs[rng.integers(0, 500, 8)]
    runs = [(10, 2, r, {}) for r in radii(vecs, adj, 500, 1, metric, queries, 10)]
    compare(vecs, adj, 500, 1, metric, queries, runs)


def test_every_argument_the_reference_accepts():
    rng = np.random.default_rng(4)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 500, 16, 12, 24)
    queries = (vecs[rng.integers(0, 500, 6)] + 0.1 * rng.normal(size=(6, 16))).astype(F32)
    L = 12
    r = radii(vecs, adj, 500, 1, O.L2, queries, L)
    runs = []
    for radius in (r[2], r[3]):
        for mr in (None, L, L + 1, L + 23):
            for islack in (0.0, 0.5, 1.0):
                for rslack in (1.0, 1.5, float("inf")):
                    for inner in (None, radius / 4):
                        runs.append((L, 1 + (len(runs) % 2) * 3, radius, dict(max_returned=mr, initial_slack=islack, range_slack=rslack,
                                                                              inner_radius=inner)))
    runs += [(L, 1, float("nan"), dict(initial_slack=s)) for s in (0.0, 0.05, 1.0)]
    runs += [(L, 1, 0.0, dict(range_slack=float("inf"), initial_slack=0.0)), (L, 1, r[2], dict(range_slack=float("nan")))]
    runs += [(L, 1, r[2], dict(inner_radius=float("nan")))]
    compare(vecs, adj, 500, 1, O.L2, queries, runs)
    # a NaN radius: nothing in range; with L * initial_slack < 1 the second round runs on an empty frontier and the hops
    # are counted twice
    oidx = O.Index(vecs, adj, 500, 1, O.L2)
    got = R.range_search(oidx, queries, L, float("nan"), initial_slack=0.05)
    assert got[5].all() and int(got[0][-1]) == 0
    assert np.array_equal(got[4], 2 * oidx.search_batch(queries, L, L)[4])
    got = R.range_search(oidx, queries, L, float("nan"))
    assert not got[5].any()
    # a cap cuts a second-round hop: exactly max_returned entries were kept (none filtered at this radius)
    got = R.range_search(oidx, queries, L, r[3], max_returned=L + 23, initial_slack=0.0)
    assert (np.diff(got[0].astype(np.int64)) <= L + 23).all()


def test_edge_graphs():
    cases = [many_starts(300, 8, 2, 6, 2), many_starts(300, 8, 40, 6, 40), grid(300, 6, 3, 6, 3)]
    cases += [malformed_case(150, 6, 3, md, 6, md) for md in (1, 7, 40)]
    cases += [non_finite(200, 8, dt, m, 6, 7, nan=dt == F32)[0] for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2))]
    for case in cases:
        runs = [(L, beam, r, {}) for L in (1, 12) for beam in (1, 4)
                for r in radii(case.vecs, case.adj, case.n, case.n_start, case.metric, case.queries, max(L, 2))]
        compare(case.vecs, case.adj, case.n, case.n_start, case.metric, case.queries, runs)


def test_deleted_ids_are_walked_but_not_returned():
    rng = np.random.default_rng(5)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 500, 16, 12, 24)
    queries = (vecs[rng.integers(0, 500, 8)] + 0.1 * rng.normal(size=(8, 16))).astype(F32)
    deleted = np.zeros(501, bool)
    deleted[rng.choice(500, 120, replace=False)] = True
    r = radii(vecs, adj, 500, 1, O.L2, queries, 10)
    runs = [(10, 1, x, {}) for x in r] + [(10, 2, r[3], dict(max_returned=30))]
    compare(vecs, adj, 500, 1, O.L2, queries, runs, deleted)
    oidx = O.Index(vecs, adj, 500, 1, O.L2)
    got = R.range_search(oidx, queries, 10, r[3], deleted=deleted)
    assert not deleted[got[1]].any()
    # the walk is the same with and without the deletions: only the output differs
    assert np.array_equal(got[4], R.range_search(oidx, queries, 10, r[3])[4])


def test_argument_validation():
    """range_search.rs:515-550, and each check's boundary"""
    assert R.check(100, 0.5) is None
    assert R.check(0, 0.5) == "LZero"
    assert R.check(100, 0.5, initial_slack=1.5) == "StartingListSlackValueError"
    assert R.check(100, 0.5, range_slack=0.5) == "RangeSearchSlackValueError"
    assert R.check(100, 0.5, inner_radius=1.0) == "InnerRadiusValueError"
    assert R.check(100, 0.5, max_returned=1) == "MaxReturnedLessThanInitialL"
    assert R.check(100, 0.5, beam=0) == "BeamWidthZero"
    assert R.check(100, 0.8, beam=8, inner_radius=0.3, initial_slack=0.9, range_slack=1.2, max_returned=101) is None
    nan, inf = float("nan"), float("inf")
    assert R.check(100, 0.5, max_returned=100) is None
    assert R.check(100, 0.5, initial_slack=0.0) is None and R.check(100, 0.5, initial_slack=1.0) is None
    assert R.check(100, 0.5, initial_slack=nan) == "StartingListSlackValueError"
    assert R.check(100, 0.5, initial_slack=-0.0) is None
    assert R.check(100, 0.5, range_slack=nan) is None and R.check(100, 0.5, range_slack=inf) is None
    assert R.check(100, 0.5, inner_radius=nan) is None and R.check(100, nan, inner_radius=0.1) is None
    assert R.check(100, 0.5, inner_radius=0.5) is None
    # the reference's order: the first failing check names the error
    assert R.check(0, 0.5, beam=0, initial_slack=2.0) == "BeamWidthZero"
    assert R.check(100, 0.5, max_returned=1, initial_slack=2.0, range_slack=0.0) == "MaxReturnedLessThanInitialL"
    assert R.check(100, 0.5, initial_slack=2.0, range_slack=0.0, inner_radius=1.0) == "StartingListSlackValueError"
