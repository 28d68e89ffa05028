"""Checking and trimming a device graph: dab_count_reachable (DiskANNIndex::count_reachable_nodes), dab_degree_stats
(get_degree_stats) and dab_prune_range (prune_range).

The expected values are the restatements below, each a literal transcription of the reference's loop
(diskann/src/graph/index.rs:2161-2240 and 2656-2700): the VecDeque / HashSet walk, the DegreeStats loop in f32, and
prune_range over the oracle's robust_prune with the pool rule the library documents (distinct ids, itself and ids
without a row left out), as consolidate_node in test_delete_consolidate.py restates consolidate_vector.

CPU: the restatements reproduce the reference's own facts (the 3 x 3 grid reaches 9 nodes, 7 after the in-place
multi-delete; after prune_range the maximum degree is at most pruned_degree, as in test_final_prune).
GPU: the three calls equal the restatements, word for word and bit for bit."""
import ctypes as C
from collections import deque

import numpy as np
import pytest

import inplace_delete_oracle as D
import oracle_lib as O
from test_delete_consolidate import MAX_OCCLUSION, built, rows
from test_inplace_delete import grid3

# ---------------------------------------------------------------- the restatements


def lists_of(adj):
    max_degree = adj.shape[1] - 1
    return lambda v: [int(x) for x in adj[v, 1:1 + min(int(adj[v, 0]), max_degree)]]


def count_reachable(adj, start_points):
    """count_reachable_nodes: (expanded ids, the ids >= n_total the walk reached).  The reference fails on the first
    such id it pops (get_neighbors has no list for it); the walk here records it and goes on."""
    n_total, row = adj.shape[0], lists_of(adj)
    expanded, strays = set(), set()
    queue = deque(int(s) for s in start_points)
    while queue:
        v = queue.popleft()
        if v in expanded or v in strays:
            continue
        if v >= n_total:
            strays.add(v)
            continue
        expanded.add(v)
        queue.extend(row(v))
    return len(expanded), strays


def degree_stats(adj, ids):
    """get_degree_stats: (max_degree, avg_degree as f32, min_degree, cnt_less_than_two)"""
    row = lists_of(adj)
    max_d, min_d, total, less_than_two, count = 0, None, 0, 0, 0
    for v in ids:
        count += 1
        k = len(row(int(v)))
        max_d = max(max_d, k)
        min_d = k if min_d is None else min(min_d, k)
        total += k
        less_than_two += k < 2
    if count == 0:
        return 0, np.float32(0), 0, 0
    return max_d, np.float32(total) / np.float32(count), min_d, less_than_two


def prune_range(vecs, adj, n_points, n_start, metric, ids, degree, alpha=1.2):
    """prune_range over `ids` in order: (new adjacency, lists written)"""
    adj = np.array(adj, np.uint32, copy=True)
    n_total = adj.shape[0]
    oidx = O.Index(vecs, adj.copy(), n_points, n_start, metric)
    row = lists_of(adj)
    written = 0
    for v in ids:
        v = int(v)
        lst = row(v)
        if len(lst) <= degree:
            continue
        pool, seen = [], set()
        for u in lst:  # robust_prune_list: id itself out, and view.get finds no row for an id >= n_total
            if u != v and u < n_total and u not in seen:
                seen.add(u)
                pool.append(u)
        new = []
        if pool:
            p_ids = np.array(pool, np.uint32)
            d = O.distance_rows(oidx.vectors[v], oidx.vectors[p_ids], metric, flavour=O.AVX2)
            order = np.argsort(d, kind="stable")[:MAX_OCCLUSION]
            p_ids, d = np.ascontiguousarray(p_ids[order]), np.ascontiguousarray(d[order])
            pos = np.zeros(len(p_ids), np.uint32)
            excl = np.zeros(len(p_ids), np.uint8)
            found = O.lib().orc_robust_prune(C.byref(oidx.c), O.ptr(p_ids), O.ptr(d), O.ptr(excl), len(p_ids), degree, alpha, O.AVX2,
                                              O.ptr(pos), None)
            new = [int(x) for x in p_ids[pos[:found]]]
        adj[v, 0] = len(new)
        adj[v, 1:1 + len(new)] = new
        written += 1
    return adj, written


# ---------------------------------------------------------------- CPU: the reference's facts

@pytest.mark.parametrize("ids,live", [([4], 9), ([0, 4, 6], 7)])
def test_grid_reaches_nine_and_seven_nodes_after_the_deletes(ids, live):
    """inplace_delete.rs on setup_2d_square_using_synthetics_grid(3): the start point reaches all 10 ids, 9 after the
    TwoHopAndOneHop delete of 4 and 7 after the multi-delete of {0, 4, 6}, the start point counted"""
    vecs, adj0 = grid3()
    assert count_reachable(adj0, [9]) == (10, set())
    adj, _ = D.inplace_delete(vecs, adj0, D.deleted_words(10), ids, 9, 1, O.L2, D.TWO_HOP_AND_ONE_HOP, 3, 4, batch_size=len(ids),
                              single=len(ids) == 1)
    assert count_reachable(adj, [9]) == (live, set())


def test_the_walk_counts_each_id_once_and_follows_deleted_ids():
    adj = rows([[1, 1, 2], [0], [3], [], [0]], 3)  # 4 is not reachable from 0; 1 is listed twice
    assert count_reachable(adj, [0]) == (4, set())
    assert count_reachable(adj, [4, 4, 0]) == (5, set())
    assert count_reachable(adj, []) == (0, set())
    adj[3, 0], adj[3, 1] = 1, 77
    assert count_reachable(adj, [0]) == (4, {77})
    assert count_reachable(adj, [4]) == (5, {77})


def test_degree_stats_loop():
    adj = rows([[1, 2, 3], [0], [], [0, 1]], 3)
    assert degree_stats(adj, range(4)) == (3, np.float32(1.5), 0, 2)
    assert degree_stats(adj, [0, 0, 1]) == (3, np.float32(7) / np.float32(3), 1, 1)
    assert degree_stats(adj, []) == (0, np.float32(0), 0, 0)


def test_final_prune_trims_every_list_to_pruned_degree():
    """test_final_prune (diskann-providers diskann_async.rs:2585-2625): after prune_range the maximum degree is at most
    pruned_degree; the built graph was above it before"""
    rng, vecs, adj0, n, maxdeg = built(3, n=500)
    pruned = 8
    before = degree_stats(adj0, range(n + 1))
    assert before[0] > pruned
    adj, written = prune_range(vecs, adj0, n, 1, O.L2, range(n + 1), pruned)
    after = degree_stats(adj, range(n + 1))
    assert after[0] <= pruned and written == int((np.minimum(adj0[:, 0], maxdeg) > pruned).sum())
    short = np.minimum(adj0[:, 0], maxdeg) <= pruned
    assert np.array_equal(adj[short], adj0[short])
    again, w2 = prune_range(vecs, adj, n, 1, O.L2, range(n + 1), pruned)  # a second pass is a no-op
    assert w2 == 0 and np.array_equal(again, adj)


# ---------------------------------------------------------------- the device against the restatements
gpu = pytest.mark.gpu
DTYPES = [np.float32, np.float16, np.int8, np.uint8]
METRICS = [O.L2, O.INNER_PRODUCT, O.COSINE]
K = 10


def device(vecs, adj, n, n_start, metric):
    import diskann_b200 as dab
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, adj.shape[1] - 1)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


def same_stats(got, want):
    assert got[0] == want[0] and got[2] == want[2] and got[3] == want[3], (got, want)
    assert np.float32(got[1]).view(np.uint32) == np.float32(want[1]).view(np.uint32), (got, want)


def check_stats(g, adj, n_start, start_lists=(), id_lists=()):
    n_total = adj.shape[0]
    assert g.count_reachable() == count_reachable(adj, range(n_total - n_start, n_total))[0]
    for s in start_lists:
        assert g.count_reachable(s) == count_reachable(adj, s)[0], s
    same_stats(g.degree_stats(), degree_stats(adj, range(n_total)))
    for ids in id_lists:
        same_stats(g.degree_stats(ids), degree_stats(adj, ids))


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("metric", METRICS)
def test_device_stats_on_built_graphs(dt, metric):
    rng, vecs, adj, n, maxdeg = built(21 + metric, n=600, dt=dt, metric=metric)
    with device(vecs, adj, n, 1, metric) as g:
        check_stats(g, adj, 1, start_lists=[[0], rng.choice(n, 5), [n, n, 3, 3], []],
                    id_lists=[rng.choice(n + 1, 50), [n, n, 0], [], np.arange(n + 1)])


@gpu
def test_device_stats_on_edge_graphs():
    """disconnected components, isolated nodes, many start points, explicit lists with duplicates, an empty list"""
    rng = np.random.default_rng(3)
    n, n_start, R = 3000, 24, 16
    vecs = rng.normal(size=(n + n_start, 8)).astype(np.float32)
    lists = []
    for v in range(n):
        comp = v // 1000  # three components; every 37th node is isolated, every 41st lists only itself
        if v % 37 == 0:
            lists.append([])
        elif v % 41 == 0:
            lists.append([v])
        else:
            lists.append(list(comp * 1000 + rng.choice(1000, rng.integers(1, R + 1), replace=False)))
    for s in range(n_start):  # the start points reach the first two components only
        lists.append(list(rng.choice(2000, 4, replace=False)))
    adj = rows(lists, R)
    want = count_reachable(adj, range(n, n + n_start))[0]
    assert want < n
    with device(vecs, adj, n, n_start, O.L2) as g:
        check_stats(g, adj, n_start, start_lists=[[2500], [37], [41], [0, 0, 1000, 1000, 2999], list(range(n, n + n_start)) * 2, []],
                    id_lists=[[37, 41, 41, n + 3], rng.choice(n + n_start, 777)])


@gpu
def test_device_count_after_deletes():
    """after dab_delete -> dab_consolidate, and after dab_inplace_delete with num_to_replace 0, nodes become unreachable"""
    rng, vecs, adj0, n, maxdeg = built(5, n=800)
    ids = rng.choice(n, 400, replace=False)
    with device(vecs, adj0, n, 1, O.L2) as g:
        g.delete(ids)
        assert g.count_reachable() == count_reachable(adj0, [n])[0]  # deleted ids are walked like any other
        g.consolidate(12)
        adj = g.download_graph()
        check_stats(g, adj, 1, start_lists=[ids[:5]], id_lists=[ids])
    with device(vecs, adj0, n, 1, O.L2) as g:
        g.inplace_delete(ids, 0, "one_hop", 12, batch_size=0)
        adj = g.download_graph()
        got = g.count_reachable()
        assert got == count_reachable(adj, [n])[0] and got < n + 1 - len(ids)
        check_stats(g, adj, 1, start_lists=[ids[:5]], id_lists=[ids])


@gpu
def test_device_count_at_one_million_points():
    """1M points, max_degree 84 (C2's adjacency shape): the count equals a host walk of the downloaded adjacency"""
    import diskann_b200 as dab
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    rng = np.random.default_rng(11)
    n, maxdeg = 1_000_000, 84
    deg = rng.integers(0, maxdeg + 1, n + 1).astype(np.uint32)
    adj = np.zeros((n + 1, maxdeg + 1), np.uint32)
    adj[:, 0] = deg
    # ids below 900K link anywhere below 900K, the rest only among themselves: the start point (id n) reaches the first part
    hi = np.where(np.arange(n + 1) < 900_000, 900_000, n)[:, None]
    lo = np.where(np.arange(n + 1) < 900_000, 0, 900_000)[:, None]
    adj[:, 1:] = (lo + rng.integers(0, 1 << 30, (n + 1, maxdeg)) % (hi - lo)).astype(np.uint32)
    adj[n, 0], adj[n, 1:5] = 4, [1, 2, 3, 4]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, 4, n, 1, maxdeg) as g:
        g.upload_graph(adj)
        got = g.count_reachable()
        down = g.download_graph()
        got_many = g.count_reachable([950_000, 10])
    assert np.array_equal(down, adj)
    mask = np.arange(maxdeg)[None, :] < down[:, :1]
    src = np.repeat(np.arange(n + 1), mask.sum(1))
    graph = csr_matrix((np.ones(len(src), np.int8), (src, down[:, 1:][mask])), shape=(n + 1, n + 1))
    want = len(breadth_first_order(graph, n, directed=True, return_predecessors=False))
    assert got == want and 1 < want < n
    want_many = len(np.union1d(breadth_first_order(graph, 950_000, return_predecessors=False),
                               breadth_first_order(graph, 10, return_predecessors=False)))
    assert got_many == want_many


@gpu
def test_device_stray_ids():
    """a stray id the walk reaches fails naming the smallest; one it never reaches is ignored"""
    import diskann_b200 as dab
    rng, vecs, adj, n, maxdeg = built(9, n=300)
    adj = adj.copy()
    reach = [v for v in range(n) if adj[v, 0] > 1][:2]
    adj[reach[0], 1] = n + 50
    adj[reach[1], 2] = 0xFFFFFFF0
    iso = rows([[]], maxdeg)[0]
    adj[7] = iso  # 7 lists nothing: nothing is reached from it ...
    with device(vecs, adj, n, 1, O.L2) as g:
        with pytest.raises(dab.DabError) as e:
            g.count_reachable()
        assert e.value.code == 1 and f"reached id {n + 50}," in str(e.value)
        assert g.count_reachable([7]) == 1
        for bad in ([n + 1], [0, 5, n + 9]):
            with pytest.raises(dab.DabError) as e:
                g.count_reachable(bad)
            assert e.value.code == 1 and f"id {bad[-1]} out of range" in str(e.value)
        with pytest.raises(dab.DabError) as e:
            g.degree_stats([3, n + 1])
        assert e.value.code == 1
    adj[reach[0], 1] = 0xFFFFFFFF  # ... and an unreached list may hold strays
    lone = rows([[0xFFFFFFF5, 3]], maxdeg)[0]
    adj[8] = lone
    for v in range(n + 1):  # take 8 out of every list
        lst = [int(x) for x in adj[v, 1:1 + adj[v, 0]] if x != 8]
        adj[v] = rows([lst], maxdeg)[0]
    want, strays = count_reachable(adj, [n])
    assert 0xFFFFFFF5 not in strays
    with device(vecs, adj, n, 1, O.L2) as g:
        with pytest.raises(dab.DabError) as e:
            g.count_reachable()
        assert f"reached id {min(strays)}," in str(e.value)
        adj[reach[0], 1] = 1
        adj[reach[1], 2] = 1
        g.upload_graph(adj)
        assert g.count_reachable() == count_reachable(adj, [n])[0]
        assert count_reachable(adj, [n])[1] == set()


def check_prune(vecs, adj, n, n_start, metric, ids, degree, alpha=1.2, deleted=()):
    want, w_written = prune_range(vecs, adj, n, n_start, metric, ids if ids is not None else range(adj.shape[0]), degree, alpha)
    with device(vecs, adj, n, n_start, metric) as g:
        if len(deleted):
            g.delete(deleted)
        written = g.prune_range(ids, degree, alpha)
        got = g.download_graph()
    bad = np.flatnonzero((got != want).any(1))
    assert len(bad) == 0, (bad[:5], got[bad[:1]], want[bad[:1]])
    assert written == w_written
    return got


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("metric", METRICS)
def test_device_prune_range_equals_the_restatement(dt, metric):
    rng, vecs, adj, n, maxdeg = built(31 + metric, n=600, dt=dt, metric=metric)
    assert (adj[:, 0] > 8).any() and (adj[:, 0] <= 8).any()  # short and long lists
    check_prune(vecs, adj, n, 1, metric, None, 8)
    ids = rng.choice(n + 1, 200)  # repeats
    check_prune(vecs, adj, n, 1, metric, ids, 6, alpha=1.0, deleted=rng.choice(n, 50, replace=False))


@gpu
def test_device_prune_range_edge_lists():
    """stray ids, self-loops and repeats in over-full lists, deleted ids pruned like any other, exact ties (a lattice),
    many start points, and a list left with no pool at all"""
    rng = np.random.default_rng(13)
    side, n_start, R = 14, 12, 24
    grid = np.array([[x, y] for x in range(side) for y in range(side)], np.float32)
    n = grid.shape[0]
    vecs = np.concatenate([grid, rng.uniform(0, side, (n_start, 2)).astype(np.float32)])
    lists = [list(rng.choice(n + n_start, rng.integers(0, R + 1), replace=False)) for _ in range(n + n_start)]
    lists[3] = [3, 100000, 5, 5, 0xFFFFFFFF] + lists[3][:15]
    lists[4] = [4] + [n + n_start + i for i in range(12)]  # nothing left for the pool
    lists[5] = [6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 7]
    adj = rows(lists, R)
    deleted = rng.choice(n, 40, replace=False)
    ids = np.concatenate([[3, 4, 5, 3], deleted, rng.choice(n + n_start, 100)])
    got = check_prune(vecs, adj, n, n_start, O.L2, ids, 5, deleted=deleted)
    assert got[4, 0] == 0 and got[5, 0] <= 2
    check_prune(vecs, adj, n, n_start, O.L2, None, 5)
    check_prune(vecs, adj, n, n_start, O.COSINE, None, 10, alpha=1.4)


@gpu
@pytest.mark.parametrize("metric", METRICS)
def test_device_searches_and_stores_after_prune_range(metric):
    """searches on the pruned graph equal the oracle's searches on it; the rows, the PQ codes and the MinMax rows are
    byte-unchanged"""
    rng, vecs, adj, n, maxdeg = built(41 + metric, n=800, d=32, metric=metric)
    want, _ = prune_range(vecs, adj, n, 1, metric, range(n + 1), 8)
    queries = rng.normal(size=(48, vecs.shape[1])).astype(np.float32)
    probe = rng.choice(n + 1, (48, 20)).astype(np.uint32)
    with device(vecs, adj, n, 1, metric) as g:
        g.pq_train(vecs[:n], 8, 64, 2, 1)
        g.pq_encode_all()
        g.upload_minmax(8, 1.0)
        g.minmax_encode_all()
        pq0, mm0, d0 = g.download_pq(), g.download_minmax(), g.distances(queries, probe)
        assert g.prune_range(None, 8) > 0
        assert np.array_equal(g.download_graph(), want)
        for a, b in zip(g.download_pq(), pq0):
            assert np.array_equal(a, b)
        assert np.array_equal(g.download_minmax(), mm0)
        assert np.array_equal(g.distances(queries, probe).view(np.uint32), d0.view(np.uint32))
        got = g.search_batch(queries, K, 40)
    ref = O.Index(vecs, want, n, 1, metric).search_batch(queries, K, 40, threads=4)
    for a, b, name in zip(got, ref, ("ids", "dists", "counts", "cmps", "hops")):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), name


@gpu
def test_device_refusals_in_flight_and_paging():
    import diskann_b200 as dab
    rng, vecs, adj, n, maxdeg = built(51, n=600)
    q = rng.normal(size=(16, vecs.shape[1])).astype(np.float32)
    with device(vecs, adj, n, 1, O.L2) as g:
        graph = g.download_graph()
        for kw in (dict(pruned_degree=0), dict(pruned_degree=maxdeg + 1), dict(pruned_degree=8, alpha=0.5),
                   dict(pruned_degree=8, ids=[1, 2, n + 1])):
            with pytest.raises(dab.DabError) as e:
                g.prune_range(kw.pop("ids", None), **kw)
            assert e.value.code == 1
        assert f"id {n + 1} out of range" in str(e.value)
        assert np.array_equal(g.download_graph(), graph)
        # a batch in flight: the two read-only calls run, the prune is refused
        g.search_batch_async(2, q, K, 40)
        assert g.count_reachable() == count_reachable(adj, [n])[0]
        same_stats(g.degree_stats(), degree_stats(adj, range(n + 1)))
        with pytest.raises(dab.DabError) as e:
            g.prune_range(None, 8)
        assert e.value.code == 1 and "slot 2" in str(e.value)
        g.wait(2)
        assert np.array_equal(g.download_graph(), graph)
        # a paged session survives a prune that writes nothing and the read-only calls, and fails after a rewrite
        s = dab.PagedSearch(g, q, 40)
        s.next_page(K)
        assert g.prune_range(None, maxdeg) == 0 and g.prune_range([], 8) == 0
        g.count_reachable()
        g.degree_stats()
        s.next_page(K)
        assert g.prune_range([int(np.argmax(adj[:n, 0]))], 8) == 1
        with pytest.raises(dab.DabError):
            s.next_page(K)
