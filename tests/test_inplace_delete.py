"""Deleting points in place: dab_inplace_delete (DiskANNIndex::multi_inplace_delete with its three repair methods) and
dab_drop_deleted_neighbors, held to the oracle of oracle/inplace_delete.cpp (tests/inplace_delete_oracle.py), which
restates the reference's routines with the chunk schedule and tie rule the library documents.

CPU: the oracle reproduces the reference's own cases (diskann/src/graph/test/cases/inplace_delete.rs and
diskann-benchmark-core's test_drop_deleted), and multi_inplace_delete at chunk size 1 equals inplace_delete id by id.
GPU: every adjacency word and the deletion table equal the oracle's."""
import numpy as np
import pytest

import inplace_delete_oracle as D
import oracle_lib as O
from test_delete_consolidate import SQUARE_LISTS, built, rows, square

METHODS = [D.VISITED_AND_TOPK, D.TWO_HOP_AND_ONE_HOP, D.ONE_HOP]
SQUARE_MAX_DEGREE = 13  # graph::config::Builder::new(10, MaxDegree::default_slack(), 15, L2): pruned 10 with 1.3 slack


def listed(adj, v):
    return sorted(int(x) for x in adj[v, 1:1 + adj[v, 0]])


def square_delete(ids, method, batch_size=0, single=False):
    vecs = square()
    adj = rows(SQUARE_LISTS, SQUARE_MAX_DEGREE)
    return D.inplace_delete(vecs, adj, D.deleted_words(5), ids, 4, 1, O.L2, method, 3, 10, k_value=4, l_value=10,
                            batch_size=batch_size, single=single)


# ---------------------------------------------------------------- the reference's cases (inplace_delete.rs)

@pytest.mark.parametrize("method", METHODS)
def test_square_delete_3(method):
    adj, deleted = square_delete([3], method, single=True)
    for v in (0, 1, 2, 4):
        assert 3 not in listed(adj, v)
    assert listed(adj, 2) and 4 in listed(adj, 2)
    assert listed(adj, 4) == [0, 1, 2]
    assert list(D.deleted_ids(deleted, 5)) == [3]
    assert adj[3, 0] == 0


@pytest.mark.parametrize("method", [D.TWO_HOP_AND_ONE_HOP, D.VISITED_AND_TOPK])
def test_square_multi_delete_2_and_3(method):
    adj, deleted = square_delete([2, 3], method, batch_size=2)
    for v in (0, 1, 4):
        assert 2 not in listed(adj, v) and 3 not in listed(adj, v)
    assert 1 in listed(adj, 0) and 4 in listed(adj, 0)
    assert 0 in listed(adj, 1) and 4 in listed(adj, 1)
    assert listed(adj, 4) == [0, 1]
    assert list(D.deleted_ids(deleted, 5)) == [2, 3]


def test_isolated_node_leaves_its_neighbours_unchanged():
    """delete_isolated_node: 2 has no neighbours and no list holds it; OneHop leaves every other list as it was"""
    vecs = square()
    lists = [[1, 4], [0, 4], [], [4], [0, 1, 3]]
    adj0 = rows(lists, SQUARE_MAX_DEGREE)
    adj, _ = D.inplace_delete(vecs, adj0, D.deleted_words(5), [2], 4, 1, O.L2, D.ONE_HOP, 3, 10, single=True)
    for v in (0, 1, 3, 4):
        assert np.array_equal(adj[v], adj0[v])


def grid3():
    """setup_2d_square_using_synthetics_grid(3, start, 4): Grid::Two's 3 x 3 lattice, point i * 3 + j at (i, j) with
    its lattice neighbours in synthetic.rs's order, and the start point (id 9) at (3, 3) whose only neighbour is 8;
    pruned degree 4, max degree the same"""
    vecs = np.array([[i, j] for i in range(3) for j in range(3)] + [[3, 3]], np.float32)
    lists = []
    for i in range(3):
        for j in range(3):
            lists.append([(i - 1) * 3 + j] * (i > 0) + [(i + 1) * 3 + j] * (i < 2) + [i * 3 + j - 1] * (j > 0) + [i * 3 + j + 1] * (j < 2))
    lists.append([8])
    return vecs, rows(lists, 4)


def reachable(adj, start):
    seen, todo = {start}, [start]
    while todo:
        v = todo.pop()
        for u in adj[v, 1:1 + adj[v, 0]]:
            if int(u) not in seen:
                seen.add(int(u))
                todo.append(int(u))
    return seen


@pytest.mark.parametrize("ids,live", [([4], 9), ([0, 4, 6], 7)])
def test_grid_stays_connected(ids, live):
    """inplace_delete_two_hop_and_one_hop_wider_topology and multi_inplace_delete_wider_topology"""
    vecs, adj0 = grid3()
    adj, _ = D.inplace_delete(vecs, adj0, D.deleted_words(10), ids, 9, 1, O.L2, D.TWO_HOP_AND_ONE_HOP, 3, 4,
                              batch_size=len(ids), single=len(ids) == 1)
    for v in range(9):
        if v not in ids:
            assert not set(ids) & set(listed(adj, v)), v
    assert len(reachable(adj, 9)) == live


def test_grid_repair_is_what_keeps_it_connected():
    """without replacements (num_to_replace 0) the multi-delete of {0, 4, 6} leaves fewer nodes reachable"""
    vecs, adj0 = grid3()
    adj, _ = D.inplace_delete(vecs, adj0, D.deleted_words(10), [0, 4, 6], 9, 1, O.L2, D.TWO_HOP_AND_ONE_HOP, 0, 4, batch_size=3)
    assert len(reachable(adj, 9)) < 7


def stray_overflow():
    """a source whose list holds a stray id and overflows max_degree when the delete appends to it"""
    vecs = np.array([[0, 0], [1, 0], [2, 0], [3, 0], [4, 0], [5, 0], [2.5, 0]], np.float32)
    lists = [[1, 0xFFFFFFF0, 5], [0, 2, 3], [1, 3, 0], [1, 2, 4], [3, 5, 2], [4, 3, 1], [0, 5]]
    return vecs, rows(lists, 3)


@pytest.mark.parametrize("method", METHODS)
def test_stray_ids_are_left_out_of_the_prune_pool(method):
    vecs, adj0 = stray_overflow()
    adj, _ = D.inplace_delete(vecs, adj0, D.deleted_words(7), [1], 6, 1, O.L2, method, 3, 3, k_value=4, l_value=10, single=True)
    assert 1 not in listed(adj, 0)
    if method != D.VISITED_AND_TOPK:  # 0 gains 2 and 3 from 1's neighbours: four ids, pruned to three without the stray one
        assert 0xFFFFFFF0 not in listed(adj, 0) and {2, 3} & set(listed(adj, 0))


def test_drop_deleted_on_a_built_graph():
    """test_drop_deleted (diskann-benchmark-core streaming/graph/drop_deleted.rs): on the graph built over Grid::Four's
    4^4 lattice (build_test_index: pruned degree 5, max degree 8, L 20, the start point at (4, 4, 4, 4)), with the even
    ids soft-deleted, drop_deleted_neighbors leaves every odd list non-empty and free of even ids."""
    n = 256
    vecs = np.array([[(i >> 6) & 3, (i >> 4) & 3, (i >> 2) & 3, i & 3] for i in range(n)] + [[4, 4, 4, 4]], np.float32)
    adj0 = O.build_graph(vecs, n, 1, O.L2, 5, 8, 20)
    words = D.deleted_words(n + 1, np.arange(0, n, 2))
    adj, written = D.drop_deleted_neighbors(adj0, words, n, 1, 5)
    assert written > 0
    for v in range(1, n, 2):
        l = listed(adj, v)
        assert l and not any(u < n and u % 2 == 0 for u in l)


@pytest.mark.parametrize("method", METHODS)
def test_multi_at_chunk_size_1_equals_single_deletes(method):
    rng, vecs, adj0, n, maxdeg = built(7, n=300)
    ids = rng.choice(n, 30, replace=False)
    pre = D.deleted_words(n + 1, rng.choice(n, 10, replace=False))
    a = D.inplace_delete(vecs, adj0, pre, ids, n, 1, O.L2, method, 3, 12, k_value=20, l_value=50, batch_size=1)
    b = D.inplace_delete(vecs, adj0, pre, ids, n, 1, O.L2, method, 3, 12, k_value=20, l_value=50, single=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------- the device against the oracle
gpu = pytest.mark.gpu
DTYPES = {np.float32: "f32", np.float16: "f16", np.int8: "i8", np.uint8: "u8"}
METRICS = [O.L2, O.INNER_PRODUCT, O.COSINE]


def device(vecs, adj, n, n_start, metric):
    import diskann_b200 as dab
    g = dab.GpuIndex(dab.DType[DTYPES[vecs.dtype.type]], dab.Metric(metric), vecs.shape[1], n, n_start, adj.shape[1] - 1)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


def check_device(vecs, adj0, n, pre, ids, metric, method, batch_size, num_to_replace=3, k_value=20, l_value=50, degree=12):
    want_adj, want_del = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1, pre), ids, n, 1, metric, method, num_to_replace, degree,
                                          k_value=k_value, l_value=l_value, batch_size=batch_size)
    with device(vecs, adj0, n, 1, metric) as g:
        if len(pre):
            g.delete(pre)
        g.inplace_delete(ids, num_to_replace, method, degree, k_value=k_value, l_value=l_value, batch_size=batch_size)
        got = g.download_graph()
        status = g.delete_status(np.arange(n, dtype=np.uint32))
    assert np.array_equal(got, want_adj)
    assert np.array_equal(np.flatnonzero(status).astype(np.uint32), D.deleted_ids(want_del, n + 1))


@gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("method", METHODS)
def test_device_equals_oracle(dt, metric, method):
    rng, vecs, adj0, n, maxdeg = built(11, n=400, dt=dt, metric=metric)
    for frac, batch_size in ((0.01, 1), (0.1, 37), (0.5, 0)):
        ids = rng.choice(n, int(n * frac), replace=False)
        pre = rng.choice(ids, len(ids) // 4, replace=False)  # some already soft-deleted
        check_device(vecs, adj0, n, pre, ids, metric, method, batch_size)


@gpu
@pytest.mark.parametrize("method", METHODS)
def test_device_edge_lists_and_parameters(method):
    rng, vecs, adj0, n, maxdeg = built(13, n=300)
    adj = adj0.copy()
    adj[5, 1:4] = [n + 7, 0xFFFFFFFF, n + 1]  # stray ids
    adj[7, 2] = adj[7, 1]                       # a repeat
    ids = np.concatenate([[int(adj[5, 4]), int(adj[7, 1])], rng.choice(np.arange(10, n), 20, replace=False)])
    ids = np.unique(ids)
    rng.shuffle(ids)
    for ntr, bs in ((0, 0), (3, 7), (5, 1)):
        check_device(vecs, adj, n, [], ids, O.L2, method, bs, num_to_replace=ntr, k_value=60, l_value=40)


@gpu
def test_device_exact_ties():
    """integer rows on a lattice: many exactly tied distances follow (distance, position in the replace candidates)"""
    rng = np.random.default_rng(3)
    n = 300
    base = rng.integers(0, 3, (n, 8)).astype(np.int8)
    vecs = np.concatenate([base, base[:1]])
    adj = O.build_graph(vecs, n, 1, O.L2, 12, 15, 30)
    for method in METHODS:
        check_device(vecs, adj, n, [], rng.choice(n, 40, replace=False), O.L2, method, 0, num_to_replace=4)


@gpu
@pytest.mark.parametrize("only_orphans", [False, True])
def test_device_drop_deleted_neighbors(only_orphans):
    rng, vecs, adj0, n, maxdeg = built(17, n=400)
    ids = rng.choice(n, 60, replace=False)
    adj1, words = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1), ids[:30], n, 1, O.L2, D.ONE_HOP, 3, 12)
    words = D.deleted_words(n + 1, ids)  # half of them soft-deleted only: their lists stay
    want, want_n = D.drop_deleted_neighbors(adj1, words, n, 1, 12, only_orphans)
    with device(vecs, adj1, n, 1, O.L2) as g:
        g.delete(ids)
        got_n = g.drop_deleted_neighbors(12, only_orphans)
        got = g.download_graph()
    assert np.array_equal(got, want) and got_n == want_n


@gpu
def test_device_search_after_and_release_insert():
    """searches on the repaired graph equal the oracle's, and release -> insert reuses the ids"""
    import insert_oracle as I
    rng, vecs, adj0, n, maxdeg = built(19, n=500)
    ids = rng.choice(n, 50, replace=False)
    want_adj, words = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1), ids, n, 1, O.L2, D.VISITED_AND_TOPK, 3, 12, batch_size=0)
    queries = rng.normal(size=(32, vecs.shape[1])).astype(np.float32)
    oidx = O.Index(vecs, want_adj, n, 1, O.L2)
    full = oidx.search_batch(queries, 30 + 1, 30)
    with device(vecs, adj0, n, 1, O.L2) as g:
        g.inplace_delete(ids, 3, "visited_and_topk", 12, batch_size=0)
        got = g.search_batch(queries, 10, 30)
        for q in range(len(queries)):
            live = [int(x) for x in full[0][q] if x != 0xFFFFFFFF and x < n and x not in set(ids.tolist())][:10]
            assert [int(x) for x in got[0][q][:len(live)]] == live
        g.release(ids)
        fresh = rng.normal(size=(len(ids), vecs.shape[1])).astype(np.float32)
        g.insert(ids, fresh, 12, 30)
        got_adj = g.download_graph()
    vecs2 = vecs.copy()
    vecs2[ids] = fresh
    released = want_adj.copy()
    released[ids, 0] = 0
    want2 = I.insert_batched(vecs2, released, ids, n, 1, O.L2, 12, maxdeg, 30)
    assert np.array_equal(got_adj, want2)


@gpu
def test_device_refusals_change_nothing():
    import diskann_b200 as dab
    rng, vecs, adj0, n, maxdeg = built(23, n=200)
    with device(vecs, adj0, n, 1, O.L2) as g:
        g.delete([5])
        bad = [([n], {}), ([3, 3], {}), ([3], {"method": 7}), ([3], {"pruned_degree": 0}), ([3], {"pruned_degree": maxdeg + 1}),
               ([3], {"alpha": 0.5}), ([3], {"l_value": 0}), ([3], {"l_value": 1024})]
        for ids, kw in bad:
            args = dict(num_to_replace=3, method=0, pruned_degree=12)
            args.update(kw)
            with pytest.raises(dab.DabError):
                g.inplace_delete(ids, **args)
            assert np.array_equal(g.download_graph(), adj0)
            assert list(np.flatnonzero(g.delete_status(np.arange(n, dtype=np.uint32)))) == [5]
        with pytest.raises(dab.DabError):
            g.drop_deleted_neighbors(0)


@gpu
@pytest.mark.parametrize("method", METHODS)
def test_device_stray_id_in_an_overflowing_list(method):
    vecs, adj0 = stray_overflow()
    for bs in (1, 0):
        check_device(vecs, adj0, 6, [], [1], O.L2, method, bs, k_value=4, l_value=10, degree=3)


@gpu
@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("store", ["fp", "pq", "sq", "minmax"])
def test_device_searches_after_the_delete(monkeypatch, tables, store):
    """k-NN searches over the repaired graph (full precision, PQ, SQ, MinMax, with and without rerank, and with visited
    tables small enough to force the overflow re-run) equal the oracle's on the oracle's graph, ids, distances, counts,
    cmps and hops; the quantized store is byte-unchanged"""
    import diskann_b200 as dab
    from test_delete_consolidate import K, filtered
    from test_minmax_search import MinMaxOracle, compress, make_transform
    from test_quantized_in_flight import minmax_case, pq_case, sq_case
    if tables == "overflow":
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    L = 60
    if store in ("fp", "pq"):
        n, d, vecs, adj0, maxdeg, piv, off, codes, batches, _ = pq_case(O.L2)
    elif store == "sq":
        n, d, vecs, adj0, maxdeg, quantizer, sq_rows, batches, _ = sq_case(O.L2, 8)
    else:
        n, d, vecs, adj0, maxdeg, mm_rows, batches, _ = minmax_case(8, None)
    rng = np.random.default_rng(29)
    ids = rng.choice(n, n // 20, replace=False)
    adj, words = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1), ids, n, 1, O.L2, D.VISITED_AND_TOPK, 3, maxdeg, batch_size=0)
    deleted = np.zeros(n + 1, bool)
    deleted[ids] = True
    q = batches[0]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        if store == "pq":
            g.upload_pq(piv, off, codes)
            rows_of = g.download_pq
        elif store == "sq":
            g.upload_sq(*quantizer, rows=sq_rows)
            rows_of = g.download_sq
        elif store == "minmax":
            g.upload_minmax(8, 1.0, make_transform(None, d), rows=mm_rows)
            rows_of = g.download_minmax
        before = rows_of() if store != "fp" else None
        g.inplace_delete(ids, 3, "visited_and_topk", maxdeg, batch_size=0)
        assert np.array_equal(g.download_graph(), adj)
        if store != "fp":
            for a, b in zip(before if store == "pq" else [before], rows_of() if store == "pq" else [rows_of()]):
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
        for r in ((False,) if store == "fp" else (False, True)):
            if store == "fp":
                full = O.Index(vecs, adj, n, 1, O.L2).search_batch(q, L + 1, L, threads=4)
                got = g.search_batch(q, K, L)
            elif store == "pq":
                oidx = O.Index(vecs, adj, n, 1, O.L2, pq=(piv, off, codes))
                full = (oidx.search_batch_rerank if r else oidx.search_batch)(q, L + 1, L, threads=4)
                got = g.search_batch_pq(q, K, L, 1, rerank=r)
            elif store == "sq":
                oidx = O.Index(vecs, adj, n, 1, O.L2, sq=(sq_rows,) + tuple(quantizer))
                full = (oidx.search_batch_rerank if r else oidx.search_batch)(q, L + 1, L, threads=4)
                got = g.search_batch_sq(q, K, L, 1, rerank=r)
            else:
                full = MinMaxOracle(vecs, adj, n, 1, O.L2, mm_rows, 8).search(q, compress(q, None, 8), L + 1, L, rerank=r)
                got = g.search_batch_minmax(q, K, L, 1, rerank=r)
            for a, b in zip(got, filtered(full, deleted, K)):
                assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (store, r, tables)


@gpu
def test_device_refusals_generation_and_paged_sessions():
    """refusals leave the graph, the table and open paged sessions alone; a call that writes a list ends them"""
    import ctypes as C
    import diskann_b200 as dab
    from diskann_b200 import _lib
    rng, vecs, adj0, n, maxdeg = built(31, n=200)
    q = rng.normal(size=(8, vecs.shape[1])).astype(np.float32)
    with device(vecs, adj0, n, 1, O.L2) as g:
        g.delete([5])
        s = dab.PagedSearch(g, q, 40)
        s.next_page(10)
        # NULL ids with n > 0
        assert _lib.lib().dab_inplace_delete(g._h, None, 3, 0, 3, 20, 50, 12, C.c_float(1.2), 1) == 1
        assert _lib.lib().dab_drop_deleted_neighbors(g._h, maxdeg + 1, 0, None) == 1
        # a batch in flight
        g.search_batch_async(1, q, 10, 40)
        for call in (lambda: g.inplace_delete([3], 3, 0, 12), lambda: g.drop_deleted_neighbors(12)):
            with pytest.raises(dab.DabError) as e:
                call()
            assert e.value.code == 1 and "slot 1" in str(e.value)
        g.wait(1)
        assert np.array_equal(g.download_graph(), adj0)
        assert list(np.flatnonzero(g.delete_status(np.arange(n, dtype=np.uint32)))) == [5]
        s.next_page(10)  # the generation did not move
        g.drop_deleted_neighbors(12)  # 5 is only soft-deleted: lists that hold it are written
        with pytest.raises(dab.DabError):
            s.next_page(10)
        s.close()
        s = dab.PagedSearch(g, q, 40)
        s.next_page(10)
        g.inplace_delete([7], 3, "one_hop", 12)
        with pytest.raises(dab.DabError):
            s.next_page(10)
        s.close()
    # vectors and graph missing
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, vecs.shape[1], n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        with pytest.raises(dab.DabError) as e:
            g.inplace_delete([3], 3, "one_hop", 12)
        assert e.value.code == 5
        with pytest.raises(dab.DabError) as e:
            g.drop_deleted_neighbors(12)
        assert e.value.code == 5
