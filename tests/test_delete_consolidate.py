"""Deleting points from an index: the deletion table (dab_delete / dab_release / dab_delete_status), searches that leave
deleted ids out of their results, and dab_consolidate, which repairs the graph around them on the device.

The expected consolidation is `consolidate`, below: a literal restatement of the reference's loop
`for id in 0..n_total { consolidate_vector(id) }` (diskann/src/graph/index.rs:1819-1931) with the canonical pool order
the library documents, the oracle's Distance<T,T> and the oracle's robust_prune (occlude_list without saturation).  The
expected search results are the oracle's searches at k = L + #start with deleted ids dropped and the first k kept:
filtering commutes with the traversal-order (and stable rerank) sort, and deletions do not change the traversal."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O

MAX_OCCLUSION = 750  # graph/config/defaults.rs:13


# ---------------------------------------------------------------- the restatement

def consolidate_node(oidx, adj, deleted, v, degree, alpha):
    """consolidate_vector(v) over `adj` (rows [len, ids...]) in place; True when v's list was written."""
    n_total, max_degree = adj.shape[0], adj.shape[1] - 1
    n_points = oidx.n_points

    def dead(u):  # deleted, or a status lookup that fails
        return u >= n_total or (u < n_points and deleted[u])

    def row(u):
        return [int(x) for x in adj[u, 1:1 + min(int(adj[u, 0]), max_degree)]]

    if dead(v):
        return False  # ConsolidateKind::Deleted
    pool, seen, dels = [], set(), []
    for u in row(v):
        if dead(u):
            dels.append(u)
        elif u not in seen:
            seen.add(u)
            pool.append(u)
    if not dels and len(pool) <= degree:
        return False
    for u in dels:
        if u >= n_total:
            continue
        for w in row(u):
            if not dead(w) and w not in seen:
                seen.add(w)
                pool.append(w)
    pool = [u for u in pool if u != v]
    if len(pool) < degree:
        new = pool
    else:
        ids = np.array(pool, np.uint32)
        d = O.distance_rows(oidx.vectors[v], oidx.vectors[ids], oidx.metric, flavour=O.AVX2)
        order = np.argsort(d, kind="stable")[:MAX_OCCLUSION]  # SortedNeighbors::new, ties in pool order
        ids, d = np.ascontiguousarray(ids[order]), np.ascontiguousarray(d[order])
        pos = np.zeros(len(ids), np.uint32)
        excl = np.zeros(len(ids), np.uint8)
        found = O.lib().orc_robust_prune(C.byref(oidx.c), O.ptr(ids), O.ptr(d), O.ptr(excl), len(ids), degree, alpha, O.AVX2,
                                          O.ptr(pos), None)
        new = [int(x) for x in ids[pos[:found]]]
    adj[v, 0] = len(new)
    adj[v, 1:1 + len(new)] = new
    return True


def consolidate(vecs, adj, n_points, n_start, metric, deleted, degree, alpha=1.2, order=None):
    """(new adjacency, lists written) of consolidate_vector over every id, in `order` (default ascending)."""
    adj = np.array(adj, np.uint32, copy=True)
    oidx = O.Index(vecs, adj, n_points, n_start, metric)
    deleted = np.asarray(deleted, bool)
    written = 0
    for v in (range(adj.shape[0]) if order is None else order):
        written += consolidate_node(oidx, adj, deleted, int(v), degree, alpha)
    return adj, written


def square():
    """the 2 x 2 grid of synthetic.rs (Grid::Two) with its start point at (0.5, 0.5), id 4"""
    vecs = np.array([[0, 0], [0, 1], [1, 0], [1, 1], [0.5, 0.5]], np.float32)
    return vecs


def rows(lists, max_degree):
    adj = np.zeros((len(lists), max_degree + 1), np.uint32)
    for i, l in enumerate(lists):
        adj[i, 0] = len(l)
        adj[i, 1:1 + len(l)] = l
    return adj


def listed(adj, v):
    return sorted(int(x) for x in adj[v, 1:1 + adj[v, 0]])


SQUARE_LISTS = [[1, 4], [0, 4], [3, 4], [2, 4], [0, 1, 2, 3]]  # generate_2d_square_adjacency_list
REPAIR_LISTS = [[1, 2, 4], [0, 3, 4], [0, 3, 4], [1, 2, 4], [0, 1, 2, 3]]


# ---------------------------------------------------------------- CPU: the reference's closed-form cases

def test_consolidate_repairs_after_deletion():
    """cases/consolidate.rs consolidate_repairs_after_deletion: 3 deleted, pruned_degree 4"""
    deleted = np.array([0, 0, 0, 1], bool)
    adj, _ = consolidate(square(), rows(REPAIR_LISTS, 4), 4, 1, O.L2, deleted, 4)
    assert [listed(adj, v) for v in (0, 1, 2, 4)] == [[1, 2, 4], [0, 2, 4], [0, 1, 4], [0, 1, 2]]
    assert listed(adj, 3) == [1, 2, 4]  # a deleted node is left alone


def test_consolidate_prune_only_no_deleted_neighbors():
    """consolidate_prune_only_no_deleted_neighbors: the start node's four neighbours pruned to pruned_degree 2"""
    adj0 = rows(SQUARE_LISTS, 4)
    adj, written = consolidate(square(), adj0, 4, 1, O.L2, np.zeros(4, bool), 2)
    assert adj[4, 0] <= 2 and written == 1
    assert np.array_equal(adj[:4], adj0[:4])


def test_consolidate_nothing_to_do_and_deleted_vertex():
    """consolidate_nothing_to_do_returns_complete and consolidate_deleted_vertex_returns_deleted"""
    adj0 = rows(SQUARE_LISTS, 4)
    adj, written = consolidate(square(), adj0, 4, 1, O.L2, np.zeros(4, bool), 4)
    assert written == 0 and np.array_equal(adj, adj0)
    oidx = O.Index(square(), adj0.copy(), 4, 1, O.L2)
    assert not consolidate_node(oidx, adj0.copy(), np.array([0, 0, 0, 1], bool), 3, 4, 1.2)


def built(seed, n=600, d=16, R=12, dt=np.float32, metric=O.L2):
    rng = np.random.default_rng(seed)
    base = rng.normal(size=(n, d)).astype(np.float32)
    if dt == np.int8:
        base = np.clip(np.round(base * 40), -127, 127).astype(np.int8)
    elif dt == np.uint8:
        base = np.clip(np.round(base * 40 + 128), 0, 255).astype(np.uint8)
    elif dt == np.float16:
        base = base.astype(np.float16)
    vecs = np.concatenate([base, base[:1]])
    maxdeg = int(R * 1.3)
    adj = O.build_graph(vecs, n, 1, metric, R, maxdeg, 30)
    return rng, vecs, adj, n, maxdeg


@pytest.mark.parametrize("frac", [0.01, 0.1, 0.5])
def test_consolidation_properties_on_built_graphs(frac):
    rng, vecs, adj0, n, maxdeg = built(3)
    deleted = np.zeros(n, bool)
    deleted[rng.choice(n, max(1, int(frac * n)), replace=False)] = True
    adj, written = consolidate(vecs, adj0, n, 1, O.L2, deleted, 12)
    n_total = adj.shape[0]
    touched = np.zeros(n_total, bool)
    for v in range(n_total):
        nb = adj[v, 1:1 + adj[v, 0]]
        if v < n and deleted[v]:
            assert np.array_equal(adj[v], adj0[v])
            continue
        assert not any(u >= n_total or (u < n and deleted[u]) for u in nb), v
        touched[v] = not np.array_equal(adj[v], adj0[v])
        old = adj0[v, 1:1 + adj0[v, 0]]
        if not any(u < n and deleted[u] for u in old) and len(set(old.tolist())) <= 12:
            assert not touched[v], v  # nothing to do: byte-identical
    assert written >= touched.sum() > 0
    shuffled, written2 = consolidate(vecs, adj0, n, 1, O.L2, deleted, 12, order=rng.permutation(n_total))
    assert np.array_equal(shuffled, adj) and written2 == written
    again, written3 = consolidate(vecs, adj, n, 1, O.L2, deleted, 12)
    assert written3 == 0 and np.array_equal(again, adj)


# ---------------------------------------------------------------- GPU

gpu = pytest.mark.gpu


def device_consolidate(vecs, adj, n, n_start, metric, deleted, degree, alpha=1.2):
    import diskann_b200 as dab
    with dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, adj.shape[1] - 1) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        ids = np.flatnonzero(deleted).astype(np.uint32)
        if len(ids):
            g.delete(ids)
        written = g.consolidate(degree, alpha)
        return g.download_graph(), written


def check_consolidate(vecs, adj, n, n_start, metric, deleted, degree, alpha=1.2):
    want, w_written = consolidate(vecs, adj, n, n_start, metric, deleted, degree, alpha)
    got, g_written = device_consolidate(vecs, adj, n, n_start, metric, deleted, degree, alpha)
    bad = np.flatnonzero((got != want).any(1))
    assert len(bad) == 0, (bad[:5], got[bad[:1]], want[bad[:1]])
    assert g_written == w_written
    return got


@gpu
@pytest.mark.parametrize("dt", [np.float32, np.float16, np.int8, np.uint8])
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE])
@pytest.mark.parametrize("frac", [0.01, 0.1, 0.5])
def test_device_consolidation_equals_the_restatement(dt, metric, frac):
    rng, vecs, adj, n, maxdeg = built(11 + metric, n=800, d=24, R=12, dt=dt, metric=metric)
    deleted = np.zeros(n, bool)
    deleted[rng.choice(n, max(1, int(frac * n)), replace=False)] = True
    check_consolidate(vecs, adj, n, 1, metric, deleted, 12)
    check_consolidate(vecs, adj, n, 1, metric, deleted, 8)  # pruned_degree < the build's: every long list is pruned
    check_consolidate(vecs, adj, n, 1, metric, np.zeros(n, bool), 8)  # nothing deleted: prune only


@gpu
def test_device_consolidation_of_a_pool_beyond_750_and_stray_ids():
    """node 0 lists 40 deleted nodes with 40 distinct live neighbours each: a pool of 1600 ids (more than the prune's
    shared memory holds), cut to its 750 closest.  Other rows carry out-of-range ids, repeats and self-loops."""
    rng = np.random.default_rng(5)
    R, n = 40, 2000
    vecs = np.concatenate([rng.normal(size=(n, 8)).astype(np.float32), np.zeros((1, 8), np.float32)])
    lists = [list(rng.choice(n, R, replace=False)) for _ in range(n + 1)]
    hubs = list(range(1, 41))
    lists[0] = hubs
    live = np.arange(41, n)
    for i, h in enumerate(hubs):
        lists[h] = list(live[i * R:(i + 1) * R])
    lists[50] = [50, 51, 51, 9999, 52] + lists[50][:10]  # self-loop, repeat, out of range
    lists[60] = [60] + list(rng.choice(n, 20, replace=False))
    adj = rows(lists, R)
    deleted = np.zeros(n, bool)
    deleted[hubs] = True
    deleted[rng.choice(np.arange(2000 - 400, n), 30, replace=False)] = True
    for degree in (R, 24):
        got = check_consolidate(vecs, adj, n, 1, O.L2, deleted, degree)
        assert got[0, 0] > 0


@gpu
def test_device_consolidation_of_the_closed_form_cases():
    got = check_consolidate(square(), rows(REPAIR_LISTS, 4), 4, 1, O.L2, np.array([0, 0, 0, 1], bool), 4)
    assert [listed(got, v) for v in (0, 1, 2, 4)] == [[1, 2, 4], [0, 2, 4], [0, 1, 4], [0, 1, 2]]
    got = check_consolidate(square(), rows(SQUARE_LISTS, 4), 4, 1, O.L2, np.zeros(4, bool), 2)
    assert got[4, 0] <= 2
    adj0 = rows(SQUARE_LISTS, 4)
    got, written = device_consolidate(square(), adj0, 4, 1, O.L2, np.zeros(4, bool), 4)
    assert written == 0 and np.array_equal(got, adj0)


@gpu
def test_device_consolidation_on_edge_graphs():
    """many start points, exact ties (a lattice) and stray ids"""
    rng = np.random.default_rng(9)
    side = 12
    grid = np.array([[x, y] for x in range(side) for y in range(side)], np.float32)
    n, n_start, R = grid.shape[0], 20, 10
    vecs = np.concatenate([grid, rng.uniform(0, side, (n_start, 2)).astype(np.float32)])
    adj = O.build_graph(vecs, n, n_start, O.L2, 8, R, 20)
    adj[7, 1] = 100000  # out of range
    deleted = np.zeros(n, bool)
    deleted[rng.choice(n, 30, replace=False)] = True
    check_consolidate(vecs, adj, n, n_start, O.L2, deleted, 8)
    check_consolidate(vecs, adj, n, n_start, O.L2, deleted, 5)


# ---- searches with tombstones

K = 10


def filtered(full, deleted, k):
    """the oracle's results at k' = L + #start -> RemoveDeletedIdsAndCopy: the first k entries that are not deleted"""
    ids, dists, counts, cmps, hops = full
    nq = ids.shape[0]
    out_i = np.full((nq, k), 0xFFFFFFFF, np.uint32)
    out_d = np.full((nq, k), np.inf, np.float32)
    out_c = np.zeros(nq, np.uint32)
    for q in range(nq):
        keep = [j for j in range(counts[q]) if not deleted[ids[q, j]]][:k]
        out_i[q, :len(keep)] = ids[q, keep]
        out_d[q, :len(keep)] = dists[q, keep]
        out_c[q] = len(keep)
    return out_i, out_d, out_c, cmps, hops


def in_flight_helpers():
    from test_quantized_in_flight import check_in_flight, minmax_case, pq_case, same, sq_case
    return check_in_flight, pq_case, sq_case, minmax_case, same


@gpu
@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("L", [16, 200])  # search_kernel_v3 (short lists) and search_kernel_v2
@pytest.mark.parametrize("frac", [0.05, 0.9])
def test_full_precision_search_with_tombstones(monkeypatch, tables, L, frac):
    import diskann_b200 as dab
    check_in_flight, pq_case, _, _, _ = in_flight_helpers()
    if tables == "overflow":
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    n, d, vecs, adj, maxdeg, _, _, _, batches, _ = pq_case(O.L2)
    rng = np.random.default_rng(int(frac * 100) + L)
    deleted = np.zeros(n + 1, bool)
    deleted[rng.choice(n, int(frac * n), replace=False)] = True
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    full = [oidx.search_batch(q, L + 1, L, threads=4) for q in batches]
    want = [filtered(f, deleted, K) for f in full]
    if frac > 0.5:
        assert any((w[2] < K).any() for w in want)  # counts fall below k
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        before = [g.search_batch(q, K, L) for q in batches]
        g.delete(np.flatnonzero(deleted))
        check_in_flight(g, lambda q, r: g.search_batch(q, K, L), lambda s, q, r: g.search_batch_async(s, q, K, L),
                        lambda s, *a, rerank: g.search_batch_device_async(s, a[0], a[1], K, L, 1, *a[2:]),
                        batches, {False: want, True: want}, ("fp", L, frac, tables))
        for b, w in zip(before, want):  # the traversal does not change
            assert np.array_equal(b[3], w[3]) and np.array_equal(b[4], w[4])


@gpu
@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("store", ["pq", "sq", "minmax"])
def test_quantized_search_with_tombstones(monkeypatch, tables, store):
    import diskann_b200 as dab
    from test_minmax_search import MinMaxOracle, compress, make_transform
    check_in_flight, pq_case, sq_case, minmax_case, _ = in_flight_helpers()
    if tables == "overflow":
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    L = 60
    if store == "pq":
        n, d, vecs, adj, maxdeg, piv, off, codes, batches, _ = pq_case(O.L2)
        oidx = O.Index(vecs, adj, n, 1, O.L2, pq=(piv, off, codes))
    elif store == "sq":
        n, d, vecs, adj, maxdeg, quantizer, sq_rows, batches, _ = sq_case(O.L2, 8)
        nbits, shift, scale, ssn, mean_norm = quantizer
        oidx = O.Index(vecs, adj, n, 1, O.L2, sq=(sq_rows, nbits, shift, scale, ssn, mean_norm))
    else:
        n, d, vecs, adj, maxdeg, mm_rows, batches, _ = minmax_case(8, None)
        moidx = MinMaxOracle(vecs, adj, n, 1, O.L2, mm_rows, 8)
    rng = np.random.default_rng(17)
    deleted = np.zeros(n + 1, bool)
    deleted[rng.choice(n, n // 5, replace=False)] = True
    want = {}
    for r in (False, True):
        if store == "minmax":
            full = [moidx.search(q, compress(q, None, 8), L + 1, L, rerank=r) for q in batches]
        else:
            full = [(oidx.search_batch_rerank if r else oidx.search_batch)(q, L + 1, L, threads=4) for q in batches]
        want[r] = [filtered(f, deleted, K) for f in full]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        if store == "pq":
            g.upload_pq(piv, off, codes)
        elif store == "sq":
            g.upload_sq(*quantizer, rows=sq_rows)
        else:
            g.upload_minmax(8, 1.0, make_transform(None, d), rows=mm_rows)
        g.delete(np.flatnonzero(deleted))
        sync = getattr(g, f"search_batch_{store}")
        host = getattr(g, f"search_batch_{store}_async")
        dev = getattr(g, f"search_batch_{store}_device_async")
        check_in_flight(g, lambda q, r: sync(q, K, L, 1, rerank=r), lambda s, q, r: host(s, q, K, L, 1, rerank=r),
                        lambda s, *a, rerank: dev(s, a[0], a[1], K, L, 1, *a[2:], rerank=rerank), batches, want, (store, tables))


@gpu
def test_launches_paging_status_errors_and_slots():
    import diskann_b200 as dab
    _, pq_case, _, _, same = in_flight_helpers()
    n, d, vecs, adj, maxdeg, _, _, _, batches, _ = pq_case(O.L2)
    q = batches[0]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)

        def launches():
            c = dab.launch_count()
            out = g.search_batch(q, K, 40)
            return dab.launch_count() - c, out

        base, plain = launches()
        ids = np.array([3, 5, 7, 3], np.uint32)
        # paged sessions ignore deletions; dab_delete does not end them
        s = dab.PagedSearch(g, q, 40)
        page0 = s.next_page(K)
        g.delete(ids)
        assert list(g.delete_status([3, 4, 5, 7, n])) == [True, False, True, True, False]
        page1 = s.next_page(K)
        s2 = dab.PagedSearch(g, q, 40)
        same(s2.next_page(K), page0, "page 0 with tombstones")
        same(s2.next_page(K), page1, "page 1 with tombstones")
        assert launches()[0] == base + 1  # the filter
        # argument errors change nothing
        graph = g.download_graph()
        for bad in ([1, n], [n + 5]):
            with pytest.raises(dab.DabError) as e:
                g.delete(bad)
            assert e.value.code == 1 and str(bad[-1]) in str(e.value)
        with pytest.raises(dab.DabError) as e:
            g.release([3, 4])
        assert e.value.code == 1 and "id 4 is not deleted" in str(e.value)
        with pytest.raises(dab.DabError) as e:
            g.delete_status([n + 1])
        assert e.value.code == 1
        for args in ((0, 1.2), (maxdeg + 1, 1.2), (8, 0.5)):
            with pytest.raises(dab.DabError) as e:
                g.consolidate(*args)
            assert e.value.code == 1
        assert list(g.delete_status(ids)) == [True] * 4 and np.array_equal(g.download_graph(), graph)
        # batches in flight: every mutating call is refused until the slot is joined
        out = g.search_batch_async(2, q, K, 40)
        for fn, arg in ((g.delete, [9]), (g.release, [3]), (g.consolidate, 8)):
            with pytest.raises(dab.DabError) as e:
                fn(arg)
            assert e.value.code == 1 and "slot 2" in str(e.value)
        g.wait(2)
        assert list(g.delete_status([9, 3])) == [False, True] and np.array_equal(g.download_graph(), graph)
        # release empties the rows and ends paged sessions; with no tombstone left the fast path is back
        g.release(ids)
        assert list(g.delete_status(ids)) == [False] * 4
        assert all(g.download_graph(int(i), 1)[0, 0] == 0 for i in ids)
        with pytest.raises(dab.DabError):
            s2.next_page(K)
        g.upload_graph(adj)
        n_now, again = launches()
        assert n_now == base
        same(again, plain, "no tombstones")
        # consolidation that rewrites a list ends paged sessions
        g.delete([11])
        s3 = dab.PagedSearch(g, q, 40)
        s3.next_page(K)
        assert g.consolidate(int(maxdeg * 0.8)) > 0
        with pytest.raises(dab.DabError):
            s3.next_page(K)


@gpu
def test_broadcast_carries_the_deletion_table():
    import torch

    import diskann_b200 as dab
    if torch.cuda.device_count() < 2:
        pytest.skip("replication needs two GPUs; this machine has fewer")
    _, pq_case, _, _, same = in_flight_helpers()
    n, d, vecs, adj, maxdeg, _, _, _, batches, _ = pq_case(O.L2)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg, device=0) as a, \
            dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg, device=1) as b:
        a.upload_vectors(vecs)
        a.upload_graph(adj)
        a.delete(np.arange(0, n, 7))
        check = _lib_broadcast(a, b)
        assert check == 0
        assert np.array_equal(b.delete_status(np.arange(n)), a.delete_status(np.arange(n)))
        same(b.search_batch(batches[0], K, 40), a.search_batch(batches[0], K, 40), "replica")


def _lib_broadcast(*handles):
    import diskann_b200 as dab
    arr = (C.c_void_p * len(handles))(*[h._h.value for h in handles])
    return dab.lib().dab_broadcast(arr, len(handles))
