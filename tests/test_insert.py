"""Inserting points into an index as it stands: dab_insert (DiskANNIndex::insert, diskann/src/graph/index.rs:226-341, and
multi_insert, :815-1030) and the oracle's orc_insert_batched that it is held to.

The oracle's insert (oracle/insert.cpp) restates the multi_insert loop that orc_build_batched runs, over chunks of the
caller's ids, so it is first pinned to the existing builds and to the reference's single-insert lattice baseline; on the H100 the
device's adjacency must then equal it word for word, and the searches over the result must equal the oracle's."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle_lib as O
from insert_oracle import insert_batched
from test_oracle_golden import grid as lattice

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
K = 10


def build_schedule(n, batch_size=0):
    """the batch sizes of dab_build / orc_build_batched (orc_build_batch_size)"""
    if batch_size == 0:
        batch_size = max(1024, min(65536, n // 16))
    out, inserted = [], 0
    while inserted < n:
        b = min(batch_size, max(1, inserted // 8), n - inserted)
        out.append(b)
        inserted += b
    return out


def rows_of(rng, dt, n, d):
    base = rng.normal(size=(n, d)).astype(np.float32)
    if dt == np.float16:
        return base.astype(np.float16)
    if dt == np.int8:
        return np.clip(np.round(base * 40), -127, 127).astype(np.int8)
    if dt == np.uint8:
        return np.clip(np.round(base * 40 + 128), 0, 255).astype(np.uint8)
    return base


def dataset(seed, n=1200, d=16, dt=np.float32):
    rng = np.random.default_rng(seed)
    base = rows_of(rng, dt, n, d)
    f = base.astype(np.float32)
    vecs = np.concatenate([base, base[np.argmin(((f - f.mean(0)) ** 2).sum(1))][None]])
    return rng, vecs


# ---------------------------------------------------------------- CPU: the oracle's insert

@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT])
def test_oracle_insert_over_the_build_schedule_equals_the_batched_build(metric):
    _, vecs = dataset(1)
    n, R, maxdeg, L = vecs.shape[0] - 1, 12, 15, 30
    want = O.build_graph_batched(vecs, n, 1, metric, R, maxdeg, L)
    adj = np.zeros_like(want)
    first = 0
    for b in build_schedule(n):
        adj = insert_batched(vecs, adj, np.arange(first, first + b), n, 1, metric, R, maxdeg, L, batch_size=b)
        first += b
    assert np.array_equal(adj, want)


def test_oracle_insert_one_by_one_equals_the_sequential_build():
    _, vecs = dataset(2, n=500)
    n = vecs.shape[0] - 1
    want = O.build_graph(vecs, n, 1, O.L2, 10, 13, 24)
    sets_appends = O.last_build_counts()
    got, counts = insert_batched(vecs, np.zeros_like(want), np.arange(n), n, 1, O.L2, 10, 13, 24, batch_size=1, counts=True)
    assert np.array_equal(got, want)
    assert counts == sets_appends


def test_oracle_insert_reproduces_the_reference_single_insert_lattice():
    """grid_insert.rs, 1-D, 100 points (the case test_grid_insert_baselines reproduces exactly), inserted by two calls:
    ids 0-49, then 50-99, one point at a time."""
    g = json.load(open(os.path.join(GOLDEN, "grid_insert.json")))
    case = next(c for c in g["cases"] if c["grid_dims"] == 1)
    data, _, n = lattice(1, case["grid_size"])
    max_degree = 2
    pruned = min(max(max_degree - 2, 2), max_degree)
    adj = np.zeros((n + 1, max_degree + 1), np.uint32)
    sets = appends = 0
    for ids in (np.arange(0, 50), np.arange(50, 100)):
        adj, (s, a) = insert_batched(data, adj, ids, n, 1, O.L2, pruned, max_degree, 100, 1.2, batch_size=1, tie_mode=1,
                                     counts=True)
        sets, appends = sets + s, appends + a
    assert (sets, appends) == (case["set_neighbors"], case["append_neighbors"])
    idx = O.Index(data, adj, n, 1, O.L2)
    for s in case["searches"]:
        q = np.array([s["query"]], np.float32)
        ids, dists, counts, cmps, hops = idx.search_batch(q, 10, 10, beam=s["beam_width"], flavour=O.SIMD)
        assert int(counts[0]) == s["num_results"]
        assert int(hops[0]) == s["hops"] and int(cmps[0]) == s["comparisons"]
        assert [float(x) for x in dists[0]] == [r[1] for r in s["results"]]
        assert [int(i) for i in ids[0]] == [r[0] for r in s["results"]]


def test_null_handle_is_refused_before_any_device_work():
    import diskann_b200 as dab
    L = dab.lib()
    assert L.dab_insert(None, None, None, 0, 8, 20, 1.2, 0) == 1
    assert b"dab_insert" in L.dab_last_error()


# ---------------------------------------------------------------- GPU

gpu = pytest.mark.gpu


def same(got, want, what):
    for a, b, name in zip(got, want, ("ids", "dists", "counts", "cmps", "hops")):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def check_graph(got, want, what):
    bad = np.flatnonzero((got != want).any(1))
    assert len(bad) == 0, (what, bad[:5], got[bad[:1]], want[bad[:1]])


def queries_for(rng, vecs, nq=64):
    f = vecs[:-1].astype(np.float32)
    q = f[rng.choice(f.shape[0], nq, replace=False)] + 0.1 * rng.normal(size=(nq, f.shape[1])).astype(np.float32)
    if vecs.dtype == np.float16:
        return q.astype(np.float16)
    if vecs.dtype == np.int8:
        return np.clip(np.round(q), -127, 127).astype(np.int8)
    if vecs.dtype == np.uint8:
        return np.clip(np.round(q), 0, 255).astype(np.uint8)
    return q.astype(np.float32)


@gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.COSINE), (np.float16, O.INNER_PRODUCT),
                                       (np.int8, O.L2), (np.uint8, O.COSINE_NORMALIZED)])
def test_inserts_in_the_build_schedule_equal_the_device_build(dt, metric):
    import diskann_b200 as dab
    _, vecs = dataset(5, n=1500, d=24, dt=dt)
    n, R, maxdeg, L = vecs.shape[0] - 1, 12, 15, 30
    with dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, 1, maxdeg) as a, \
            dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, 1, maxdeg) as b:
        a.upload_vectors(vecs)
        a.build(R, L)
        want = a.download_graph()
        b.upload_vectors(vecs[n:], first=n)  # the start point only: the graph is grown by inserts alone
        first = 0
        for size in build_schedule(n):
            ids = np.arange(first, first + size, dtype=np.uint32)
            b.insert(ids, vecs[ids], R, L)
            first += size
        check_graph(b.download_graph(), want, "schedule")


def linked_80(seed, n=2000, d=16, R=12, maxdeg=15, L=40):
    """a graph over a shuffled 80 % of the ids (the oracle's inserts in chunks of 64); the rest are rows no list reaches"""
    rng, vecs = dataset(seed, n=n, d=d)
    order = rng.permutation(n).astype(np.uint32)
    linked, rest = order[:int(0.8 * n)], order[int(0.8 * n):]
    adj = insert_batched(vecs, np.zeros((n + 1, maxdeg + 1), np.uint32), linked, n, 1, O.L2, R, maxdeg, L, batch_size=64)
    return rng, vecs, adj, linked, rest


@gpu
@pytest.mark.parametrize("batch", [1, 37, 512, 0])
def test_inserts_into_a_built_graph_equal_the_oracle(batch):
    import diskann_b200 as dab
    rng, vecs, adj0, linked, rest = linked_80(7)
    n, d, R, maxdeg, L = vecs.shape[0] - 1, vecs.shape[1], 12, 15, 40
    want = insert_batched(vecs, adj0, rest, n, 1, O.L2, R, maxdeg, L, batch_size=batch)
    stale = vecs.copy()
    stale[rest] = rng.normal(size=(len(rest), d)).astype(np.float32) * 100  # what the slots held before
    q = queries_for(rng, vecs)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(stale)
        g.upload_graph(adj0)
        g.insert(rest, vecs[rest], R, L, batch_size=batch)
        check_graph(g.download_graph(), want, batch)
        for Ls in (16, 100):
            same(g.search_batch(q, K, Ls), O.Index(vecs, want, n, 1, O.L2).search_batch(q, K, Ls, threads=4), (batch, Ls))


@gpu
def test_reinserting_live_points_equals_the_oracle():
    import diskann_b200 as dab
    rng, vecs = dataset(9, n=1500, d=16)
    n, d, R, maxdeg, L = vecs.shape[0] - 1, 16, 12, 15, 40
    adj0 = O.build_graph_batched(vecs, n, 1, O.L2, R, maxdeg, L)
    ids = rng.choice(n, 150, replace=False).astype(np.uint32)
    new = vecs.copy()
    new[ids] = rng.normal(size=(len(ids), d)).astype(np.float32)
    want = insert_batched(new, adj0, ids, n, 1, O.L2, R, maxdeg, L, batch_size=32)
    q = queries_for(rng, new)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.insert(ids, new[ids], R, L, batch_size=32)
        check_graph(g.download_graph(), want, "live")
        same(g.search_batch(q, K, 60), O.Index(new, want, n, 1, O.L2).search_batch(q, K, 60, threads=4), "live")


@gpu
def test_delete_consolidate_release_then_insert_into_the_released_slots():
    import diskann_b200 as dab
    from test_delete_consolidate import filtered
    rng, vecs = dataset(13, n=2000, d=16)
    n, d, R, maxdeg, L = vecs.shape[0] - 1, 16, 12, 15, 40
    adj0 = O.build_graph_batched(vecs, n, 1, O.L2, R, maxdeg, L)
    gone = rng.choice(n, n // 10, replace=False).astype(np.uint32)
    released, kept = gone[:160], gone[160:]  # the rest stay deleted
    new = vecs.copy()
    new[released] = rng.normal(size=(len(released), d)).astype(np.float32)
    q = queries_for(rng, new)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.delete(gone)
        g.consolidate(R)
        g.release(released)
        after_release = g.download_graph()
        with pytest.raises(dab.DabError) as e:
            g.insert(kept[:1], new[kept[:1]], R, L)
        assert e.value.code == 1 and f"id {kept[0]} is deleted" in str(e.value) and "release it first" in str(e.value)
        g.insert(released, new[released], R, L, batch_size=64)
        want = insert_batched(new, after_release, released, n, 1, O.L2, R, maxdeg, L, batch_size=64)
        check_graph(g.download_graph(), want, "cycle")
        deleted = np.zeros(n + 1, bool)
        deleted[kept] = True
        got = g.search_batch(q, K, 60)
        same(got, filtered(O.Index(new, want, n, 1, O.L2).search_batch(q, 61, 60, threads=4), deleted, K), "cycle")
        assert not np.isin(got[0], kept).any()


STORES = ["pq", "sq8", "sq4", "minmax8"]


@gpu
@pytest.mark.parametrize("store", STORES)
def test_inserts_keep_every_quantized_store_in_step(store):
    import diskann_b200 as dab
    from test_gpu_parity import sq_quantizer
    from test_minmax_search import MinMaxOracle, compress, make_transform
    rng, vecs = dataset(17, n=1500, d=32)
    n, d, R, maxdeg, L = vecs.shape[0] - 1, 32, 12, 15, 40
    adj0 = O.build_graph_batched(vecs, n, 1, O.L2, R, maxdeg, L)
    ids = np.concatenate([rng.choice(n, 100, replace=False)]).astype(np.uint32)
    new = vecs.copy()
    new[ids] = rng.normal(size=(len(ids), d)).astype(np.float32)
    want = insert_batched(new, adj0, ids, n, 1, O.L2, R, maxdeg, L)
    q = queries_for(rng, new)
    t = make_transform("double_same", d)
    nbits = 4 if store == "sq4" else 8
    quantizer = (nbits,) + sq_quantizer(vecs[:n], O.L2)

    def set_up(g, rows_from_encode):
        if store == "pq":
            if rows_from_encode is None:
                g.pq_train(vecs[:1000], 8, 64, 3, 5)
            else:
                g.upload_pq(*rows_from_encode)
            g.pq_encode_all()
            g.upload_sq(*quantizer)  # a store without rows
        elif store.startswith("sq"):
            g.upload_sq(*quantizer)
            g.sq_encode_all()
            g.upload_minmax(8, 1.0, t)  # a store without rows
        else:
            g.upload_minmax(8, 1.0, t)
            g.minmax_encode_all()
            g.upload_sq(*quantizer)  # a store without rows

    def rows(g):
        return g.download_pq() if store == "pq" else g.download_sq() if store.startswith("sq") else g.download_minmax()

    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g, \
            dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as ref:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        set_up(g, None)
        g.insert(ids, new[ids], R, L)
        check_graph(g.download_graph(), want, store)
        got_rows = rows(g)
        ref.upload_vectors(new)
        set_up(ref, got_rows[:2] if store == "pq" else None)
        want_rows = rows(ref)
        for a, b in zip(got_rows if store == "pq" else [got_rows], want_rows if store == "pq" else [want_rows]):
            assert np.array_equal(a, b), store
        with pytest.raises(dab.DabError) as e:  # the store without rows still has none
            g.download_minmax() if store.startswith("sq") else g.download_sq()
        assert e.value.code == 5
        if store == "pq":
            oracle = O.Index(new, want, n, 1, O.L2, pq=got_rows).search_batch_rerank(q, K, 60, threads=4)
            got = g.search_batch_pq(q, K, 60, 1, rerank=True)
        elif store.startswith("sq"):
            oracle = O.Index(new, want, n, 1, O.L2, sq=(got_rows,) + quantizer).search_batch_rerank(q, K, 60, threads=4)
            got = g.search_batch_sq(q, K, 60, 1, rerank=True)
        else:
            oracle = MinMaxOracle(new, want, n, 1, O.L2, got_rows, 8).search(q, compress(q, t, 8), K, 60, rerank=True)
            got = g.search_batch_minmax(q, K, 60, 1, rerank=True)
        same(got, oracle, store)


@gpu
def test_exhaustive_scans_see_the_inserted_rows():
    import diskann_b200 as dab
    rng, vecs, adj0, linked, rest = linked_80(19, n=3000, d=32)
    n, d = vecs.shape[0] - 1, 32
    new = vecs.copy()
    new[rest] = rng.normal(size=(len(rest), d)).astype(np.float32)
    q = queries_for(rng, new)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, 15) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.flat_knn_tc(q, K)  # the tensor-core operand is built from the old rows
        g.insert(rest, new[rest], 12, 40)
        want = O.bruteforce_knn(new[:n], q, O.L2, K)
        for got in (g.flat_knn(q, K), g.flat_knn_tc(q, K)):
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


@gpu
def test_refusals_change_nothing():
    import diskann_b200 as dab
    from test_gpu_parity import sq_quantizer
    from test_minmax_search import make_transform
    rng, vecs = dataset(23, n=1000, d=32)
    n, d, R, maxdeg, L = vecs.shape[0] - 1, 32, 12, 15, 40
    adj0 = O.build_graph_batched(vecs, n, 1, O.L2, R, maxdeg, L)
    q = queries_for(rng, vecs)
    probe = np.tile(np.arange(n, dtype=np.uint32), (4, 1))[:, :n]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        with pytest.raises(dab.DabError) as e:
            g.insert([1], vecs[1:2], R, L)
        assert e.value.code == 5  # no vectors
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.upload_sq(8, *sq_quantizer(vecs[:n], O.L2))
        g.sq_encode_all()
        g.upload_minmax(8, 1.0, make_transform("double_same", d))
        g.minmax_encode_all()
        g.delete([7])

        def state():
            return g.download_graph(), g.download_sq(), g.download_minmax(), g.distances(q[:4], probe)

        before = state()
        row = vecs[3:6].copy()
        for ids, rows, args, code, text in (
                ([5, n], row[:2], (R, L), 1, f"id {n} is not a data point"),     # the start point
                ([5, n + 9], row[:2], (R, L), 1, f"id {n + 9} is not a data point"),
                ([5, 6, 5], row, (R, L), 1, "id 5 appears more than once"),
                ([5, 7], row[:2], (R, L), 1, "id 7 is deleted"),
                ([5], row[:1], (0, L), 1, "pruned_degree"),
                ([5], row[:1], (maxdeg + 1, L), 1, "pruned_degree"),
                ([5], row[:1], (R, 0), 1, "l_build"),
                ([5], row[:1], (R, L, 0.5), 1, "alpha")):
            with pytest.raises(dab.DabError) as e:
                g.insert(ids, rows, *args)
            assert e.value.code == code and text in str(e.value) and "dab_insert" in str(e.value), (ids, str(e.value))
        assert dab.lib().dab_insert(g._h, None, None, 2, R, L, 1.2, 0) == 1
        # a NaN row fails MinMax's check before anything is written
        bad = row.copy()
        bad[1, 4] = np.nan
        with pytest.raises(dab.DabError) as e:
            g.insert([20, 21, 22], bad, R, L)
        assert e.value.code == 1 and "row 1 contains NaN after the transform" in str(e.value)
        for a, b in zip(state(), before):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
        # n == 0: checks only, nothing launched
        c = dab.launch_count()
        g.insert(np.zeros(0, np.uint32), np.zeros((0, d), np.float32), R, L)
        assert dab.launch_count() == c
        # a batch in flight: refused until joined; then the same call succeeds
        g.search_batch_async(1, q, K, 40)
        with pytest.raises(dab.DabError) as e:
            g.insert([20], row[:1], R, L)
        assert e.value.code == 1 and "slot 1" in str(e.value)
        g.wait(1)
        for a, b in zip(state(), before):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
        # an open paged session fails its next page after an insert
        s = dab.PagedSearch(g, q, 40)
        s.next_page(K)
        g.insert([20], row[:1], R, L)
        with pytest.raises(dab.DabError):
            s.next_page(K)
        s.close()
