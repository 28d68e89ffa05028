"""Diversity-aware search over the PQ, SQ and MinMax stores: dab_search_batch_diverse_{pq,sq,minmax}[_device].

The reference's Diverse::search is generic over the search strategy (diverse_search.rs:189-234): it traverses with the
strategy's accessor and hands best.iter().take(L) to the strategy's post-processor, which for the quantized in-memory
strategies is Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-400, full_precision.rs:356-399).  Only
the traversal distances change — the quantized accessor's, the ones dab_search_batch_{pq,sq,minmax} compute — and, with
rerank, the post-processed list is reordered by full-precision distance.

CPU: the oracle's table entry point (orc_search_batch_diverse_table, oracle/diverse_table.cpp) fed the full-precision distances equals
orc_search_batch_diverse bit for bit, failed removals included, over row types, metrics, cardinalities, beams and
exact-tie graphs; with rerank its results keep the diverse limit, are a subset of the post-processed list of the same
traversal and are sorted by full-precision distance.
GPU: the device equals the oracle fed each store's exhaustive distances (test_paged_search_quantized.py pins them to
the oracle's quantized searches) bit for bit — ids, distance bits, counts, cmps and hops — over every PQ table kind and
chunk layout, every SQ and MinMax width and metric, every MinMax transform kind, every row type, rerank 0 and 1,
cardinalities 1, 2, 64 and distinct, diverse_k from 1 to 2^32 - 1, edge graphs, deletions and re-inserted ids and
forced overflow re-runs; every refusal is reported before any launch and leaves the index usable."""
import functools

import numpy as np
import pytest

import diskann_b200 as dab
import diverse_oracle as D
import diverse_table_oracle as DT
import oracle_lib as O
from test_paged_search import built
from test_paged_search_quantized import MMStore, PQStore, SQStore, pq_store, sq_store
from test_traversal_edges import grid as tie_grid, malformed_case, many_starts

FIVE = ("ids", "dists", "counts", "cmps", "hops")
INVALID_ARGUMENT, NOT_READY = 1, 5


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def attributes(total, kind, seed):
    """(values, present) for every id: `kind` a cardinality, "distinct", or "half" (cardinality 5, every other id
    without an attribute)"""
    rng = np.random.default_rng(seed)
    present = np.ones(total, np.uint8)
    if kind == "distinct":
        return rng.permutation(total).astype(np.uint32), present
    card = 5 if kind == "half" else kind
    values = rng.integers(0, card, total).astype(np.uint32)
    if kind == "half":
        present[::2] = 0
    return values, present


def diverse_ok(ids, values, present, dk):
    """every id has an attribute and no attribute value is held by more than dk of them"""
    ids = np.asarray(ids, np.int64)
    return bool(present[ids].all()) and (len(ids) == 0 or np.unique(values[ids], return_counts=True)[1].max() <= dk)


def fp_tables(vecs, metric, queries):
    """QueryDist of the oracle for every (query, id): f16 queries widened once, the avx2 flavour of the searches"""
    wide = queries.astype(np.float32) if vecs.dtype == np.float16 else queries
    return np.stack([O.distance_rows(q, vecs, metric, O.AVX2) for q in wide])


def store_tables(store, queries):
    return np.stack([store.distances(q) for q in queries])


# ---------------------------------------------------------------- CPU

@functools.lru_cache(maxsize=None)
def cpu_case(dt, metric):
    return built(600, 16, dt, metric, 40, seed=5 + (dt == np.float16))


CPU_RUNS = [(10, 10, 1, 1), (10, 40, 1, 3), (10, 40, 4, 10), (5, 120, 2, 2), (10, 30, 1, 1 << 30)]


@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.int8, O.L2),
                                       (np.uint8, O.COSINE_NORMALIZED), (np.float16, O.INNER_PRODUCT)])
@pytest.mark.parametrize("kind", [1, 2, 64, "distinct", "half"])
def test_table_of_full_precision_distances_is_the_diverse_search(dt, metric, kind):
    vecs, adj, n, n_start, metric, qs = cpu_case(dt, metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = fp_tables(vecs, metric, qs)
    values, present = attributes(n + n_start, kind, 3)
    for k, L, beam, dk in CPU_RUNS:
        want = D.search_batch(oidx, qs, k, L, dk, values, present, beam=beam)
        got = DT.search_batch_table(oidx, tables, None, k, L, dk, values, present, beam=beam)
        same(got, want, (k, L, beam, dk))
        assert np.array_equal(got[5], want[5])


def test_table_equals_the_diverse_search_on_exact_ties():
    case = tie_grid(800, 8, 3, 30, 3)
    tables = fp_tables(case.vecs, case.metric, case.queries)
    failed = 0
    for card in (2, 5, 64):
        values = (np.arange(case.total) % card).astype(np.uint32)
        for k, L, beam, dk in [(10, 30, 1, 1), (10, 60, 2, 3), (5, 200, 4, 2)]:
            want = D.search_batch(case.oracle, case.queries, k, L, dk, values, beam=beam)
            got = DT.search_batch_table(case.oracle, tables, None, k, L, dk, values, beam=beam)
            same(got, want, (card, k, L, beam, dk))
            assert np.array_equal(got[5], want[5])
            failed += int(want[5].sum())
    assert failed > 0, "no removal failed"


def post_processed_list(adj, n, n_start, table, k, L, dk, values, present):
    """search_internal over the oracle's DiverseNeighborQueue with the distances of `table`, then its post_process:
    (best.iter().take(L) ids, cmps, hops)"""
    total = n + n_start
    q = D.DiverseQueue(L, k, dk, {i: int(values[i]) for i in range(total) if present[i]})
    visited = set(range(n, total))
    for s in range(n, total):
        q.insert(s, float(table[s]))
    cmps, hops = n_start, 0
    while q.has_notvisited_node():
        node = q.closest_notvisited()[0]
        fresh = [int(j) for j in adj[node][1:1 + adj[node][0]] if j not in visited and (visited.add(int(j)) or True) and j < total]
        for j in fresh:
            q.insert(j, float(table[j]))
        cmps += len(fresh)
        hops += 1
    q.post_process()
    return [i for i, _ in q.iter()], cmps, hops


@pytest.mark.parametrize("kind,nbits", [("pq", None), ("sq", 8), ("mm", 4)])
def test_rerank_keeps_the_limit_and_sorts_the_post_processed_list(kind, nbits):
    vecs, adj, n, n_start, metric, qs = case = cpu_case(np.float32, O.L2)
    store = pq_store(case, 4) if kind == "pq" else sq_store(case, nbits) if kind == "sq" else MMStore(vecs, nbits, "double_same", metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs)
    deleted = np.zeros(n + n_start, bool)
    deleted[::7] = True
    for dk, card in ((1, 5), (3, 5), (2, 64)):
        values, present = attributes(n + n_start, card, dk)
        for dl in (None, deleted):
            k, L = 10, 60
            got = DT.search_batch_table(oidx, tables, qs, k, L, dk, values, present, deleted=dl, rerank=True)
            for qi in range(qs.shape[0]):
                # the post-processed list of the same traversal, start points and deleted ids dropped
                pl, cmps, hops = post_processed_list(adj, n, n_start, tables[qi], k, L, dk, values, present)
                pl = np.array([i for i in pl if i < n and (dl is None or not dl[i])], np.uint32)
                assert (int(got[3][qi]), int(got[4][qi])) == (cmps, hops)
                ids = got[0][qi][:got[2][qi]]
                assert got[2][qi] == min(k, len(pl))
                assert set(ids.tolist()) <= set(pl.tolist())
                fp = O.distance_rows(qs[qi], vecs[ids.astype(np.int64)], metric, O.AVX2)
                assert np.array_equal(fp.view(np.uint32), got[1][qi][:got[2][qi]].view(np.uint32))
                assert all(a <= b for a, b in zip(fp, fp[1:]))
                # the first k by full-precision distance among the list, ties in list order
                full = O.distance_rows(qs[qi], vecs[pl.astype(np.int64)], metric, O.AVX2)
                assert np.array_equal(ids, pl[np.argsort(full, kind="stable")[:k]])
                if got[5][qi] == 0:
                    assert diverse_ok(ids, values, present, dk)


# ---------------------------------------------------------------- GPU

def kind_of(store):
    return {PQStore: "pq", SQStore: "sq", MMStore: "minmax"}[type(store)]


def gpu_index(case, store, max_degree=None):
    vecs, adj, n, n_start, metric = case[:5]
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree or adj.shape[1] - 1)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    store.upload(g)
    return g


def check(g, store, case, runs, values, present, deleted=None, tables=None, reranks=(False, True)):
    """every (k, L, beam, diverse_k) of `runs`, with and without rerank, on the device against the oracle fed the
    store's distances; returns the oracle's failed removals"""
    vecs, adj, n, n_start, metric, qs = case[:6]
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs) if tables is None else tables
    fn = getattr(g, f"search_batch_diverse_{kind_of(store)}")
    failed = 0
    for k, L, beam, dk in runs:
        for rr in reranks:
            want = DT.search_batch_table(oidx, tables, qs, k, L, dk, values, present, beam=beam, deleted=deleted, rerank=rr)
            same(fn(qs, k, L, dk, beam, rerank=rr), want[:5], (kind_of(store), k, L, beam, dk, rr))
            failed += int(want[5].sum())
    return failed


RUNS = [(10, 10, 1, 1), (10, 40, 1, 3), (10, 40, 4, 10), (5, 200, 2, 2), (20, 20, 1, 3)]
NQ = 300


@functools.lru_cache(maxsize=None)
def gpu_case(dt, metric, d=64):
    return built(2000, d, dt, metric, NQ, seed=31 + d)


def run_store(case, store, kinds=(5,), runs=RUNS):
    vecs, adj, n, n_start = case[:4]
    tables = store_tables(store, case[5])
    with gpu_index(case, store) as g:
        for kind in kinds:
            values, present = attributes(n + n_start, kind, 7)
            g.upload_attributes(values, present)
            check(g, store, case, runs, values, present, tables=tables)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.int8, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.uint8, O.COSINE_NORMALIZED)])
@pytest.mark.parametrize("chunks", [16, 8, 7])  # chunks of 4, of 8, of 9 and 10
def test_pq_equals_the_oracle(dt, metric, chunks):
    case = gpu_case(dt, metric)
    run_store(case, pq_store(case, chunks), kinds=(5, "half") if chunks == 16 else (5,))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_sq_equals_the_oracle(nbits, metric):
    dt = {8: np.float32, 4: np.float16, 2: np.int8, 1: np.uint8}[nbits]
    case = gpu_case(dt, metric)
    run_store(case, sq_store(case, nbits))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_minmax_equals_the_oracle(nbits, metric):
    dt = {8: np.float32, 4: np.float16, 2: np.uint8, 1: np.int8}[nbits]
    case = gpu_case(dt, metric, d=48)  # 48: PaddingHadamard pads to 64
    for kind in (None, "padding_natural", "double_same"):
        run_store(case, MMStore(case[0], nbits, kind, metric), runs=RUNS[:3])


def three_stores(case):
    return [pq_store(case, 8), sq_store(case, 8), MMStore(case[0], 8, "double_same", case[4])]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [1, 2, 64, "distinct"])
def test_cardinalities(kind):
    case = gpu_case(np.float32, O.L2)
    for store in three_stores(case):
        run_store(case, store, kinds=(kind,), runs=RUNS + [(10, 700, 1, 3)])


@pytest.mark.gpu
def test_diverse_k_up_to_2_to_the_32():
    case = gpu_case(np.float32, O.INNER_PRODUCT)
    for store in three_stores(case):
        run_store(case, store, kinds=(1, 5), runs=[(10, 40, 1, 1), (10, 40, 1, 7), (10, 40, 4, 1 << 30), (5, 300, 1, 0xFFFFFFFF)])


def as_tuple(c):
    return (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 70])
def test_many_start_points(n_start):
    case = as_tuple(many_starts(1500, 16, n_start, 100, n_start))
    for store in three_stores(case):
        run_store(case, store, runs=RUNS[:4])


@pytest.mark.gpu
@pytest.mark.parametrize("max_degree", [1, 7, 40])
def test_malformed_rows(max_degree):
    c = malformed_case(800, 8, 3, max_degree, 80, max_degree)
    case = as_tuple(c)
    values, present = attributes(c.total, "half", max_degree)
    for store in three_stores(case):
        with gpu_index(case, store, c.max_degree) as g:
            g.upload_attributes(values, present)
            check(g, store, case, RUNS[:4], values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("card", [2, 5, 64])
def test_exact_ties_drift(card):
    c = tie_grid(1200, 8, 3, 100, 3)
    case = as_tuple(c)
    values = (np.arange(c.total) % card).astype(np.uint32)
    present = np.ones(c.total, np.uint8)
    runs = [(10, 30, 1, 1), (10, 60, 2, 3), (5, 200, 4, 2)]
    failed = 0
    for store in three_stores(case):
        with gpu_index(case, store) as g:
            g.upload_attributes(values, present)
            failed += check(g, store, case, runs, values, present)
    assert failed > 0, "no removal failed"


@pytest.mark.gpu
def test_overflow_reruns(monkeypatch):
    """visited tables of 256 slots and local-queue pools of one to four entries: every query is re-run, some several
    times, and the rerank or the filter of deleted ids runs over the whole batch again"""
    case = gpu_case(np.float32, O.L2, d=32)
    vecs, adj, n, n_start, metric, qs = case
    values, present = attributes(n + 1, 5, 2)
    deleted = np.zeros(n + 1, bool)
    gone = np.random.default_rng(3).choice(n, 150, replace=False).astype(np.uint32)
    deleted[gone] = True
    for store in three_stores(case):
        tables = store_tables(store, qs)
        for env in ({"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_DIVERSE_POOL": "1"}, {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_DIVERSE_POOL": "4"}):
            for var, val in env.items():
                monkeypatch.setenv(var, val)
            with gpu_index(case, store) as g:
                g.upload_attributes(values, present)
                check(g, store, case, RUNS[:4], values, present, tables=tables)
                g.delete(gone)
                check(g, store, case, RUNS[1:3], values, present, deleted=deleted, tables=tables)
            for var in env:
                monkeypatch.delenv(var)


def encoded(store, vecs):
    """the store with every row of `vecs` encoded by its quantizer"""
    f = np.ascontiguousarray(vecs.astype(np.float32))
    if isinstance(store, PQStore):
        codes = np.zeros_like(store.codes)
        for i in range(f.shape[0]):
            assert O.lib().orc_pq_encode(O.ptr(store.piv), store.piv.shape[0], f.shape[1], O.ptr(store.off), codes.shape[1], O.ptr(f[i]),
                                         O.ptr(codes[i])) == 0
        return PQStore(store.piv, store.off, codes, store.metric)
    if isinstance(store, SQStore):
        return SQStore(O.sq_encode_rows(f, store.quantizer[0], store.quantizer[1], store.nbits), store.nbits, store.quantizer, store.metric)
    return MMStore(vecs, store.nbits, store.kind, store.metric)


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    case = gpu_case(np.float32, O.L2, d=32)
    vecs, adj, n, n_start, metric, qs = case
    values, present = attributes(n + 1, 5, 9)
    gone = rng.choice(n, 200, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    fresh = (vecs[rng.integers(0, n, 200)] + 0.2 * rng.normal(size=(200, vecs.shape[1]))).astype(np.float32)
    vecs2 = vecs.copy()
    vecs2[gone] = fresh
    for store in three_stores(case):
        with gpu_index(case, store) as g:
            g.upload_attributes(values, present)
            g.delete(gone)
            check(g, store, case, RUNS[:4], values, present, deleted=deleted)
            # released ids take new rows, whose codes the insert writes to the store, and new attributes
            g.release(gone)
            v2, p2 = values.copy(), present.copy()
            v2[gone] = rng.integers(100, 103, 200)
            p2[gone[::3]] = 0
            g.upload_attributes(v2, p2)
            g.insert(gone, fresh, 16, 30)
            case2 = (vecs2, g.download_graph(), n, n_start, metric, qs)
            check(g, store, case2, RUNS[:4], v2, p2, tables=store_tables(encoded(store, vecs2), qs))


@pytest.mark.gpu
def test_device_form():
    import torch
    case = gpu_case(np.float32, O.L2)
    qs = case[5]
    nq, k, L = qs.shape[0], 10, 50
    values, present = attributes(case[2] + 1, 5, 6)
    for store in three_stores(case):
        kind = kind_of(store)
        with gpu_index(case, store) as g:
            g.upload_attributes(values, present)
            d_q = torch.from_numpy(qs).cuda()
            for rr in (False, True):
                want = getattr(g, f"search_batch_diverse_{kind}")(qs, k, L, 2, 2, rerank=rr)
                bufs = (torch.full((nq, k), 7, dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
                        *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
                getattr(g, f"search_batch_diverse_{kind}_device")(d_q.data_ptr(), nq, k, L, 2, 2, *(b.data_ptr() for b in bufs), rerank=rr)
                got = [b.cpu().numpy() for b in bufs]  # complete on return: read without a device-wide synchronize
                same(got, want, (kind, rr))


@pytest.mark.gpu
def test_refusals_before_any_launch():
    case = built(600, 16, np.float32, O.L2, 16, seed=31)
    vecs, adj, n, n_start, metric, qs = case
    L_ = dab.lib()
    values, present = attributes(n + 1, 5, 1)

    def fails(code, fn, *args, staged=False, **kw):
        launches = dab.launch_count()
        with pytest.raises(dab.DabError) as e:
            fn(*args, **kw)
        assert e.value.code == code, str(e.value)
        # a NaN after the transform is found by the staging of the queries, before any traversal
        assert staged or dab.launch_count() == launches, ("a refused call launched a kernel", str(e.value))
        return str(e.value)

    pq, sq = pq_store(case, 4), sq_store(case, 8)
    mm = MMStore(vecs, 8, "double_same", O.L2)
    with dab.GpuIndex(dab.DType.f32, O.L2, 16, n, 1, adj.shape[1] - 1) as g:
        g.upload_graph(adj)
        calls = [g.search_batch_diverse_pq, g.search_batch_diverse_sq, g.search_batch_diverse_minmax]
        # no attribute table
        for fn in calls:
            assert "dab_upload_attributes" in fails(INVALID_ARGUMENT, fn, qs, 10, 20, 2)
        g.upload_attributes(values, present)
        # stores never uploaded, or set up without rows: the synchronous calls' messages
        assert "no PQ codes" in fails(NOT_READY, g.search_batch_diverse_pq, qs, 10, 20, 2)
        assert "no scalar-quantized rows" in fails(NOT_READY, g.search_batch_diverse_sq, qs, 10, 20, 2)
        assert "no MinMax rows" in fails(NOT_READY, g.search_batch_diverse_minmax, qs, 10, 20, 2)
        g.upload_pq(pq.piv, pq.off)
        assert "no PQ codes" in fails(NOT_READY, g.search_batch_diverse_pq, qs, 10, 20, 2)
        g.upload_sq(8, *sq.quantizer)
        assert "no scalar-quantized rows" in fails(NOT_READY, g.search_batch_diverse_sq, qs, 10, 20, 2)
        g.upload_minmax(8, 1.0, mm.t)
        assert "no MinMax rows" in fails(NOT_READY, g.search_batch_diverse_minmax, qs, 10, 20, 2)
        for s in (pq, sq, mm):
            s.upload(g)
        for fn in calls:
            # the arguments of dab_search_batch_diverse
            for kk, LL, beam, dk, what in ((0, 20, 1, 2, "k"), (10, 20, 1, 0, "diverse k_value"), (10, 9, 1, 2, "l_value"),
                                           (10, 1025, 1, 2, "1024"), (10, 20, 0, 2, "beam_width"), (10, 20, 65, 2, "beam_width")):
                assert what in fails(INVALID_ARGUMENT, fn, qs, kk, LL, dk, beam)
            # rerank without the full-precision vectors
            assert "rerank needs the full-precision vectors" in fails(NOT_READY, fn, qs, 10, 20, 2, rerank=True)
            assert fn(qs, 10, 20, 2)[2].all()  # without rerank the rows are not needed
        # a MinMax query holding a NaN fails the call, naming it
        bad = qs.copy()
        bad[3, 4] = np.nan
        assert "query 3 contains NaN after the transform (InputContainsNaN)" in fails(INVALID_ARGUMENT, g.search_batch_diverse_minmax, bad,
                                                                                     10, 20, 2, staged=True)
        g.upload_vectors(vecs)
        want_tables = [store_tables(s, qs) for s in (pq, sq, mm)]
        for s, t in zip((pq, sq, mm), want_tables):  # the index is usable after every refusal
            check(g, s, case, [(10, 20, 1, 2)], values, present, tables=t)
        # the shared memory of the kernel: L = 1024 with 64 beams of wide rows does not fit
    n2, md = 100, 200
    vz = np.zeros((n2 + 1, 16), np.float32)
    az = np.zeros((n2 + 1, md + 1), np.uint32)
    with dab.GpuIndex(dab.DType.f32, O.L2, 16, n2, 1, md) as g:
        g.upload_vectors(vz)
        g.upload_graph(az)
        g.upload_attributes(np.zeros(n2 + 1, np.uint32))
        g.upload_sq(8, *sq.quantizer)
        g.sq_encode_all()
        assert "shared memory" in fails(INVALID_ARGUMENT, g.search_batch_diverse_sq, np.zeros((4, 16), np.float32), 10, 1024, 1, 64)
        assert g.search_batch_diverse_sq(np.zeros((4, 16), np.float32), 10, 1024, 1, 8)[2].tolist() == [0] * 4
    with dab.GpuIndex(dab.DType.f32, O.COSINE, 16, n, 1, adj.shape[1] - 1) as g:
        g.upload_graph(adj)
        g.upload_attributes(values, present)
        sq.upload(g)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(INVALID_ARGUMENT, g.search_batch_diverse_sq, qs, 10, 20, 2)
