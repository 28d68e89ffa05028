"""Filtered search over the PQ, SQ and MinMax stores: dab_search_batch_filtered_{pq,sq,minmax}[_device].

The reference's InlineFilterSearch::search is generic over the search strategy (inline_filter_search.rs:89-160), and
graph::ext::labeled::Filtered wraps the quantized strategies too (labeled.rs:96-129), with their post-processor
Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-400, full_precision.rs:356-399).  Only the traversal
distances change — the quantized accessor's, the ones dab_search_batch_{pq,sq,minmax} compute — and, with rerank, the
first L matches are reordered by full-precision distance.

CPU: the table oracle (tests/filtered_table_oracle.py: orc_search_batch_filtered over a one-dimensional view whose
distances are the table's) fed the full-precision distances equals orc_search_batch_filtered bit for bit over row
types, metrics, selectivities, both modes, beams, adaptive L, many start points, edge graphs and deletions; with rerank
its results are the first k, in stable full-precision order, of the first L matches of the same traversal.
GPU: the device equals the oracle fed each store's exhaustive distances (test_paged_search_quantized.py pins them to
the oracle's quantized searches) bit for bit — ids, distance bits, counts, cmps and hops — with rerank 0 and 1, over every
PQ table kind and chunk layout, every SQ and MinMax width and metric, every MinMax transform kind, every row type,
selectivities, beams, adaptive L up to floor(L * scale) = 1024, many start points, malformed rows, exact ties, forced
overflow re-runs, deleted and re-inserted ids, the device forms and empty batches; an accept-all filter is the k-NN
traversal of the store; every refusal is reported before any launch and leaves the index usable."""
import functools

import numpy as np
import pytest

import diskann_b200 as dab
import filtered_oracle as F
import filtered_table_oracle as FT
import oracle_lib as O
from test_diverse_search_quantized import encoded
from test_filtered_search import SELECTIVITY, random_labels
from test_filtered_search_gpu import masks_for
from test_gpu_parity import trained_pq
from test_paged_search import built
from test_paged_search_quantized import MMStore, PQStore, as_f32, pq_store, sq_store
from test_traversal_edges import clustered, grid as tie_grid, malformed_case, many_starts, non_finite

FIVE = ("ids", "dists", "counts", "cmps", "hops")
INVALID_ARGUMENT, NOT_READY = 1, 5
EMPTY = 0xFFFFFFFF


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def fp_tables(vecs, metric, queries):
    """QueryDist of the oracle for every (query, id): f16 queries widened once, the avx2 flavour of the searches"""
    wide = queries.astype(np.float32) if vecs.dtype == np.float16 else queries
    return np.stack([O.distance_rows(q, vecs, metric, O.AVX2) for q in wide])


def store_tables(store, queries):
    return np.stack([store.distances(q) for q in queries])


# ---------------------------------------------------------------- CPU

# (k, L, beam, match_all, mask, adaptive_l)
CPU_RUNS = [(10, 20, 1, False, 1, None), (10, 20, 2, True, 1, None), (10, 20, 4, False, 0b110, (40, 2.0)),
            (10, 20, 1, True, 0b101, (60, 8.0)), (10, 30, 2, True, 0, None), (5, 12, 1, False, 1, (30, 16.0)), (10, 25, 1, False, 1, (1, 1.0))]


@functools.lru_cache(maxsize=None)
def cpu_case(dt, metric):
    rng = np.random.default_rng(6)
    n, n_start = 300, 2
    base = clustered(rng, n, 16)
    if dt in (np.int8, np.uint8):
        base = np.clip(base * 30 + (0 if dt == np.int8 else 100), -128 if dt == np.int8 else 0, 127 if dt == np.int8 else 255)
    vecs = np.concatenate([base, base[:n_start]]).astype(dt)
    adj = O.build_graph(vecs, n, n_start, metric, 16, 20, 30)
    return vecs, adj, n, n_start, metric, vecs[rng.integers(0, n, 6)]


@pytest.mark.parametrize("dt,metric", [(np.float32, O.COSINE), (np.float16, O.INNER_PRODUCT), (np.int8, O.L2), (np.uint8, O.COSINE),
                                       (np.float32, O.L2)])
def test_table_of_full_precision_distances_is_the_filtered_search(dt, metric):
    vecs, adj, n, n_start, metric, qs = cpu_case(dt, metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = fp_tables(vecs, metric, qs)
    rng = np.random.default_rng(4)
    for sel in SELECTIVITY:
        labels = random_labels(rng, n + n_start, sel)
        for k, L, beam, match_all, mask, adaptive in CPU_RUNS:
            args = (k, L, labels, mask, match_all, adaptive, beam)
            same(FT.search_batch_table(oidx, tables, None, *args), F.search_batch(oidx, qs, *args), (sel, k, L, beam, match_all, mask, adaptive))


def edge_cases():
    return [many_starts(300, 8, 70, 6, 4), malformed_case(300, 8, 3, 24, 6, 1), tie_grid(300, 6, 2, 6, 2),
            non_finite(200, 8, np.float32, O.L2, 6, 3)[0], non_finite(200, 8, np.float32, O.INNER_PRODUCT, 6, 4)[0]]


def test_table_equals_the_filtered_search_on_edge_graphs_and_deletions():
    rng = np.random.default_rng(8)
    for c in edge_cases():
        tables = fp_tables(c.vecs, c.metric, c.queries)
        labels = random_labels(rng, c.total, 0.4)
        deleted = rng.random(c.total) < 0.3
        for start_label in (0, 1):  # start points rejected and accepted
            labels[c.n:] = start_label
            for k, L, beam, match_all, mask, adaptive in CPU_RUNS:
                for dl in (None, deleted):
                    args = (k, L, labels, mask, match_all, adaptive, beam, dl)
                    same(FT.search_batch_table(c.oracle, tables, None, *args), F.search_batch(c.oracle, c.queries, *args),
                         (c.n_start, start_label, k, L, beam, adaptive, dl is None))


@pytest.mark.parametrize("kind,nbits", [("pq", None), ("sq", 8), ("mm", 4)])
def test_rerank_sorts_the_first_l_matches(kind, nbits):
    vecs, adj, n, n_start, metric, qs = case = built(600, 16, np.float32, O.L2, 40, seed=5)
    store = pq_store(case, 4) if kind == "pq" else sq_store(case, nbits) if kind == "sq" else MMStore(vecs, nbits, "double_same", metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs)
    rng = np.random.default_rng(2)
    deleted = np.zeros(n + n_start, bool)
    deleted[::7] = True
    for sel in (0.5, 0.1):
        labels = random_labels(rng, n + n_start, sel)
        for dl in (None, deleted):
            for k, L, beam, adaptive in ((10, 40, 1, None), (5, 30, 2, (50, 4.0))):
                args = (labels, 1, False, adaptive, beam, dl)
                got = FT.search_batch_table(oidx, tables, qs, k, L, *args, rerank=True)
                # the first L matches of the same traversal, start points and deleted ids dropped, in matched-list order
                plain = FT.search_batch_table(oidx, tables, None, L, L, *args)
                assert np.array_equal(got[3], plain[3]) and np.array_equal(got[4], plain[4])
                for qi in range(qs.shape[0]):
                    pl = plain[0][qi][:plain[2][qi]]
                    cnt = int(got[2][qi])
                    assert cnt == min(k, len(pl))
                    full = O.distance_rows(qs[qi], vecs[pl.astype(np.int64)], metric, O.AVX2)
                    order = np.argsort(full, kind="stable")[:k]
                    assert np.array_equal(got[0][qi][:cnt], pl[order])
                    assert np.array_equal(got[1][qi][:cnt].view(np.uint32), full[order].view(np.uint32))
                    assert (got[0][qi][cnt:] == EMPTY).all()


# ---------------------------------------------------------------- GPU

def kind_of(store):
    return {PQStore: "pq", MMStore: "minmax"}.get(type(store), "sq")


def gpu_index(case, store, labels, max_degree=None, vectors=True):
    vecs, adj, n, n_start, metric = case[:5]
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree or adj.shape[1] - 1)
    if vectors:
        g.upload_vectors(vecs)
    g.upload_graph(adj)
    g.upload_labels(labels)
    store.upload(g)
    return g


def check(g, store, case, runs, labels, deleted=None, tables=None, reranks=(False, True)):
    """every (k, L, beam, match_all, adaptive_l) of `runs`, with and without rerank, on the device against the oracle fed
    the store's distances"""
    vecs, adj, n, n_start, metric, qs = case[:6]
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs) if tables is None else tables
    fn = getattr(g, f"search_batch_filtered_{kind_of(store)}")
    for k, L, beam, match_all, adaptive in runs:
        masks = masks_for(qs.shape[0], L, match_all)
        for rr in reranks:
            want = FT.search_batch_table(oidx, tables, qs, k, L, labels, masks, match_all, adaptive, beam=beam, deleted=deleted, rerank=rr)
            got = fn(qs, masks, k, L, beam, match_all, adaptive, rerank=rr)
            same(got, want, (kind_of(store), k, L, beam, match_all, adaptive, rr))


# (k, L, beam, match_all, adaptive_l)
RUNS = [(10, 10, 1, False, None), (10, 40, 2, True, None), (10, 40, 1, False, (50, 2.0)), (10, 64, 4, False, (200, 8.0)),
        (5, 100, 1, True, (1000, 8.0)), (10, 20, 1, False, (30, 3.7))]
NQ = 200


@functools.lru_cache(maxsize=None)
def gpu_case(dt, metric, d=64):
    return built(2000, d, dt, metric, NQ, seed=31 + d)


def run_store(case, store, sels=(0.1,), runs=RUNS):
    n, n_start = case[2], case[3]
    tables = store_tables(store, case[5])
    for sel in sels:
        labels = random_labels(np.random.default_rng(int(sel * 1000) + 1), n + n_start, sel)
        with gpu_index(case, store, labels) as g:
            check(g, store, case, runs, labels, tables=tables)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.int8, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.uint8, O.COSINE_NORMALIZED)])
@pytest.mark.parametrize("chunks", [16, 8, 7])  # chunks of 4, of 8, of 9 and 10
def test_pq_equals_the_oracle(dt, metric, chunks):
    case = gpu_case(dt, metric)
    run_store(case, pq_store(case, chunks), sels=(0.5, 0.01) if chunks == 16 else (0.1,))


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
        run_store(case, MMStore(case[0], nbits, kind, metric), runs=RUNS[:4])


def three_stores(case):
    return [pq_store(case, 8), sq_store(case, 8), MMStore(case[0], 8, "double_same", case[4])]


@pytest.mark.gpu
@pytest.mark.parametrize("selectivity", SELECTIVITY)
def test_selectivities(selectivity):
    case = gpu_case(np.float32, O.L2)
    for store in three_stores(case):
        run_store(case, store, sels=(selectivity,), runs=RUNS + [(1, 1, 1, True, (1, 1024.0))])


@pytest.mark.gpu
def test_adaptive_regions_and_the_longest_list():
    """samples that fire with specificity >= 0.5, in [0.1, 0.5), below 0.1 and at zero; floor(L * scale) == 1024"""
    case = gpu_case(np.float32, O.INNER_PRODUCT, d=32)
    runs = [(10, 64, 1, False, (100, 16.0)), (10, 128, 2, False, (300, 8.0)), (10, 256, 4, False, (64, 4.0)),
            (10, 100, 1, False, (500, 10.24))]
    for store in three_stores(case):
        run_store(case, store, sels=(0.8, 0.3, 0.03, 0.0), runs=runs)


def as_tuple(c):
    return (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 70])
def test_many_start_points(n_start):
    c = many_starts(1500, 16, n_start, 100, n_start)
    case = as_tuple(c)
    labels = random_labels(np.random.default_rng(n_start), c.total, 0.3)
    runs = RUNS[:4] + [(5, 10, 1, False, (1, 2.0)), (5, 10, 2, False, (5, 1.5))]
    for store in three_stores(case):
        tables = store_tables(store, c.queries)
        for start_label in (0, 1):
            labels[c.n:] = start_label
            with gpu_index(case, store, labels) as g:
                check(g, store, case, runs, labels, tables=tables)


@pytest.mark.gpu
@pytest.mark.parametrize("max_degree", [1, 7, 40])
def test_malformed_rows(max_degree):
    c = malformed_case(800, 8, 3, max_degree, 80, max_degree)
    case = as_tuple(c)
    labels = random_labels(np.random.default_rng(max_degree), c.total, 0.2)
    for store in three_stores(case):
        with gpu_index(case, store, labels, c.max_degree) as g:
            check(g, store, case, RUNS, labels)


def few_centers_pq(case, chunks, centers):
    """a PQ table of `centers` pivots: rows that share a code have bit-identical distances"""
    f = as_f32(case[0])
    piv, off = trained_pq(np.random.default_rng(3), f[:case[2]], chunks, centers)
    codes = np.zeros((f.shape[0], chunks), np.uint8)
    for i in range(f.shape[0]):
        assert O.lib().orc_pq_encode(O.ptr(piv), centers, f.shape[1], O.ptr(off), chunks, O.ptr(f[i]), O.ptr(codes[i])) == 0
    return PQStore(piv, off, codes, case[4])


@pytest.mark.gpu
def test_exact_ties():
    """a PQ store of 4 centers over 2 chunks (at most 16 distinct distances a query) and the tie grid under every store:
    the matched list's order among equal distances is the earlier match first, and the results do hold ties"""
    case = gpu_case(np.float32, O.L2, d=32)
    few = few_centers_pq(case, 2, 4)
    c = as_tuple(tie_grid(1200, 8, 3, 100, 3))
    for cs, store in [(case, few)] + [(c, s) for s in three_stores(c)]:
        labels = random_labels(np.random.default_rng(3), cs[2] + cs[3], 0.5)
        with gpu_index(cs, store, labels) as g:
            check(g, store, cs, RUNS, labels)
    # the few-centre store's results, equal to the oracle's, do hold exact ties
    qs = case[5]
    labels = random_labels(np.random.default_rng(4), case[2] + case[3], 0.5)
    masks = masks_for(qs.shape[0], 0, False)
    want = FT.search_batch_table(O.Index(*case[:5]), store_tables(few, qs), None, 10, 40, labels, masks)
    with gpu_index(case, few, labels) as g:
        same(g.search_batch_filtered_pq(qs, masks, 10, 40), want, "few centres")
    dists, counts = want[1], want[2]
    tied = sum(int(len(np.unique(dists[q][:counts[q]])) < counts[q]) for q in range(qs.shape[0]))
    assert tied > qs.shape[0] // 2, f"only {tied} queries returned tied distances"


@pytest.mark.gpu
def test_overflow_reruns_and_deletions(monkeypatch):
    """visited tables of 256 slots: every query is re-run from its start points, takes the same adaptive decision, and
    the rerank or the filter of deleted ids runs over the whole batch again"""
    case = gpu_case(np.float32, O.L2, d=32)
    vecs, adj, n, n_start, metric, qs = case
    labels = random_labels(np.random.default_rng(11), n + n_start, 0.05)
    gone = np.random.default_rng(3).choice(n, 150, replace=False).astype(np.uint32)
    deleted = np.zeros(n + n_start, bool)
    deleted[gone] = True
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    for store in three_stores(case):
        tables = store_tables(store, qs)
        with gpu_index(case, store, labels) as g:
            check(g, store, case, RUNS, labels, tables=tables)
            g.delete(gone)
            check(g, store, case, RUNS[1:4], labels, deleted=deleted, tables=tables)


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    case = gpu_case(np.float32, O.L2, d=32)
    vecs, adj, n, n_start, metric, qs = case
    labels = random_labels(rng, n + n_start, 0.3)
    gone = rng.choice(n, 200, replace=False).astype(np.uint32)
    deleted = np.zeros(n + n_start, bool)
    deleted[gone] = True
    fresh = (vecs[rng.integers(0, n, 200)] + 0.2 * rng.normal(size=(200, vecs.shape[1]))).astype(np.float32)
    vecs2 = vecs.copy()
    vecs2[gone] = fresh
    for store in three_stores(case):
        lab = labels.copy()
        with gpu_index(case, store, lab) as g:
            g.delete(gone)
            check(g, store, case, RUNS[:4], lab, deleted=deleted)
            # released ids take new rows, whose codes the insert writes to the store, and new labels
            g.release(gone)
            lab[gone] = random_labels(rng, 200, 0.9)
            g.upload_labels(lab)
            g.insert(gone, fresh, 16, 30)
            case2 = (vecs2, g.download_graph(), n, n_start, metric, qs)
            check(g, store, case2, RUNS[:4], lab, tables=store_tables(encoded(store, vecs2), qs))


@pytest.mark.gpu
def test_accept_all_is_the_knn_traversal_of_the_store():
    """an empty ALL mask and no adaptive L: search_batch_{store}'s hops, its cmps less the start points, and its ids up
    to exact ties"""
    case = gpu_case(np.float32, O.L2)
    qs, n, n_start = case[5], case[2], case[3]
    labels = random_labels(np.random.default_rng(1), n + n_start, 0.5)
    for store in three_stores(case):
        kind = kind_of(store)
        with gpu_index(case, store, labels) as g:
            for beam in (1, 3):
                got = getattr(g, f"search_batch_filtered_{kind}")(qs, 0, 10, 40, beam, match_all=True)
                want = getattr(g, f"search_batch_{kind}")(qs, 10, 40, beam)
                assert np.array_equal(got[4], want[4]) and np.array_equal(got[3], want[3] - n_start), (kind, beam)
                assert np.array_equal(got[2], want[2]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), (kind, beam)
                # the list puts a later insertion first among equal distances and the matched list an earlier match:
                # a tie group that the k-th result cuts may keep other ids, so it is compared by size (the distances)
                for q in range(qs.shape[0]):
                    for d in np.unique(want[1][q])[:-1]:
                        assert set(got[0][q][got[1][q] == d]) == set(want[0][q][want[1][q] == d]), (kind, beam, q)


@pytest.mark.gpu
def test_device_form_and_empty_batches():
    import torch
    case = gpu_case(np.float32, O.L2)
    qs = case[5]
    nq, k, L = qs.shape[0], 10, 50
    labels = random_labels(np.random.default_rng(6), case[2] + case[3], 0.1)
    masks = masks_for(nq, 0, False)
    L_ = dab.lib()
    for store in three_stores(case):
        kind = kind_of(store)
        with gpu_index(case, store, labels) as g:
            d_q = torch.from_numpy(qs).cuda()
            d_m = torch.from_numpy(masks.view(np.int64)).cuda()
            launches = dab.launch_count()
            for fn in (getattr(L_, f"dab_search_batch_filtered_{kind}"), getattr(L_, f"dab_search_batch_filtered_{kind}_device")):
                assert fn(g._h, None, 0, k, L, 1, None, 0, 0, 1.0, 1, None, None, None, None, None) == 0
            assert dab.launch_count() == launches, "an empty batch launched a kernel"
            for rr in (False, True):
                want = getattr(g, f"search_batch_filtered_{kind}")(qs, masks, k, L, 2, adaptive_l=(100, 4.0), rerank=rr)
                bufs = (torch.full((nq, k), 7, dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
                        *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
                getattr(g, f"search_batch_filtered_{kind}_device")(d_q.data_ptr(), nq, k, L, 2, d_m.data_ptr(), *(b.data_ptr() for b in bufs),
                                                                   adaptive_l=(100, 4.0), rerank=rr)
                got = [b.cpu().numpy() for b in bufs]  # complete on return: read without a device-wide synchronize
                same(got, want, (kind, rr))


@pytest.mark.gpu
def test_refusals_before_any_launch():
    case = built(600, 16, np.float32, O.L2, 16, seed=31)
    vecs, adj, n, n_start, metric, qs = case
    labels = random_labels(np.random.default_rng(1), n + 1, 0.3)

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
        calls = [g.search_batch_filtered_pq, g.search_batch_filtered_sq, g.search_batch_filtered_minmax]
        # no label table
        for fn in calls:
            assert "dab_upload_labels" in fails(INVALID_ARGUMENT, fn, qs, 1, 10, 20)
        g.upload_labels(labels)
        # no store uploaded, or one set up without rows: the synchronous calls' messages
        assert "no PQ codes" in fails(NOT_READY, g.search_batch_filtered_pq, qs, 1, 10, 20)
        assert "no scalar-quantized rows" in fails(NOT_READY, g.search_batch_filtered_sq, qs, 1, 10, 20)
        assert "no MinMax rows" in fails(NOT_READY, g.search_batch_filtered_minmax, qs, 1, 10, 20)
        g.upload_pq(pq.piv, pq.off)
        assert "no PQ codes" in fails(NOT_READY, g.search_batch_filtered_pq, qs, 1, 10, 20)
        for s in (pq, sq, mm):
            s.upload(g)
        for fn in calls:
            # the arguments of dab_search_batch_filtered, under the called API's name where it names one
            for kk, LL, beam, adaptive, what in ((0, 20, 1, None, "k"), (10, 9, 1, None, "l_value"), (10, 20, 0, None, "beam_width"),
                                                 (10, 20, 65, None, "beam_width"), (10, 20, 1, (100, 0.99), "scale"),
                                                 (10, 20, 1, (100, float("nan")), "scale"), (10, 1024, 1, None, "L + #start"),
                                                 (10, 512, 1, (100, 2.01), "floor(L * scale)")):
                assert what in fails(INVALID_ARGUMENT, fn, qs, 1, kk, LL, beam, adaptive_l=adaptive)
            # rerank without the full-precision vectors
            msg = fails(NOT_READY, fn, qs, 1, 10, 20, rerank=True)
            assert "rerank needs the full-precision vectors" in msg and fn.__name__.replace("search_batch", "dab_search_batch") in msg
            assert fn(qs, 1, 10, 20)[2].shape == (16,)  # without rerank the rows are not needed
        # a MinMax query holding a NaN fails the call, naming it
        bad = qs.copy()
        bad[3, 4] = np.nan
        assert "query 3 contains NaN after the transform (InputContainsNaN)" in fails(INVALID_ARGUMENT, g.search_batch_filtered_minmax, bad,
                                                                                     1, 10, 20, staged=True)
        g.upload_vectors(vecs)
        for s in (pq, sq, mm):  # the index is usable after every refusal
            check(g, s, case, [(10, 20, 1, False, (30, 2.0))], labels)
    # the shared memory of the kernel with the store's query area: L = 512 grown to 1024 with 64 beams of wide rows does
    # not fit, 8 beams do
    n2, md = 100, 200
    vz = np.zeros((n2 + 1, 16), np.float32)
    az = np.zeros((n2 + 1, md + 1), np.uint32)
    with dab.GpuIndex(dab.DType.f32, O.L2, 16, n2, 1, md) as g:
        g.upload_vectors(vz)
        g.upload_graph(az)
        g.upload_labels(np.ones(n2 + 1, np.uint64))
        g.upload_sq(8, *sq.quantizer)
        g.sq_encode_all()
        z = np.zeros((4, 16), np.float32)
        assert "shared memory" in fails(INVALID_ARGUMENT, g.search_batch_filtered_sq, z, 1, 10, 512, 64, adaptive_l=(10, 2.0))
        assert g.search_batch_filtered_sq(z, 1, 10, 512, 8, adaptive_l=(10, 2.0))[2].tolist() == [0] * 4
    with dab.GpuIndex(dab.DType.f32, O.COSINE, 16, n, 1, adj.shape[1] - 1) as g:
        g.upload_graph(adj)
        g.upload_labels(labels)
        sq.upload(g)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(INVALID_ARGUMENT, g.search_batch_filtered_sq, qs, 1, 10, 20)
