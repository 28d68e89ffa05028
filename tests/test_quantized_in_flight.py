"""Batches in flight on the PQ, SQ and MinMax traversals: dab_search_batch_{pq,sq,minmax}[_device]_async / dab_wait.

Every slot is filled with a batch of uneven size before any is joined, the slots are joined out of order, and each
batch's ids, distance bits, counts, cmps and hops must equal the synchronous call's and the oracle's — with tables sized
as usual and with 256-slot visited tables, whose overflowed queries are re-run (and the batch re-ranked) inside
dab_wait.  Then batches of different kinds share the slots with synchronous calls on the handle's stream, and the slot
rules and launch-time errors hold."""
import functools

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
from test_gpu_parity import clustered, make_index, sq_quantizer, trained_pq
from test_minmax_search import MinMaxOracle, compress, index_rows, make_transform

pytestmark = pytest.mark.gpu

FIVE = ("ids", "dists", "counts", "cmps", "hops")
SIZES = (200, 64, 333, 1)  # one batch per slot
ORDER = (2, 0, 3, 1)       # the order the slots are joined in
K, L, BEAM = 10, 60, 1


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def fill_and_join(g, launch, batches):
    """launch(slot, queries) queues a batch and returns its outputs; every slot is filled before the first join"""
    assert len(batches) == dab.MAX_SLOTS
    outs = [launch(s, q) for s, q in enumerate(batches)]
    for s in ORDER:
        g.wait(s)
    return outs


def fill_and_join_device(g, launch, batches):
    """the device flavour: launch(slot, d_queries, nq, d_ids, d_dists, d_counts, d_cmps, d_hops)"""
    import torch
    bufs = []
    for q in batches:
        nq = q.shape[0]
        bufs.append((torch.from_numpy(q.view(np.uint8).copy()).cuda(), torch.empty((nq, K), dtype=torch.int32, device="cuda"),
                     torch.empty((nq, K), dtype=torch.float32, device="cuda"),
                     *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3))))
    torch.cuda.synchronize()  # the slots' streams do not wait for torch's
    for s, (q, b) in enumerate(zip(batches, bufs)):
        launch(s, b[0].data_ptr(), q.shape[0], *(t.data_ptr() for t in b[1:]))
    for s in ORDER:
        g.wait(s)
    return [[t.cpu().numpy() for t in b[1:]] for b in bufs]


def check_in_flight(g, sync, host_async, device_async, batches, want, what):
    """sync(q, rerank), host_async(slot, q, rerank), device_async(slot, d_q, nq, ..., rerank) against want[rerank][i]"""
    if "overflow" in what:  # the visited sets of some queries of every batch pass 7/8 of a 256-slot table
        assert all((w[3] > 224).any() for w in want[False] if w[3].shape[0] > 1), what
    for rerank in (False, True):
        for i, q in enumerate(batches):
            same(sync(q, rerank), want[rerank][i], (what, "sync", rerank, i))
        for rounds in range(2):  # slots are reusable
            outs = fill_and_join(g, lambda s, q: host_async(s, q, rerank), batches)
            for i, got in enumerate(outs):
                same(got, want[rerank][i], (what, "host", rerank, rounds, i))
        outs = fill_and_join_device(g, lambda s, *a: device_async(s, *a, rerank=rerank), batches)
        for i, got in enumerate(outs):
            same(got, want[rerank][i], (what, "device", rerank, i))


def set_tables(monkeypatch, tables):
    if tables == "overflow":
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")


# ---------------------------------------------------------------- PQ

@functools.lru_cache(maxsize=None)
def pq_case(metric):
    rng = np.random.default_rng(41 + metric)
    n, d, chunks = 3000, 64, 16
    vecs, adj, maxdeg = make_index(rng, np.float32, metric, n, d, 24, 40)
    piv, off = trained_pq(rng, vecs[:n], chunks)
    codes = np.zeros((n + 1, chunks), np.uint8)
    for i in range(n + 1):
        assert O.lib().orc_pq_encode(O.ptr(piv), 256, d, O.ptr(off), chunks, O.ptr(vecs[i]), O.ptr(codes[i])) == 0
    batches = [clustered(rng, m, d) for m in SIZES]
    oidx = O.Index(vecs, adj, n, 1, metric, pq=(piv, off, codes))
    want = {False: [oidx.search_batch(q, K, L, beam=BEAM, threads=4) for q in batches],
            True: [oidx.search_batch_rerank(q, K, L, beam=BEAM, threads=4) for q in batches]}
    return n, d, vecs, adj, maxdeg, piv, off, codes, batches, want


@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("path", ["smem_pivots", "global_lut"])
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE])  # TableL2, TableIP, DirectCosine
def test_pq_batches_in_flight_equal_the_synchronous_call_and_the_oracle(monkeypatch, metric, path, tables):
    if path == "global_lut":
        monkeypatch.setenv("DAB_TEST_PQ_GLOBAL_LUT", "1")
    set_tables(monkeypatch, tables)
    n, d, vecs, adj, maxdeg, piv, off, codes, batches, want = pq_case(metric)
    with dab.GpuIndex(dab.DType.f32, metric, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_pq(piv, off, codes)
        check_in_flight(g, lambda q, r: g.search_batch_pq(q, K, L, BEAM, rerank=r),
                        lambda s, q, r: g.search_batch_pq_async(s, q, K, L, BEAM, rerank=r),
                        lambda s, *a, rerank: g.search_batch_pq_device_async(s, a[0], a[1], K, L, BEAM, *a[2:], rerank=rerank),
                        batches, want, ("pq", metric, path, tables))


# ---------------------------------------------------------------- SQ

@functools.lru_cache(maxsize=None)
def sq_case(metric, nbits):
    rng = np.random.default_rng(43 + 10 * metric + nbits)
    n, d = 3000, 64
    vecs, adj, maxdeg = make_index(rng, np.float32, metric, n, d, 24, 40)
    shift, scale, ssn, mean_norm = sq_quantizer(vecs, metric)
    rows = O.sq_encode_rows(vecs, shift, scale, nbits)
    batches = [clustered(rng, m, d) for m in SIZES]
    oidx = O.Index(vecs, adj, n, 1, metric, sq=(rows, nbits, shift, scale, ssn, mean_norm))
    want = {False: [oidx.search_batch(q, K, L, beam=BEAM, threads=4) for q in batches],
            True: [oidx.search_batch_rerank(q, K, L, beam=BEAM, threads=4) for q in batches]}
    return n, d, vecs, adj, maxdeg, (nbits, shift, scale, ssn, mean_norm), rows, batches, want


@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("metric,nbits", [(O.L2, 8), (O.INNER_PRODUCT, 4)])
def test_sq_batches_in_flight_equal_the_synchronous_call_and_the_oracle(monkeypatch, metric, nbits, tables):
    set_tables(monkeypatch, tables)
    n, d, vecs, adj, maxdeg, quantizer, rows, batches, want = sq_case(metric, nbits)
    with dab.GpuIndex(dab.DType.f32, metric, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_sq(*quantizer, rows=rows)
        check_in_flight(g, lambda q, r: g.search_batch_sq(q, K, L, BEAM, rerank=r),
                        lambda s, q, r: g.search_batch_sq_async(s, q, K, L, BEAM, rerank=r),
                        lambda s, *a, rerank: g.search_batch_sq_device_async(s, a[0], a[1], K, L, BEAM, *a[2:], rerank=rerank),
                        batches, want, ("sq", metric, nbits, tables))


# ---------------------------------------------------------------- MinMax

@functools.lru_cache(maxsize=None)
def minmax_case(nbits, kind):
    rng = np.random.default_rng(47 + nbits)
    n, d = 2500, 64
    vecs = index_rows(rng, np.float32, n, d)
    maxdeg = 31
    adj = O.build_graph(vecs, n, 1, O.L2, 24, maxdeg, 40)
    t = make_transform(kind, d)
    rows = compress(vecs, t, nbits)
    batches = [np.ascontiguousarray(vecs[rng.integers(0, n, m)]) for m in SIZES]
    oidx = MinMaxOracle(vecs, adj, n, 1, O.L2, rows, nbits)
    want = {r: [oidx.search(q, compress(q, t, nbits), K, L, beam=BEAM, rerank=r) for q in batches] for r in (False, True)}
    return n, d, vecs, adj, maxdeg, rows, batches, want


@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("kind", [None, "double_same"])
@pytest.mark.parametrize("nbits", [8, 4])
def test_minmax_batches_in_flight_equal_the_synchronous_call_and_the_oracle(monkeypatch, nbits, kind, tables):
    set_tables(monkeypatch, tables)
    n, d, vecs, adj, maxdeg, rows, batches, want = minmax_case(nbits, kind)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_minmax(nbits, 1.0, make_transform(kind, d), rows=rows)
        check_in_flight(g, lambda q, r: g.search_batch_minmax(q, K, L, BEAM, rerank=r),
                        lambda s, q, r: g.search_batch_minmax_async(s, q, K, L, BEAM, rerank=r),
                        lambda s, *a, rerank: g.search_batch_minmax_device_async(s, a[0], a[1], K, L, BEAM, *a[2:], rerank=rerank),
                        batches, want, ("minmax", nbits, kind, tables))


# ---------------------------------------------------------------- kinds mixed, slot rules, errors

def mixed_index(g):
    """the SQ case's index with its SQ rows and a MinMax-8 store beside them"""
    n, d, vecs, adj, maxdeg, quantizer, rows, batches, _ = sq_case(O.L2, 8)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    g.upload_sq(*quantizer, rows=rows)
    g.upload_minmax(8, 1.0, None, rows=compress(vecs, None, 8))
    return batches


@pytest.mark.parametrize("tables", ["sized", "overflow"])
def test_kinds_mixed_on_the_slots_and_the_handle_stream(monkeypatch, tables):
    """A full-precision, an SQ and a MinMax batch in flight on three slots, with synchronous quantized calls on the
    handle's stream in between: each equals its synchronous result."""
    set_tables(monkeypatch, tables)
    n, d, vecs, adj, maxdeg = sq_case(O.L2, 8)[:5]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        b = mixed_index(g)
        want_fp = g.search_batch(b[0], K, L)
        want_sq = g.search_batch_sq(b[1], K, L, rerank=True)
        want_mm = g.search_batch_minmax(b[2], K, L, rerank=True)
        want_sq2 = g.search_batch_sq(b[3], K, L)
        want_mm2 = g.search_batch_minmax(b[0], K, L)
        fp = g.search_batch_async(0, b[0], K, L)
        sq = g.search_batch_sq_async(1, b[1], K, L, rerank=True)
        sync_mm = g.search_batch_minmax(b[0], K, L)
        mm = g.search_batch_minmax_async(2, b[2], K, L, rerank=True)
        sync_sq = g.search_batch_sq(b[3], K, L)
        for s in (2, 0, 1):
            g.wait(s)
        same(fp, want_fp, "fp")
        same(sq, want_sq, "sq")
        same(mm, want_mm, "minmax")
        same(sync_sq, want_sq2, "sync sq")
        same(sync_mm, want_mm2, "sync minmax")


def test_slot_rules_and_launch_time_errors():
    """A slot holding a batch of any kind rejects another; a slot out of range is rejected; waiting on an idle slot is a
    no-op; every error the synchronous call reports before it launches is returned by the launching call and leaves the
    slot idle; a MinMax NaN query fails at dab_wait with the synchronous call's message and the slot is reusable."""
    n, d, vecs, adj, maxdeg, quantizer, rows, batches, _ = sq_case(O.L2, 8)
    lib = dab.lib()

    def fails(code, fn, *args, **kw):
        with pytest.raises(dab.DabError) as e:
            fn(*args, **kw)
        assert e.value.code == code, str(e.value)
        return str(e.value)

    def idle(g, slot):
        """the slot takes a batch and returns the synchronous call's results"""
        out = g.search_batch_sq_async(slot, batches[1], K, L)
        g.wait(slot)
        same(out, g.search_batch_sq(batches[1], K, L), ("idle", slot))

    q = batches[1]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_graph(adj)
        g.wait(3)  # idle: no-op
        # stores that are not ready
        assert "no PQ codes" in fails(5, g.search_batch_pq_async, 0, q, K, L)
        assert "no scalar-quantized rows" in fails(5, g.search_batch_sq_async, 0, q, K, L)
        assert "no MinMax rows" in fails(5, g.search_batch_minmax_async, 0, q, K, L)
        g.upload_sq(*quantizer, rows=rows)
        g.upload_minmax(8, 1.0, None, rows=compress(vecs, None, 8))
        # rerank without the full-precision rows
        assert "rerank needs the full-precision vectors" in fails(5, g.search_batch_sq_async, 0, q, K, L, rerank=True)
        assert "rerank needs the full-precision vectors" in fails(5, g.search_batch_minmax_async, 1, q, K, L, rerank=True)
        g.upload_vectors(vecs)
        # L + #start > 1024
        assert "L + #start must be <= 1024" in fails(1, g.search_batch_sq_async, 0, q, K, 1024)
        assert "L + #start must be <= 1024" in fails(1, g.search_batch_minmax_async, 2, q, K, 1024)
        # NULL buffers, both flavours
        for name in ("dab_search_batch_sq_async", "dab_search_batch_sq_device_async", "dab_search_batch_minmax_async",
                     "dab_search_batch_minmax_device_async", "dab_search_batch_pq_async", "dab_search_batch_pq_device_async"):
            assert getattr(lib, name)(g._h, 0, None, 5, K, L, 1, 0, None, None, None, None, None) == 1, name
            assert b"NULL argument" in lib.dab_last_error()
        # slot out of range
        assert "out of range" in fails(1, g.search_batch_sq_async, dab.MAX_SLOTS, q, K, L)
        assert "out of range" in fails(1, g.search_batch_minmax_async, dab.MAX_SLOTS, q, K, L)
        for s in range(dab.MAX_SLOTS):
            idle(g, s)
        # a slot holding a batch of another kind
        g.search_batch_async(1, q, K, L)
        assert "still has a batch in flight" in fails(1, g.search_batch_sq_async, 1, q, K, L)
        assert "still has a batch in flight" in fails(1, g.search_batch_minmax_async, 1, q, K, L)
        g.wait(1)
        g.search_batch_minmax_async(2, q, K, L)
        assert "still has a batch in flight" in fails(1, g.search_batch_async, 2, q, K, L)
        assert "still has a batch in flight" in fails(1, g.search_batch_sq_async, 2, q, K, L)
        g.wait(2)
        # a MinMax query holding a NaN: the launch succeeds, dab_wait fails with the synchronous call's message
        bad = q.copy()
        bad[3, 4] = np.nan
        sync_msg = fails(1, g.search_batch_minmax, bad, K, L)
        assert "query 3 contains NaN after the transform (InputContainsNaN)" in sync_msg
        g.search_batch_minmax_async(0, bad, K, L, rerank=True)
        assert fails(1, g.wait, 0) == sync_msg
        g.wait(0)  # idle again
        idle(g, 0)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.Cosine, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_sq(*quantizer, rows=rows)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(1, g.search_batch_sq_async, 0, q, K, L)
        g.wait(0)


def test_replacing_a_store_under_a_batch_in_flight_never_reruns_on_the_freed_store(monkeypatch):
    """The calls that free a quantized store wait for the slots first, and a batch planned on the old store is never
    launched again: with 256-slot visited tables its overflowed queries would need a re-run, so dab_wait fails with
    its own message instead.  The slot is idle afterwards and the new store searches as the synchronous call does."""
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    n, d, vecs, adj, maxdeg, quantizer, rows, batches, _ = sq_case(O.L2, 8)
    piv, off = trained_pq(np.random.default_rng(5), vecs[:n], 16)
    mm_rows = compress(vecs, None, 8)
    q = batches[0]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_sq(*quantizer, rows=rows)
        g.upload_minmax(8, 1.0, None, rows=mm_rows)
        g.upload_pq(piv, off)
        g.pq_encode_all()
        kinds = [(g.search_batch_sq_async, g.search_batch_sq, lambda: g.upload_sq(*quantizer, rows=rows)),
                 (g.search_batch_minmax_async, g.search_batch_minmax, lambda: g.upload_minmax(8, 1.0, None, rows=mm_rows)),
                 (g.search_batch_pq_async, g.search_batch_pq, lambda: (g.upload_pq(piv, off), g.pq_encode_all()))]
        for slot, (launch, sync, replace) in enumerate(kinds):
            launch(slot, q, K, L, rerank=True)
            replace()
            with pytest.raises(dab.DabError) as e:
                g.wait(slot)
            assert e.value.code == 1 and "replaced while the batch was in flight" in str(e.value), str(e.value)
            g.wait(slot)  # idle
            out = launch(slot, q, K, L, rerank=True)
            g.wait(slot)
            same(out, sync(q, K, L, rerank=True), ("after the replacement", slot))
