"""Diversity-aware search on the device (dab_upload_attributes, dab_search_batch_diverse[_device]) bit for bit against
the oracle's Diverse::search (oracle/diverse_search.cpp, pinned in test_diverse_search.py): ids, distance bits, counts,
cmps and hops over every row type and metric, attribute cardinalities from one to all-distinct, ids and start points
without attributes, diverse_k below, at and above k, lists from k to several hundred entries, beams of 1 and 4, the
edge graphs of test_traversal_edges.py (many start points, malformed rows, non-finite rows, exact ties), deletions,
inserts into released ids, and the overflow re-runs of the visited tables and of the local-queue pool."""
import numpy as np
import pytest

import diskann_b200 as dab
import diverse_oracle as D
import oracle_lib as O
from test_gpu_parity import make_index
from test_traversal_edges import grid, malformed_case, many_starts, non_finite

FIVE = ("ids", "dists", "counts", "cmps", "hops")
INVALID_ARGUMENT = 1  # DAB_ERR_INVALID_ARGUMENT (include/diskann_b200.h)


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


def gpu_index(vecs, adj, n, n_start, metric, max_degree):
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


def check(g, oidx, queries, runs, values, present, deleted=None):
    """every (k, L, beam, diverse_k) of `runs` on the device against the oracle; returns the oracle's failed removals"""
    failed = 0
    for k, L, beam, dk in runs:
        want = D.search_batch(oidx, queries, k, L, dk, values, present, beam=beam, deleted=deleted)
        same(g.search_batch_diverse(queries, k, L, dk, beam), want[:5], (k, L, beam, dk))
        failed += int(want[5].sum())
    return failed


RUNS = [(10, 10, 1, 1), (10, 40, 1, 3), (10, 40, 4, 10), (10, 64, 1, 25), (5, 300, 4, 2), (20, 20, 1, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric,d,n,R,Lb", [
    (np.float32, O.L2, 128, 3000, 24, 40),
    (np.float32, O.INNER_PRODUCT, 64, 2000, 16, 30),
    (np.float32, O.COSINE, 48, 2000, 16, 30),
    (np.float32, O.COSINE_NORMALIZED, 32, 2000, 16, 30),
    (np.float16, O.L2, 64, 2000, 16, 30),
    (np.float16, O.INNER_PRODUCT, 96, 2000, 16, 30),
    (np.float16, O.COSINE, 64, 2000, 16, 30),
    (np.int8, O.L2, 128, 2000, 16, 30),
    (np.int8, O.COSINE, 64, 2000, 16, 30),
    (np.uint8, O.L2, 128, 2000, 16, 30),
    (np.uint8, O.INNER_PRODUCT, 40, 2000, 16, 30),
])
def test_row_types_and_metrics(dt, metric, d, n, R, Lb):
    rng = np.random.default_rng(d + n)
    vecs, adj, maxdeg = make_index(rng, dt, metric, n, d, R, Lb)
    nq = 200
    queries = vecs[rng.integers(0, n, nq)].astype(np.float32) + 0.1 * rng.normal(size=(nq, d)).astype(np.float32)
    if dt in (np.int8, np.uint8):
        info = np.iinfo(dt)
        queries = np.clip(np.round(queries), info.min, info.max)
    queries = queries.astype(dt)
    oidx = O.Index(vecs, adj, n, 1, metric)
    with gpu_index(vecs, adj, n, 1, metric, maxdeg) as g:
        for kind in (1, 5, "distinct"):
            values, present = attributes(n + 1, kind, d)
            g.upload_attributes(values, present)
            check(g, oidx, queries, RUNS, values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [1, 2, 5, 64, "distinct", "half"])
def test_cardinalities(kind):
    rng = np.random.default_rng(7)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 4000, 64, 24, 40)
    n = 4000
    queries = (vecs[rng.integers(0, n, 300)] + 0.1 * rng.normal(size=(300, 64))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    values, present = attributes(n + 1, kind, 3)
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
        g.upload_attributes(values, present)
        check(g, oidx, queries, RUNS + [(10, 700, 1, 3), (10, 1024, 2, 1)], values, present)


@pytest.mark.gpu
def test_start_points_without_attributes():
    case = many_starts(1500, 16, 33, 100, 3)
    values, present = attributes(case.total, 5, 4)
    present[case.n:] = 0
    present[case.n + 7] = 1  # one start point keeps its attribute: the search starts from it alone
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
        g.upload_attributes(values, present)
        check(g, case.oracle, case.queries, RUNS, values, present)
        present[case.n + 7] = 0
        g.upload_attributes(values[case.n:], present[case.n:], first=case.n)
        got = g.search_batch_diverse(case.queries, 10, 20, 2)
        assert (got[2] == 0).all() and (got[4] == 0).all() and (got[3] == case.n_start).all()
        check(g, case.oracle, case.queries, RUNS[:2], values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 70])
def test_many_start_points(n_start):
    case = many_starts(1500, 16, n_start, 100, n_start)
    values, present = attributes(case.total, 5, n_start)
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
        g.upload_attributes(values, present)
        check(g, case.oracle, case.queries, RUNS, values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("max_degree", [1, 7, 40])
def test_malformed_rows(max_degree):
    case = malformed_case(800, 8, 3, max_degree, 80, max_degree)
    values, present = attributes(case.total, "half", max_degree)
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
        g.upload_attributes(values, present)
        check(g, case.oracle, case.queries, RUNS, values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.L2)])
def test_non_finite_rows(dt, metric):
    case, _ = non_finite(800, 16, dt, metric, 80, 7, nan=dt == np.float32)
    values, present = attributes(case.total, 5, 1)
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
        g.upload_attributes(values, present)
        check(g, case.oracle, case.queries, RUNS, values, present)


@pytest.mark.gpu
@pytest.mark.parametrize("card", [2, 5, 64])
def test_exact_ties_drift(card, monkeypatch):
    """exact ties make removals fail: the local queues drift from the list, and a pool of 4 entries overflows"""
    case = grid(1200, 8, 3, 100, 3)
    values = (np.arange(case.total) % card).astype(np.uint32)
    present = np.ones(case.total, np.uint8)
    runs = [(10, 30, 1, 1), (10, 60, 2, 3), (5, 200, 4, 2), (10, 100, 1, 10)]
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
        g.upload_attributes(values, present)
        assert check(g, case.oracle, case.queries, runs, values, present) > 0, "no removal failed"
    for var, val in (("DAB_TEST_DIVERSE_POOL", "4"), ("DAB_TEST_VISITED_LOG2", "8")):
        monkeypatch.setenv(var, val)
        with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
            g.upload_attributes(values, present)
            check(g, case.oracle, case.queries, runs, values, present)
        monkeypatch.delenv(var)


@pytest.mark.gpu
def test_overflow_reruns(monkeypatch):
    """visited tables of 256 slots and local-queue pools of one entry: every query is re-run, some several times"""
    rng = np.random.default_rng(11)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    n = 3000
    queries = (vecs[rng.integers(0, n, 200)] + 0.1 * rng.normal(size=(200, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    values, present = attributes(n + 1, 5, 2)
    for env in ({"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_DIVERSE_POOL": "1"}, {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_DIVERSE_POOL": "3"}):
        for var, val in env.items():
            monkeypatch.setenv(var, val)
        with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
            g.upload_attributes(values, present)
            check(g, oidx, queries, RUNS, values, present)
        for var in env:
            monkeypatch.delenv(var)


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    n = 3000
    queries = (vecs[rng.integers(0, n, 200)] + 0.1 * rng.normal(size=(200, 32))).astype(np.float32)
    values, present = attributes(n + 1, 5, 9)
    gone = rng.choice(n, 300, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
        g.upload_attributes(values, present)
        g.delete(gone)
        check(g, O.Index(vecs, adj, n, 1, O.L2), queries, RUNS, values, present, deleted)
        # released ids take new rows and new attributes; the table was left as it was by delete and release
        g.release(gone)
        fresh = (vecs[rng.integers(0, n, 300)] + 0.2 * rng.normal(size=(300, 32))).astype(np.float32)
        values[gone] = rng.integers(100, 103, 300)
        present[gone[::3]] = 0
        for i in gone:
            g.upload_attributes(values[i:i + 1], present[i:i + 1], first=int(i))
        g.insert(gone, fresh, 16, 30)
        vecs2 = vecs.copy()
        vecs2[gone] = fresh
        adj2 = g.download_graph()
        check(g, O.Index(vecs2, adj2, n, 1, O.L2), queries, RUNS, values, present)


@pytest.mark.gpu
def test_device_form_and_argument_errors():
    import torch
    rng = np.random.default_rng(2)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 2000, 32, 16, 30)
    n, nq, k, L = 2000, 100, 10, 50
    queries = (vecs[rng.integers(0, n, nq)] + 0.1 * rng.normal(size=(nq, 32))).astype(np.float32)
    values, present = attributes(n + 1, 5, 6)
    L_ = dab.lib()
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
        launches = dab.launch_count()
        h = g._h
        # no attribute table yet
        assert L_.dab_search_batch_diverse(h, O.ptr(queries), nq, k, L, 1, 2, None, None, None, None, None) == INVALID_ARGUMENT
        assert b"dab_upload_attributes" in L_.dab_last_error()
        g.upload_attributes(values, present)
        for kk, LL, beam, dk, what in ((0, L, 1, 2, b"k"), (k, L, 1, 0, b"diverse k_value"), (k, k - 1, 1, 2, b"l_value"),
                                       (k, 1025, 1, 2, b"1024"), (k, L, 0, 2, b"beam_width")):
            for fn in (L_.dab_search_batch_diverse, L_.dab_search_batch_diverse_device):
                assert fn(h, O.ptr(queries), nq, kk, LL, beam, dk, None, None, None, None, None) == INVALID_ARGUMENT, what
                assert what in L_.dab_last_error(), (what, L_.dab_last_error())
        assert dab.launch_count() == launches, "an argument error launched a kernel"
        v = np.zeros(4, np.uint32)
        assert L_.dab_upload_attributes(h, O.ptr(v), None, n - 2, 4) == INVALID_ARGUMENT
        assert L_.dab_upload_attributes(h, None, None, 0, 4) == INVALID_ARGUMENT
        # diverse_k > k is accepted, as in the reference
        g.search_batch_diverse(queries, k, L, k + 5)
        want = g.search_batch_diverse(queries, k, L, 2, 2)
        d_q = torch.from_numpy(queries).cuda()
        bufs = (torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
                *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
        g.search_batch_diverse_device(d_q.data_ptr(), nq, k, L, 2, 2, *(b.data_ptr() for b in bufs))
        torch.cuda.synchronize()
        got = [b.cpu().numpy() for b in bufs]
        same(got, want, "device form")


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.INNER_PRODUCT, O.L2])
def test_diverse_k_beyond_32_bits_of_local_capacity(metric):
    """diverse_k * L / k past 2^32 (diverse_k = 2^30, "no limit"): every local queue is larger than the index, so the
    search is the k-NN search over a list of L without eviction by attribute; inner product gives negative distances"""
    rng = np.random.default_rng(13)
    vecs, adj, maxdeg = make_index(rng, np.float32, metric, 2000, 32, 16, 30)
    n = 2000
    queries = (vecs[rng.integers(0, n, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, metric)
    with gpu_index(vecs, adj, n, 1, metric, maxdeg) as g:
        for kind in (1, 5):
            values, present = attributes(n + 1, kind, 8)
            g.upload_attributes(values, present)
            check(g, oidx, queries, [(10, 40, 1, 1 << 30), (10, 40, 4, 0xFFFFFFFF), (5, 300, 1, 1 << 22)], values, present)
            got = g.search_batch_diverse(queries, 10, 40, 1 << 30)
            assert (got[2] == 10).all()


@pytest.mark.gpu
def test_shared_memory_limit_is_an_argument_error():
    """L = 1024 with 64 beams of 200-neighbour rows needs more than 200 KB of shared memory per CTA: refused with the
    other argument errors, before any launch"""
    n, d, md = 100, 32, 200
    vecs = np.zeros((n + 1, d), np.float32)
    adj = np.zeros((n + 1, md + 1), np.uint32)
    L_ = dab.lib()
    queries = np.zeros((4, d), np.float32)
    with gpu_index(vecs, adj, n, 1, O.L2, md) as g:
        g.upload_attributes(np.zeros(n + 1, np.uint32))
        launches = dab.launch_count()
        for fn in (L_.dab_search_batch_diverse, L_.dab_search_batch_diverse_device):
            assert fn(g._h, O.ptr(queries), 4, 10, 1024, 64, 1, None, None, None, None, None) == INVALID_ARGUMENT
            assert b"shared memory" in L_.dab_last_error()
        assert dab.launch_count() == launches
        assert g.search_batch_diverse(queries, 10, 1024, 1, 8)[2].tolist() == [0] * 4  # a fitting beam runs
