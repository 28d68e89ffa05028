"""Filtered search on the device (dab_upload_labels, dab_search_batch_filtered[_device]) bit for bit against the oracle's
InlineFilterSearch (oracle/filtered_search.cpp, pinned in test_filtered_search.py): ids, distance bits, counts, cmps and
hops over every row type and metric, selectivities from accept-all to accept-none in ANY and ALL modes, beams 1 / 2 / 4,
adaptive L off and in every multiplier region up to L * scale = 1024, many start points (accepted, rejected, lists that
reconfigure cuts), deletions and inserted points, the edge graphs of test_traversal_edges.py, the visited-table re-runs,
empty batches, the device-pointer call and the argument checks."""
import numpy as np
import pytest

import diskann_b200 as dab
import filtered_oracle as F
import oracle_lib as O
from test_filtered_search import random_labels
from test_gpu_parity import make_index
from test_traversal_edges import grid, malformed_case, many_starts, non_finite

FIVE = ("ids", "dists", "counts", "cmps", "hops")
INVALID_ARGUMENT = 1  # DAB_ERR_INVALID_ARGUMENT (include/diskann_b200.h)
SELECTIVITY = (1.0, 0.5, 0.1, 0.01, 0.0)
# (k, L, beam, match_all, adaptive_l)
RUNS = [(10, 10, 1, False, None), (10, 40, 2, True, None), (10, 40, 1, False, (50, 2.0)), (10, 64, 4, False, (200, 8.0)),
        (5, 100, 1, True, (1000, 8.0)), (10, 20, 1, False, (30, 3.7))]


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def gpu_index(vecs, adj, n, n_start, metric, max_degree, labels):
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    g.upload_labels(labels)
    return g


def masks_for(nq, seed, match_all):
    """ANY: bit 0 (the selectivity bit) and, for every third query, bits 0 and 3; ALL: bit 0 and, for every third query,
    bits 0 and 5; one query in seven with the empty mask"""
    m = np.ones(nq, np.uint64)
    m[::3] |= np.uint64(1 << (5 if match_all else 3))
    m[::7] = 0
    return m


def check(g, oidx, queries, labels, runs, deleted=None):
    for k, L, beam, match_all, adaptive in runs:
        masks = masks_for(queries.shape[0], L, match_all)
        want = F.search_batch(oidx, queries, k, L, labels, masks, match_all, adaptive, beam=beam, deleted=deleted)
        same(g.search_batch_filtered(queries, masks, k, L, beam, match_all, adaptive), want, (k, L, beam, match_all, adaptive))


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
    nq = 150
    queries = vecs[rng.integers(0, n, nq)].astype(np.float32) + 0.1 * rng.normal(size=(nq, d)).astype(np.float32)
    if dt in (np.int8, np.uint8):
        info = np.iinfo(dt)
        queries = np.clip(np.round(queries), info.min, info.max)
    queries = queries.astype(dt)
    oidx = O.Index(vecs, adj, n, 1, metric)
    labels = random_labels(rng, n + 1, 0.1)
    with gpu_index(vecs, adj, n, 1, metric, maxdeg, labels) as g:
        check(g, oidx, queries, labels, RUNS)


@pytest.mark.gpu
@pytest.mark.parametrize("selectivity", SELECTIVITY)
def test_selectivities(selectivity):
    rng = np.random.default_rng(int(selectivity * 1000))
    n = 4000
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, n, 64, 24, 40)
    queries = (vecs[rng.integers(0, n, 300)] + 0.1 * rng.normal(size=(300, 64))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    labels = random_labels(rng, n + 1, selectivity)
    runs = RUNS + [(10, 128, 1, False, (1000, 8.0)), (10, 512, 2, False, (100, 2.0)), (1, 1, 1, True, (1, 1024.0))]
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg, labels) as g:
        check(g, oidx, queries, labels, runs)


@pytest.mark.gpu
def test_adaptive_regions_and_the_longest_list():
    """samples that fire with specificity >= 0.5, in [0.1, 0.5), below 0.1 and at zero; L * scale == 1024 exactly"""
    rng = np.random.default_rng(21)
    n = 5000
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, n, 32, 24, 40)
    queries = (vecs[rng.integers(0, n, 200)] + 0.1 * rng.normal(size=(200, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    for sel in (0.8, 0.3, 0.03, 0.003, 0.0):
        labels = random_labels(rng, n + 1, sel)
        runs = [(10, 64, 1, False, (100, 16.0)), (10, 128, 2, False, (300, 8.0)), (10, 256, 4, False, (64, 4.0)),
                (10, 100, 1, False, (500, 10.24))]
        with gpu_index(vecs, adj, n, 1, O.L2, maxdeg, labels) as g:
            check(g, oidx, queries, labels, runs)


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 70])
def test_many_start_points(n_start):
    """start points accepted and rejected, and adaptive L's reconfigure cutting a list of L + #start entries"""
    case = many_starts(1500, 16, n_start, 100, n_start)
    rng = np.random.default_rng(n_start)
    labels = random_labels(rng, case.total, 0.3)
    runs = RUNS + [(5, 10, 1, False, (1, 2.0)), (5, 10, 2, False, (5, 1.5))]
    for start_label in (0, 1):
        labels[case.n:] = start_label
        with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree, labels) as g:
            check(g, case.oracle, case.queries, labels, runs)


@pytest.mark.gpu
@pytest.mark.parametrize("max_degree", [1, 7, 40])
def test_malformed_rows(max_degree):
    case = malformed_case(800, 8, 3, max_degree, 80, max_degree)
    labels = random_labels(np.random.default_rng(max_degree), case.total, 0.2)
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree, labels) as g:
        check(g, case.oracle, case.queries, labels, RUNS)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.L2)])
def test_non_finite_rows(dt, metric):
    case, _ = non_finite(800, 16, dt, metric, 80, 7, nan=dt == np.float32)
    labels = random_labels(np.random.default_rng(1), case.total, 0.5)
    with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree, labels) as g:
        check(g, case.oracle, case.queries, labels, RUNS)


@pytest.mark.gpu
def test_exact_ties(monkeypatch):
    case = grid(1200, 8, 3, 100, 3)
    labels = random_labels(np.random.default_rng(3), case.total, 0.5)
    for env in (None, "8"):
        if env:
            monkeypatch.setenv("DAB_TEST_VISITED_LOG2", env)
        with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree, labels) as g:
            check(g, case.oracle, case.queries, labels, RUNS)


@pytest.mark.gpu
def test_overflow_reruns(monkeypatch):
    """visited tables of 256 slots: queries are re-run from their start points and take the same adaptive decision"""
    rng = np.random.default_rng(11)
    n = 3000
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, n, 32, 16, 30)
    queries = (vecs[rng.integers(0, n, 200)] + 0.1 * rng.normal(size=(200, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    labels = random_labels(rng, n + 1, 0.05)
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg, labels) as g:
        check(g, oidx, queries, labels, RUNS)


@pytest.mark.gpu
def test_deleted_and_inserted_points():
    rng = np.random.default_rng(5)
    n = 3000
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, n, 32, 16, 30)
    queries = (vecs[rng.integers(0, n, 200)] + 0.1 * rng.normal(size=(200, 32))).astype(np.float32)
    labels = random_labels(rng, n + 1, 0.3)
    gone = rng.choice(n, 300, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg, labels) as g:
        g.delete(gone)
        check(g, O.Index(vecs, adj, n, 1, O.L2), queries, labels, RUNS, deleted)
        # released ids take new rows and new labels; delete and release left the table as it was
        g.release(gone)
        fresh = (vecs[rng.integers(0, n, 300)] + 0.2 * rng.normal(size=(300, 32))).astype(np.float32)
        labels[gone] = random_labels(rng, 300, 0.9)
        for i in gone[:100]:
            g.upload_labels(labels[i:i + 1], first=int(i))
        g.upload_labels(labels[:n])
        g.insert(gone, fresh, 16, 30)
        vecs2 = vecs.copy()
        vecs2[gone] = fresh
        check(g, O.Index(vecs2, g.download_graph(), n, 1, O.L2), queries, labels, RUNS)


@pytest.mark.gpu
def test_device_form_empty_batches_and_argument_errors():
    import torch
    rng = np.random.default_rng(2)
    n, nq, k, L = 2000, 100, 10, 50
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, n, 32, 16, 30)
    queries = (vecs[rng.integers(0, n, nq)] + 0.1 * rng.normal(size=(nq, 32))).astype(np.float32)
    labels = random_labels(rng, n + 1, 0.1)
    masks = masks_for(nq, 0, False)
    L_ = dab.lib()
    g = dab.GpuIndex(dab.DType.f32, O.L2, 32, n, 1, maxdeg)
    with g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        launches = dab.launch_count()
        h = g._h
        args = lambda kk, LL, beam, samples, scale: (h, O.ptr(queries), nq, kk, LL, beam, O.ptr(masks), 0, samples, scale, None, None,
                                                      None, None, None)
        for fn in (L_.dab_search_batch_filtered, L_.dab_search_batch_filtered_device):
            assert fn(*args(k, L, 1, 0, 1.0)) == INVALID_ARGUMENT
            assert b"dab_upload_labels" in L_.dab_last_error()
        g.upload_labels(labels)
        for kk, LL, beam, samples, scale, what in ((0, L, 1, 0, 1.0, b"k"), (k, k - 1, 1, 0, 1.0, b"l_value"),
                                                   (k, L, 0, 0, 1.0, b"beam_width"), (k, L, 65, 0, 1.0, b"beam_width"),
                                                   (k, L, 1, 100, 0.99, b"scale"), (k, L, 1, 100, float("nan"), b"scale"),
                                                   (k, 1024, 1, 0, 1.0, b"L + #start"), (k, 512, 1, 100, 2.01, b"floor(L * scale)"),
                                                   (k, 100, 1, 100, float("inf"), b"floor(L * scale)")):
            for fn in (L_.dab_search_batch_filtered, L_.dab_search_batch_filtered_device):
                assert fn(*args(kk, LL, beam, samples, scale)) == INVALID_ARGUMENT, what
                assert what in L_.dab_last_error(), (what, L_.dab_last_error())
        v = np.zeros(4, np.uint64)
        assert L_.dab_upload_labels(h, O.ptr(v), n - 2, 4) == INVALID_ARGUMENT
        assert L_.dab_upload_labels(h, None, 0, 4) == INVALID_ARGUMENT
        # an empty batch is a no-op
        assert L_.dab_search_batch_filtered(h, None, 0, k, L, 1, None, 0, 0, 1.0, None, None, None, None, None) == 0
        assert L_.dab_search_batch_filtered_device(h, None, 0, k, L, 1, None, 0, 0, 1.0, None, None, None, None, None) == 0
        assert dab.launch_count() == launches, "an argument error or an empty batch launched a kernel"
        # the scale is not read without adaptive L
        assert g.search_batch_filtered(queries, masks, k, L, adaptive_l=None)[2].shape == (nq,)
        ids, dists = np.empty((nq, k), np.uint32), np.empty((nq, k), np.float32)
        assert L_.dab_search_batch_filtered(h, O.ptr(queries), nq, k, L, 1, O.ptr(masks), 0, 0, 0.99, O.ptr(ids), O.ptr(dists), None, None,
                                            None) == 0
        want = g.search_batch_filtered(queries, masks, k, L, 2, adaptive_l=(100, 4.0))
        same(want, F.search_batch(O.Index(vecs, adj, n, 1, O.L2), queries, k, L, labels, masks, False, (100, 4.0), beam=2), "host form")
        d_q = torch.from_numpy(queries).cuda()
        d_m = torch.from_numpy(masks.view(np.int64)).cuda()
        bufs = (torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
                *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
        g.search_batch_filtered_device(d_q.data_ptr(), nq, k, L, 2, d_m.data_ptr(), *(b.data_ptr() for b in bufs), adaptive_l=(100, 4.0))
        got = [b.cpu().numpy() for b in bufs]
        same(got, want, "device form")


@pytest.mark.gpu
def test_shared_memory_limit_is_an_argument_error():
    """a list of 1024 with 64 beams of 200-neighbour rows needs more than 200 KB of shared memory per CTA"""
    n, d, md = 100, 32, 200
    vecs = np.zeros((n + 1, d), np.float32)
    adj = np.zeros((n + 1, md + 1), np.uint32)
    L_ = dab.lib()
    queries = np.zeros((4, d), np.float32)
    masks = np.ones(4, np.uint64)
    with gpu_index(vecs, adj, n, 1, O.L2, md, np.ones(n + 1, np.uint64)) as g:
        launches = dab.launch_count()
        for fn in (L_.dab_search_batch_filtered, L_.dab_search_batch_filtered_device):
            assert fn(g._h, O.ptr(queries), 4, 10, 512, 64, O.ptr(masks), 0, 10, 2.0, None, None, None, None, None) == INVALID_ARGUMENT
            assert b"shared memory" in L_.dab_last_error()
        assert dab.launch_count() == launches
        assert g.search_batch_filtered(queries, masks, 10, 512, 8, adaptive_l=(10, 2.0))[2].tolist() == [0] * 4  # a fitting beam runs
