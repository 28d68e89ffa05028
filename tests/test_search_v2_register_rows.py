"""search_kernel_v2's three row paths against the oracle: bit-identical ids, distance bits, result counts, cmps and hops.

f32 rows of 32 / 64 / 96 / 128 elements are read straight into registers when level 1 of the visited set is on
(batches in flight); other rows, and synchronous calls, stage their rows in shared memory, as long as the list fits one
register tile (L + start points <= 256).  Longer lists and float Metric::Cosine read their rows from global memory.
All paths run here, synchronously and in flight, at list sizes from 25 to 1103, beam widths 1 / 2 / 4, several start
points, adjacency rows longer than the 96-word speculative buffer, and with level 1 forced to close early."""

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

FIELDS = ("ids", "dists", "counts", "cmps", "hops")


@pytest.fixture(scope="module")
def dab():
    import diskann_b200
    diskann_b200.lib()
    return diskann_b200


def make_index(rng, metric, n, d, R, L_build, n_start=1, dt=np.float32):
    centers = rng.normal(size=(32, d)).astype(np.float32)
    base = (centers[rng.integers(0, 32, n)] + 0.3 * rng.normal(size=(n, d))).astype(np.float32)
    if metric == O.COSINE_NORMALIZED:
        base /= np.linalg.norm(base, axis=1, keepdims=True)
    if dt == np.int8:
        base = np.clip(np.round(base * 40), -127, 127)
    elif dt == np.uint8:
        base = np.clip(np.round(base * 40 + 128), 0, 255)
    base = base.astype(dt)
    starts = base[rng.choice(n, n_start, replace=False)]
    vecs = np.concatenate([base, starts])
    maxdeg = int(R * 1.3)
    adj = O.build_graph(vecs, n, n_start, metric, R, maxdeg, L_build)
    queries = vecs[rng.integers(0, n, 160)].astype(np.float32) + 0.05 * rng.normal(size=(160, d)).astype(np.float32)
    if dt == np.int8:
        queries = np.clip(np.round(queries), -127, 127)
    elif dt == np.uint8:
        queries = np.clip(np.round(queries), 0, 255)
    return vecs, adj, maxdeg, queries.astype(dt)


def check(dab, vecs, adj, maxdeg, queries, n, n_start, metric, cases):
    oidx = O.Index(vecs, adj, n, n_start, metric)
    with dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        for (L, beam) in cases:
            want = oidx.search_batch(queries, 10, L, beam=beam, threads=4)
            got = g.search_batch(queries, 10, L, beam)
            for a, b, name in zip(got, want, FIELDS):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), ("synchronous", name, L, beam)
            out = g.search_batch_async(1, queries, 10, L, beam)
            g.wait(1)
            for a, b, name in zip(out, want, FIELDS):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), ("in flight", name, L, beam)


LB = [(L, beam) for L in (25, 60, 100, 200, 255) for beam in (1, 2, 4)]


@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("dim", [32, 64, 96, 128, 48, 100])
def test_rows_in_registers_and_staged_match_the_oracle(dab, dim, metric):
    """32 / 64 / 96 / 128: register rows in flight; 48 / 100: staged rows (8 per group at 100-d)."""
    rng = np.random.default_rng(dim * 7 + int(metric))
    n = 2500
    vecs, adj, maxdeg, queries = make_index(rng, metric, n, dim, 16, 30)
    check(dab, vecs, adj, maxdeg, queries, n, 1, metric, LB)


@pytest.mark.parametrize("dim", [128, 100])
def test_several_start_points_and_rows_longer_than_the_adjacency_buffer(dab, dim):
    """three start points (start batch of 3 rows, L + start points up to 256) and max degree 104 > 95."""
    rng = np.random.default_rng(dim + 1)
    n = 3000
    vecs, adj, maxdeg, queries = make_index(rng, O.L2, n, dim, 80, 100, n_start=3)
    assert maxdeg > 95 and (adj[:, 0] > 95).any()
    check(dab, vecs, adj, maxdeg, queries, n, 3, O.L2, [(25, 1), (100, 1), (100, 4), (200, 2), (253, 1)])


@pytest.mark.parametrize("dim", [128, 100])
def test_level1_forced_to_close(dab, monkeypatch, dim):
    """a 512-byte level 1 closes after a few hops, so ids go on to the (tiny) global table, which overflows and
    re-runs queries: still the oracle's answer on both row paths."""
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    rng = np.random.default_rng(dim + 2)
    n = 4000
    vecs, adj, maxdeg, queries = make_index(rng, O.L2, n, dim, 24, 40)
    check(dab, vecs, adj, maxdeg, queries, n, 1, O.L2, [(25, 1), (60, 2), (100, 1)])


@pytest.mark.parametrize("dt,dim", [(np.float16, 64), (np.float16, 96), (np.int8, 128)])
def test_staged_rows_of_other_types(dab, dt, dim):
    """f16 and i8 rows stay on the staged path (32 rows per group at these widths, so beam 4 spans groups)."""
    rng = np.random.default_rng(dim + 3)
    n = 2500
    vecs, adj, maxdeg, queries = make_index(rng, O.L2, n, dim, 16, 30, dt=dt)
    check(dab, vecs, adj, maxdeg, queries, n, 1, O.L2, [(25, 1), (100, 4), (255, 2)])


@pytest.mark.parametrize("n_start", [1, 3])
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.COSINE), (np.float16, O.INNER_PRODUCT), (np.int8, O.L2),
                                       (np.uint8, O.COSINE)])
def test_lists_longer_than_256(dab, dt, metric, n_start):
    """L + start points from 301 to 1103: lists merged tile by tile, up to five tiles of 256 entries."""
    rng = np.random.default_rng(int(metric) * 10 + n_start + np.dtype(dt).itemsize)
    n = 2500
    vecs, adj, maxdeg, queries = make_index(rng, metric, n, 64, 16, 30, n_start=n_start, dt=dt)
    check(dab, vecs, adj, maxdeg, queries, n, n_start, metric, [(L, beam) for L in (300, 700, 1100) for beam in (1, 2)])


def test_rows_too_wide_to_stage(dab):
    """6000-d f32 rows: a stage of eight (192 KB) does not fit beside the rest of the layout, so they are read from
    global memory, as for lists of any length."""
    rng = np.random.default_rng(6000)
    n = 400
    vecs, adj, maxdeg, queries = make_index(rng, O.L2, n, 6000, 8, 20)
    check(dab, vecs, adj, maxdeg, queries, n, 1, O.L2, [(40, 1), (60, 2)])


def test_the_register_path_is_the_one_dispatched(dab):
    """in flight, 128-d f32 launches the register instantiation and 100-d f32 the staged one; synchronous calls stage.
    Float Metric::Cosine and lists longer than 256 launch the instantiation for lists of any length."""
    import torch

    def kernels(g, q, in_flight, L=100):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            if in_flight:
                g.search_batch_async(0, q, 10, L)
                g.wait(0)
            else:
                g.search_batch(q, 10, L)
            torch.cuda.synchronize()
        return {e.key for e in prof.key_averages() if "search_kernel" in e.key}

    rng = np.random.default_rng(4)
    for dim, reg in ((128, True), (100, False)):
        n = 2000
        vecs, adj, maxdeg, queries = make_index(rng, O.L2, n, dim, 16, 30)
        with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, dim, n, 1, maxdeg) as g:
            g.upload_vectors(vecs)
            g.upload_graph(adj)
            flight, sync = kernels(g, queries, True), kernels(g, queries, False)
        assert flight and sync, (flight, sync)
        assert all(k.replace(" ", "").endswith(f"true,{'true' if reg else 'false'}>(dab::SearchParamsV2)") for k in flight), flight
        assert all(k.replace(" ", "").endswith("false,false>(dab::SearchParamsV2)") for k in sync), sync
    for metric, dim, L in ((O.COSINE, 64, 100), (O.L2, 128, 300)):
        n = 2000
        vecs, adj, maxdeg, queries = make_index(rng, metric, n, dim, 16, 30)
        with dab.GpuIndex(dab.DType.f32, metric, dim, n, 1, maxdeg) as g:
            g.upload_vectors(vecs)
            g.upload_graph(adj)
            for in_flight in (True, False):
                launched = kernels(g, queries, in_flight, L)
                assert launched and all("search_kernel_v2<" in k for k in launched), launched
                assert all(k.replace(" ", "").endswith(",0,false,false>(dab::SearchParamsV2)") for k in launched), launched
