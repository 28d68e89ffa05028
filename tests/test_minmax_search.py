"""Graph search over the MinMax store of an index (MinMaxElement<NBITS> as the index's vector representation,
diskann-providers/src/common/minmax_repr.rs:167-336; diskann-garnet's MinMax traversal, provider.rs:1170-1530).

CPU: the oracle's MinMax search (orc_search_batch_minmax) against the exhaustive MinMax scan and, with Rerank, the exact
full-precision scan.  GPU: dab_upload_minmax / dab_minmax_encode_all / dab_minmax_download and dab_search_batch_minmax
bit for bit against the oracle, over every width, metric, row type and transform kind, and the errors of each entry
point."""
import collections
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
from code_rows import garbage_padding
from test_minmax_transforms import oracle_apply

T = dab.Transform
FIVE = ("ids", "dists", "counts", "cmps", "hops")


_MLIB = None


def mm_oracle_lib():
    """oracle/minmax_search.cpp's entry point: liboracle_minmax_search.so (oracle/minmax_search.mk, built by build())."""
    global _MLIB
    if _MLIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_minmax_search.so")
        src = os.path.join(O.ORACLE_DIR, "minmax_search.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "minmax_search.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        L.orc_search_batch_minmax.restype = None
        L.orc_search_batch_minmax.argtypes = [C.POINTER(O.OrcIndex), vp, u64, vp, i, vp, u32, u32, u32, u32, i, i, vp, vp, vp, vp, vp]
        _MLIB = L
    return _MLIB


class MinMaxOracle:
    """The oracle's KNN::search through a MinMax store: the index of `vectors` / `adj` with canonical-front `rows` of
    `nbits` codes (keeps the arrays alive)."""

    def __init__(self, vectors, adj, n_points, n_start, metric, rows, nbits):
        self.index = O.Index(vectors, adj, n_points, n_start, metric)
        self.rows = np.ascontiguousarray(rows, np.uint8)
        assert self.rows.shape[0] == n_points + n_start
        self.nbits = nbits

    def search(self, queries, mm_queries, k, l_search, beam=1, rerank=False, flavour=O.AVX2):
        """`mm_queries`: the queries compressed by the store's quantizer; rerank=True re-scores with `queries`."""
        queries = np.ascontiguousarray(queries)
        mm_queries = np.ascontiguousarray(mm_queries, np.uint8)
        nq = queries.shape[0]
        assert mm_queries.shape == (nq, self.rows.shape[1])
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
        mm_oracle_lib().orc_search_batch_minmax(C.byref(self.index.c), O.ptr(queries), queries.strides[0], O.ptr(self.rows), self.nbits,
                                                O.ptr(mm_queries), nq, k, l_search, beam, int(bool(rerank)), flavour, O.ptr(ids),
                                                O.ptr(dists), O.ptr(counts), O.ptr(cmps), O.ptr(hops))
        return ids, dists, counts, cmps, hops


def make_transform(kind, d):
    """None, PaddingHadamard Natural (wider than d when d is not a power of two), DoubleHadamard Same, and DoubleHadamard
    Override below d (the transform subsamples)."""
    if kind is None:
        return None
    if kind == "padding_natural":
        return T.padding_hadamard(d, "natural", seed=d)
    if kind == "double_same":
        return T.double_hadamard(d, "same", seed=d)
    assert kind == "double_override"
    return T.double_hadamard(d, d * 5 // 8, seed=d)


def compress(vectors, t, nbits, grid_scale=1.0):
    """as_f32, transform_into and MinMaxQuantizer::compress on the CPU: canonical-front rows."""
    f = np.ascontiguousarray(np.asarray(vectors).astype(np.float32))
    if t is not None:
        f = oracle_apply(t, f)
    rows, _, nan = O.minmax_compress(f, nbits, grid_scale)
    assert not nan.any()
    return rows


def clustered(rng, n, d, n_centers=16, spread=0.3):
    centers = rng.normal(size=(n_centers, d)).astype(np.float32)
    return (centers[rng.integers(0, n_centers, n)] + spread * rng.normal(size=(n, d))).astype(np.float32)


def with_medoid(base):
    f = base.astype(np.float32)
    medoid = base[np.argmin(((f - f.mean(0)) ** 2).sum(1))]
    return np.concatenate([base, medoid[None]])


def reachable(adj, start):
    seen, todo = {start}, collections.deque([start])
    while todo:
        u = todo.popleft()
        for v in adj[u, 1:1 + adj[u, 0]]:
            if int(v) not in seen:
                seen.add(int(v))
                todo.append(int(v))
    return len(seen)


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


# ---------------------------------------------------------------- CPU: the oracle's MinMax search

CPU_CASES = [(O.L2, 8, None), (O.INNER_PRODUCT, 4, "double_same"), (O.COSINE, 2, None), (O.COSINE_NORMALIZED, 1, "double_same")]


def small_index(metric, nbits, kind, seed):
    rng = np.random.default_rng(seed)
    n, d = 300, 24
    vecs = with_medoid(clustered(rng, n, d))
    adj = O.build_graph(vecs, n, 1, O.L2, 12, 16, 30)
    assert reachable(adj, n) == n + 1  # connected from the start point
    t = make_transform(kind, d)
    rows = compress(vecs, t, nbits)
    return rng, n, vecs, adj, t, rows


@pytest.mark.parametrize("metric,nbits,kind", CPU_CASES)
def test_oracle_minmax_search_with_the_whole_graph_in_the_list_is_the_exhaustive_scan(metric, nbits, kind):
    """L >= n_total on a connected graph: the MinMax search returns the exhaustive MinMax top-k (ids and distance bits),
    and with Rerank the exact full-precision top-k.  Queries are kept only where the (k+1) best distances are distinct,
    so the cut has no ties."""
    rng, n, vecs, adj, t, rows = small_index(metric, nbits, kind, 100 + nbits)
    k = 10
    cand = clustered(rng, 40, vecs.shape[1])
    qrows = compress(cand, t, nbits)
    keep = []
    for i in range(cand.shape[0]):
        d = O.minmax_distances(metric, nbits, nbits, np.repeat(qrows[i:i + 1], n, 0), rows[:n])
        order = np.argsort(d, kind="stable")
        if len(np.unique(d[order[:k + 1]])) == k + 1:
            keep.append((i, order[:k], d[order[:k]]))
    assert len(keep) >= 8
    sel = np.array([i for i, _, _ in keep[:8]])
    oidx = MinMaxOracle(vecs, adj, n, 1, metric, rows, nbits)
    ids, dists, counts, _, _ = oidx.search(cand[sel], qrows[sel], k, n + 1)
    for q, (_, want_ids, want_d) in enumerate(keep[:8]):
        assert counts[q] == k
        assert np.array_equal(ids[q], want_ids)
        assert np.array_equal(dists[q].view(np.uint32), want_d.astype(np.float32).view(np.uint32))
    ids, dists, counts, _, _ = oidx.search(cand[sel], qrows[sel], k, n + 1, rerank=True)
    gt_ids, gt_d = O.bruteforce_knn(vecs[:n], cand[sel], metric, k, threads=1)
    assert np.array_equal(ids, gt_ids)
    assert np.array_equal(dists.view(np.uint32), gt_d.view(np.uint32))


@pytest.mark.parametrize("metric,nbits,kind", CPU_CASES)
def test_oracle_minmax_search_returns_the_minmax_distance_of_every_row(metric, nbits, kind):
    """At a short list every returned traversal distance is orc_minmax_distance(query row, stored row)."""
    rng, n, vecs, adj, t, rows = small_index(metric, nbits, kind, 200 + nbits)
    queries = clustered(rng, 16, vecs.shape[1])
    qrows = compress(queries, t, nbits)
    oidx = MinMaxOracle(vecs, adj, n, 1, metric, rows, nbits)
    ids, dists, counts, cmps, hops = oidx.search(queries, qrows, 10, 20, beam=2)
    assert (counts == 10).all() and (cmps > 0).all() and (hops > 0).all()
    for q in range(queries.shape[0]):
        want = O.minmax_distances(metric, nbits, nbits, np.repeat(qrows[q:q + 1], 10, 0), rows[ids[q]])
        assert np.array_equal(dists[q].view(np.uint32), want.view(np.uint32))
        assert (np.diff(dists[q]) >= 0).all()


# ---------------------------------------------------------------- GPU: the MinMax store and its traversal

def index_rows(rng, dt, n, d):
    base = clustered(rng, n, d)
    if dt == np.float16:
        base = base.astype(np.float16)
    elif dt == np.int8:
        base = np.clip(np.round(base * 40), -127, 127).astype(np.int8)
    elif dt == np.uint8:
        base = np.clip(np.round(base * 40 + 128), 0, 255).astype(np.uint8)
    return with_medoid(base)


GPU_CASES = [
    (np.float32, O.L2, 128, 8, "double_same"),
    (np.float32, O.INNER_PRODUCT, 100, 4, "padding_natural"),
    (np.float16, O.COSINE, 64, 2, None),
    (np.uint8, O.COSINE_NORMALIZED, 72, 1, "double_override"),
    (np.int8, O.L2, 37, 4, None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tables", ["sized", "overflow"])
@pytest.mark.parametrize("dt,metric,d,nbits,kind", GPU_CASES)
def test_minmax_traversal_search_identical_to_oracle(monkeypatch, dt, metric, d, nbits, kind, tables):
    """dab_minmax_encode_all + dab_minmax_download == the oracle's rows byte for byte; dab_search_batch_minmax ids,
    distance bits, counts, cmps and hops == orc_search_batch_minmax with and without Rerank at (k, L, beam) = (10, 30, 1),
    (5, 64, 2), (10, 150, 1) and a list of 601 entries; also with 256-slot visited tables, whose overflowed queries are
    re-run (the rerank then reads the re-runs' lists).  Host-uploaded rows with garbage padding bits give the same
    searches, and the device-pointer variant matches the host one."""
    if tables == "overflow":
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    rng = np.random.default_rng(d * 10 + nbits)
    n, nq = 2500, 200
    vecs = index_rows(rng, dt, n, d)
    maxdeg = 31
    adj = O.build_graph(vecs, n, 1, O.L2, 24, maxdeg, 40)
    t = make_transform(kind, d)
    out_dim = d if t is None else t.output_dim
    if kind == "padding_natural":
        assert out_dim > d
    if kind == "double_override":
        assert out_dim < d
    rows = compress(vecs, t, nbits)
    queries = vecs[rng.integers(0, n, nq)].copy()
    qrows = compress(queries, t, nbits)
    oidx = MinMaxOracle(vecs, adj, n, 1, metric, rows, nbits)
    with dab.GpuIndex(O.dtype_code(vecs), metric, d, n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.upload_minmax(nbits, 1.0, t)
        with pytest.raises(dab.DabError) as e:
            g.search_batch_minmax(queries[:2], 5, 10)
        assert e.value.code == 5
        g.minmax_encode_all()
        assert np.array_equal(g.download_minmax(), rows)
        for (k, Ls, beam) in [(10, 30, 1), (5, 64, 2), (10, 150, 1), (10, 600, 1)]:
            for rerank in (False, True):
                got = g.search_batch_minmax(queries, k, Ls, beam, rerank=rerank)
                want = oidx.search(queries, qrows, k, Ls, beam=beam, rerank=rerank)
                same(got, want, (k, Ls, beam, rerank))
        # rows handed over by the host, with garbage in the padding bits of the last code byte
        if t is not None:
            t = make_transform(kind, d)  # the index holds its own copy: a fresh object, then dropped
        g.upload_minmax(nbits, 1.0, t, rows=garbage_padding(rows, out_dim, nbits))
        del t
        assert np.array_equal(g.download_minmax(), rows)
        for rerank in (False, True):
            got = g.search_batch_minmax(queries, 10, 50, 1, rerank=rerank)
            same(got, oidx.search(queries, qrows, 10, 50, rerank=rerank), ("host rows", rerank))
        # the device-pointer variant
        import torch
        d_q = torch.from_numpy(queries.view(np.uint8).copy()).cuda()
        d_ids = torch.empty((nq, 10), dtype=torch.int32, device="cuda")
        d_d = torch.empty((nq, 10), dtype=torch.float32, device="cuda")
        d_c, d_cm, d_h = (torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3))
        for rerank in (False, True):
            g.search_batch_minmax_device(d_q.data_ptr(), nq, 10, 64, 2, d_ids.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), d_cm.data_ptr(),
                                         d_h.data_ptr(), rerank=rerank)
            torch.cuda.synchronize()
            got = [x.cpu().numpy() for x in (d_ids, d_d, d_c, d_cm, d_h)]
            same(got, g.search_batch_minmax(queries, 10, 64, 2, rerank=rerank), ("device", rerank))


@pytest.mark.gpu
def test_minmax_store_and_search_errors():
    """Each failure has its own message: search before rows, a transform of the wrong input dim, a bad width or grid
    scale, a row whose stored dim differs, a NaN query, a NaN row at encode, and L + #start > 1024."""
    rng = np.random.default_rng(5)
    n, d = 500, 32
    vecs = clustered(rng, n + 1, d)
    adj = np.zeros((n + 1, 9), np.uint32)
    adj[:, 0] = 8
    adj[:, 1:] = rng.integers(0, n + 1, (n + 1, 8))
    messages = []

    def fails(code, fn, *args, **kw):
        with pytest.raises(dab.DabError) as e:
            fn(*args, **kw)
        assert e.value.code == code, str(e.value)
        messages.append(str(e.value).split(": ", 1)[1])
        return str(e.value)

    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, 8) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        assert "dab_upload_minmax has not been called" in fails(5, g.minmax_encode_all)
        g.upload_minmax(8)
        assert "no MinMax rows" in fails(5, g.search_batch_minmax, vecs[:2], 5, 10)
        assert "the transform takes vectors of 33 values" in fails(1, g.upload_minmax, 8, 1.0, T.double_hadamard(d + 1, "same"))
        assert "nbits must be 1, 2, 4 or 8" in fails(1, g.upload_minmax, 3)
        assert "grid_scale must be positive" in fails(1, g.upload_minmax, 8, 0.0)
        rows = compress(vecs, None, 8)
        bad = rows.copy()
        bad[7, :4] = np.frombuffer(np.uint32(d - 1).tobytes(), np.uint8)
        assert "row 7 stores dim 31" in fails(1, g.upload_minmax, 8, 1.0, None, rows=bad)
        g.upload_minmax(8, 1.0, None, rows=rows)
        q = vecs[:5].copy()
        q[3, 4] = np.nan
        assert "query 3 contains NaN" in fails(1, g.search_batch_minmax, q, 5, 10)
        assert "L + #start must be <= 1024" in fails(1, g.search_batch_minmax, vecs[:2], 5, 1024)
        nan_rows = vecs.copy()
        nan_rows[7, 0] = np.nan
        g.upload_vectors(nan_rows)
        assert "row 7 contains NaN" in fails(1, g.minmax_encode_all)
        assert "no rows" in fails(5, g.download_minmax)
    assert len(set(messages)) == len(messages)
