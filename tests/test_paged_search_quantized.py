"""Paged search over the PQ, SQ and MinMax stores: dab_paged_search_begin_{pq,sq,minmax} with the shared _next / _end.

The reference's paged search is generic over the search strategy (index.rs:2075-2155), and its own grid test runs every
paged query with the quantized strategy too (diskann_async.rs:544-580).  The session is the full-precision one; only the
traversal distances change — the quantized accessor's — and pages return them (no post-processing, paged.rs:122).

CPU: the paged restatement of test_paged_search.py over each store's exhaustive quantized distances, which the oracle's
one-shot searches confirm; the reference's quantized grid check on its three lattices; and, per store, paging to
exhaustion returns every reachable node once, sorted by quantized distance.
GPU: the device equals the restatement bit for bit after every page (ids, distance bits, counts, cumulative cmps and
hops) for every PQ table kind and chunk layout, every SQ and MinMax width and metric, every MinMax transform kind and
every row type, on graphs with many start points, malformed rows and exact ties, with visited tables that overflow in
mid-session, with other work interleaved between pages; a session fails cleanly once its own store is written; and
every begin-time error of the synchronous calls is reported."""
import ctypes as C
import functools

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
from test_gpu_parity import sq_quantizer, trained_pq
from test_minmax_search import MinMaxOracle, compress, make_transform
from test_oracle_golden import grid as lattice
from test_paged_search import PyPaged, bfs, built, padded
from test_traversal_edges import grid as tie_grid, malformed_case

# ---------------------------------------------------------------- the stores' exhaustive distances (the oracle's)


def as_f32(q):
    return np.ascontiguousarray(np.asarray(q).astype(np.float32))  # T: Into<f32>; f16 widened


class PQStore:
    """a PQ table (pivots, offsets) and the codes of every row; QueryComputer::new picks the distance by metric"""

    def __init__(self, piv, off, codes, metric):
        self.piv, self.off = np.ascontiguousarray(piv, np.float32), np.ascontiguousarray(off, np.uint64)
        self.codes, self.metric = np.ascontiguousarray(codes, np.uint8), metric

    def distances(self, q):
        out = np.empty(self.codes.shape[0], np.float32)
        qf = as_f32(q)
        O.lib().orc_pq_query_distances(O.ptr(self.piv), self.piv.shape[0], self.piv.shape[1], O.ptr(self.off), self.codes.shape[1],
                                       self.metric, O.ptr(qf), O.ptr(self.codes), self.codes.shape[0], O.ptr(out))
        return out

    def upload(self, g):
        g.upload_pq(self.piv, self.off, self.codes)

    def oracle(self, case):
        vecs, adj, n, n_start, metric = case[:5]
        return O.Index(vecs, adj, n, n_start, metric, pq=(self.piv, self.off, self.codes))


class SQStore:
    """SQStore<NBITS>: the quantizer and the canonical-front rows (f32 compensation | dense codes) of every row"""

    def __init__(self, rows, nbits, quantizer, metric):
        self.rows, self.nbits, self.quantizer, self.metric = np.ascontiguousarray(rows, np.uint8), nbits, quantizer, metric
        shift, scale = quantizer[0], quantizer[1]
        dim = shift.shape[0]
        bits = np.unpackbits(self.rows[:, 4:], axis=1, bitorder="little")[:, :dim * nbits].reshape(-1, dim, nbits)
        self.row_codes = np.ascontiguousarray((bits * (1 << np.arange(nbits))).sum(2).astype(np.uint8))
        self.row_comp = self.rows[:, :4].copy().view(np.float32)[:, 0]
        self.ss = float(np.float32(scale) * np.float32(scale))

    def distances(self, q):
        """SQStore::query_computer (as_f32, the InnerProduct rescale to the mean norm, compress), then the compensated
        distance to every row"""
        shift, scale, ssn, mean_norm = self.quantizer
        qf = as_f32(q)
        if self.metric == O.INNER_PRODUCT and mean_norm != 0.0:
            norm = np.float32(np.sqrt(np.float32(-O.distance(qf, qf, O.INNER_PRODUCT, O.AVX2))))
            if norm != 0:
                qf = (qf * np.float32(np.float32(mean_norm) / norm)).astype(np.float32)
        L = O.lib()
        codes = np.zeros(qf.shape[0], np.uint8)
        comp = L.orc_sq_compress(O.ptr(shift), scale, qf.shape[0], self.nbits, O.ptr(qf), O.ptr(codes), None)
        return np.array([L.orc_sq_distance(self.metric, self.nbits, self.ss, ssn, O.ptr(codes), comp, O.ptr(self.row_codes[i]),
                                           float(self.row_comp[i]), qf.shape[0]) for i in range(self.rows.shape[0])], np.float32)

    def upload(self, g):
        g.upload_sq(self.nbits, *self.quantizer, rows=self.rows)

    def oracle(self, case):
        vecs, adj, n, n_start, metric = case[:5]
        return O.Index(vecs, adj, n, n_start, metric, sq=(self.rows, self.nbits, *self.quantizer))


class MMStore:
    """MinMaxElement<NBITS> rows behind a transform; the query is compressed by the same quantizer"""

    def __init__(self, vecs, nbits, kind, metric):
        self.nbits, self.kind, self.metric = nbits, kind, metric
        self.t = make_transform(kind, vecs.shape[1])
        self.rows = compress(vecs, self.t, nbits)

    def query_row(self, q):
        return compress(np.asarray(q)[None], self.t, self.nbits)[0]

    def distances(self, q):
        qr = self.query_row(q)
        return O.minmax_distances(self.metric, self.nbits, self.nbits, np.broadcast_to(qr, self.rows.shape), self.rows)

    def upload(self, g):
        g.upload_minmax(self.nbits, 1.0, self.t, rows=self.rows)


def pq_store(case, chunks, seed=11):
    vecs, n, metric = case[0], case[2], case[4]
    f = as_f32(vecs)
    piv, off = trained_pq(np.random.default_rng(seed), f[:n], chunks)
    codes = np.zeros((f.shape[0], chunks), np.uint8)
    for i in range(f.shape[0]):
        assert O.lib().orc_pq_encode(O.ptr(piv), 256, f.shape[1], O.ptr(off), chunks, O.ptr(f[i]), O.ptr(codes[i])) == 0
    return PQStore(piv, off, codes, metric)


def sq_store(case, nbits):
    vecs, metric = case[0], case[4]
    f = as_f32(vecs)
    quantizer = sq_quantizer(f, metric)
    return SQStore(O.sq_encode_rows(f, quantizer[0], quantizer[1], nbits), nbits, quantizer, metric)


# ---------------------------------------------------------------- the paged session over a store, restated

class QPaged(PyPaged):
    """PyPaged with the traversal distances of a quantized store: `table` holds the query's distance to every row"""

    def __init__(self, table, adj, n_points, n_start, L):
        self.adj, self.n_points, self.total, self.L = adj, n_points, n_points + n_start, L
        self.max_degree = adj.shape[1] - 1
        self.dist = lambda ids: table[ids]
        self.cap = L + n_start
        self.ids, self.ds, self.done, self.cursor = [], [], [], 0
        self.starts = set(range(n_points, self.total))
        self.visited = set(self.starts)
        self.cmps = self.hops = 0
        fresh = []
        for s in range(n_points, self.total):
            fresh += self._expand(s)
        self._insert(fresh)


def paged_to_exhaustion(store, case, q, L, ks):
    vecs, adj, n, n_start = case[:4]
    table = store.distances(q)
    s = QPaged(table, adj, n, n_start, L)
    pages, j = [], 0
    while True:
        page = s.next_page(ks[j % len(ks)])
        j += 1
        if not page:
            return table, pages, s
        pages.append(page)


# ---------------------------------------------------------------- CPU

@functools.lru_cache(maxsize=None)
def small_case(dt=np.float32, metric=O.L2):
    return built(400, 16, dt, metric, 4, seed=17)


CPU_STORES = [("pq", None), ("sq", 8), ("sq", 4), ("mm", 8), ("mm", 4)]


def make_store(kind, nbits, case, chunks=4, transform=None):
    if kind == "pq":
        return pq_store(case, chunks)
    if kind == "sq":
        return sq_store(case, nbits)
    return MMStore(case[0], nbits, transform, case[4])


@pytest.mark.parametrize("kind,nbits", CPU_STORES)
def test_store_distances_are_the_oracles_search_distances(kind, nbits):
    """the restated query side of each store (PQ table, SQ rescale and compression, MinMax compression) gives the
    distances the oracle's one-shot quantized search returns for the same ids"""
    case = small_case(np.float32, O.INNER_PRODUCT if kind == "sq" else O.L2)
    store = make_store(kind, nbits, case)
    qs = case[5]
    if kind == "mm":
        oracle = MinMaxOracle(case[0], case[1], case[2], case[3], case[4], store.rows, nbits)
        ids, dists, counts = oracle.search(qs, compress(qs, store.t, nbits), 10, 60)[:3]
    else:
        ids, dists, counts = store.oracle(case).search_batch(qs, 10, 60)[:3]
    for qi in range(qs.shape[0]):
        table = store.distances(qs[qi])
        got = table[ids[qi][:counts[qi]].astype(np.int64)]
        assert counts[qi] > 0 and np.array_equal(got.view(np.uint32), dists[qi][:counts[qi]].view(np.uint32)), qi


@pytest.mark.parametrize("kind,nbits", CPU_STORES)
def test_paged_to_exhaustion_over_each_store(kind, nbits):
    case = small_case()
    store = make_store(kind, nbits, case)
    reach = bfs(case[1], case[2], case[3])
    for q in case[5]:
        table, pages, s = paged_to_exhaustion(store, case, q, 20, (10, 1, 7, 20))
        seen = []
        for page in pages:
            ds = [d for _, d in page]
            assert all(a <= b for a, b in zip(ds, ds[1:]))
            for i, d in page:
                assert np.float32(d).view(np.uint32) == table[i].view(np.uint32)
            seen += [i for i, _ in page]
        assert len(seen) == len(set(seen)) and set(seen) == reach
        assert s.next_page(1) == []


def grid_pq(dims, size):
    """the reference's quantized grid index (diskann_async.rs:588-647): min(2, dim) chunks whose pivots are exactly the
    distinct chunk coordinates, so that every code reconstructs its row"""
    data, adj, n = lattice(dims, size)
    chunks = min(2, dims)
    off = O.pq_offsets(dims, chunks)
    uniq, codes = [], np.zeros((n + 1, chunks), np.uint8)
    for c in range(chunks):
        u, inv = np.unique(data[:, int(off[c]):int(off[c + 1])], axis=0, return_inverse=True)
        uniq.append(u)
        codes[:, c] = inv.reshape(-1)
    centers = max(len(u) for u in uniq)
    piv = np.zeros((centers, dims), np.float32)
    for c, u in enumerate(uniq):
        piv[:, int(off[c]):int(off[c + 1])] = u[np.minimum(np.arange(centers), len(u) - 1)]
    return data, adj, n, PQStore(piv, off, codes, O.L2)


def groundtruth(corpus, q):
    """search_utils.rs groundtruth: nearest last"""
    d = ((corpus.astype(np.float64) - q) ** 2).sum(1).astype(np.float32)
    order = sorted(range(len(d)), key=lambda i: d[i], reverse=True)
    return [(i, float(d[i])) for i in order]


def check_grid_pages(pages, gt):
    """test_paged_search (diskann_async.rs:374-425) with is_match (search_utils.rs:38-57): every result matches the
    next ground-truth entries within 0.01, until all of them are seen"""
    gt, seen, n = list(gt), 0, len(gt)
    for page in pages:
        for i, d in page:
            for j in range(len(gt) - 1, -1, -1):
                assert abs(gt[j][1] - d) <= 0.01, (i, d, gt[-10:])
                if gt[j][0] == i:
                    del gt[j]
                    break
            else:
                raise AssertionError(f"{i} not in the ground truth")
            seen += 1
            if seen == n:
                return
    raise AssertionError(f"paging ended after {seen} of {n} results")


GRIDS = [(1, 100), (3, 7), (4, 5)]


@pytest.mark.parametrize("dims,size", GRIDS)
def test_reference_quantized_grid_check(dims, size):
    data, adj, n, store = grid_pq(dims, size)
    case = (data, adj, n, 1, O.L2)
    for q in (np.zeros(dims, np.float32), data[n]):
        table, pages, _ = paged_to_exhaustion(store, case, q, 10, (dims + 1,))
        assert n not in {i for p in pages for i, _ in p}  # the start point is never returned
        check_grid_pages(pages, groundtruth(data[:n], q))


# ---------------------------------------------------------------- GPU

def gpu_index(case, store, vectors=True):
    vecs, adj, n, n_start, metric = case[:5]
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, adj.shape[1] - 1)
    if vectors:
        g.upload_vectors(vecs)
    g.upload_graph(adj)
    store.upload(g)
    return g


def begin(g, store, queries, L):
    kind = {PQStore: "pq", SQStore: "sq", MMStore: "minmax"}[type(store)]
    return getattr(g, f"paged_search_{kind}")(queries, L)


def device_pages(g, store, queries, L, ks, until_empty=False, max_pages=None):
    out = []
    with begin(g, store, queries, L) as s:
        j = 0
        while True:
            k = ks[j % len(ks)]
            j += 1
            r = s.next_page(k)
            out.append((k,) + r)
            if (until_empty and not r[2].any()) or (not until_empty and j == len(ks)) or (max_pages and j >= max_pages):
                break
    return out


def check_against_restatement(case, store, got, L, sample):
    vecs, adj, n, n_start, metric, qs = case[:6]
    for qi in sample:
        s = QPaged(store.distances(qs[qi]), adj, n, n_start, L)
        for k, ids, dists, counts, cmps, hops in got:
            page = s.next_page(k)
            wi, wd = padded(page, k)
            assert np.array_equal(ids[qi], wi), (qi, k)
            assert np.array_equal(dists[qi].view(np.uint32), wd.view(np.uint32)), (qi, k)
            assert (int(counts[qi]), int(cmps[qi]), int(hops[qi])) == (len(page), s.cmps, s.hops), (qi, k)


def same_pages(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))


NQ = 9000  # more queries than resident warps: the persistent grid takes several rounds
KS = (10, 1, 37, 40, 10)
SAMPLE = range(0, NQ, 1000)


@functools.lru_cache(maxsize=None)
def gpu_case(dt, metric, d=64):
    return built(2500, d, dt, metric, NQ, seed=23 + d)


def run_and_check(case, store, L=40, ks=KS, sample=SAMPLE):
    with gpu_index(case, store) as g:
        got = device_pages(g, store, case[5], L, ks)
    check_against_restatement(case, store, got, L, sample)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.int8, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.uint8, O.COSINE_NORMALIZED)])
@pytest.mark.parametrize("chunks", [16, 8, 7])  # chunks of 4, of 8, of 9 and 10
def test_pq_pages_equal_the_restatement(dt, metric, chunks):
    case = gpu_case(dt, metric)
    run_and_check(case, pq_store(case, chunks))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_sq_pages_equal_the_restatement(nbits, metric):
    dt = {8: np.float32, 4: np.float16, 2: np.int8, 1: np.uint8}[nbits]
    case = gpu_case(dt, metric)
    run_and_check(case, sq_store(case, nbits))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_minmax_pages_equal_the_restatement(nbits, metric):
    dt = {8: np.float32, 4: np.float16, 2: np.uint8, 1: np.int8}[nbits]
    case = gpu_case(dt, metric, d=48)  # 48: PaddingHadamard pads to 64
    for kind in (None, "padding_natural", "double_same"):
        run_and_check(case, MMStore(case[0], nbits, kind, metric), sample=range(0, NQ, 3000))


def edge_stores(case):
    return [pq_store(case, 2), sq_store(case, 8), MMStore(case[0], 8, None, case[4])]


def as_tuple(c):
    return (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [1, 7, 300])
def test_many_start_points(n_start):
    case = as_tuple(tie_grid(1500, 6, n_start, 64, seed=n_start))
    for store in edge_stores(case):
        run_and_check(case, store, L=60, ks=(10, 1, 37, 60, 7), sample=range(0, 64, 8))


@pytest.mark.gpu
def test_malformed_rows():
    case = as_tuple(malformed_case(1200, 8, 3, 20, 48, seed=5))
    for store in edge_stores(case):
        with gpu_index(case, store) as g:
            got = device_pages(g, store, case[5], 30, (10, 1, 30, 5), until_empty=True, max_pages=60)
        check_against_restatement(case, store, got, 30, range(0, 48, 8))


@pytest.mark.gpu
def test_exact_ties():
    case = as_tuple(tie_grid(1200, 8, 3, 48, seed=3))
    for store in edge_stores(case):
        with gpu_index(case, store) as g:
            got = device_pages(g, store, case[5], 30, (10, 1, 30), until_empty=True, max_pages=40)
        check_against_restatement(case, store, got, 30, range(0, 48, 6))


@pytest.mark.gpu
def test_visited_overflow_in_the_middle_of_a_session(monkeypatch):
    case = built(2000, 16, np.float32, O.L2, 500, seed=9)
    L, ks = 50, (10, 1, 37, 50, 50, 50)
    for store in (pq_store(case, 4), sq_store(case, 4), MMStore(case[0], 8, "double_same", O.L2)):
        monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
        with gpu_index(case, store) as g:
            want = device_pages(g, store, case[5], L, ks)
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")  # 256-slot tables: every query overflows, page after page
        with gpu_index(case, store) as g:
            got = device_pages(g, store, case[5], L, ks)
        same_pages(got, want)
        check_against_restatement(case, store, got, L, range(0, 500, 100))


@pytest.mark.gpu
def test_interleaved_work_between_pages():
    """between two pages: a synchronous search on the same store, a quantized batch in flight on a slot, a page of a
    full-precision session; the quantized session's pages equal an uninterrupted session's"""
    case = built(1500, 32, np.float32, O.L2, 300, seed=13)
    qs, L, ks = case[5], 30, (10, 5, 30, 10)
    stores = [("pq", pq_store(case, 8)), ("sq", sq_store(case, 8)), ("minmax", MMStore(case[0], 4, "double_same", O.L2))]
    with dab.GpuIndex(dab.DType.f32, O.L2, 32, case[2], 1, case[1].shape[1] - 1) as g:
        g.upload_vectors(case[0])
        g.upload_graph(case[1])
        for _, store in stores:
            store.upload(g)
        for kind, store in stores:
            want = device_pages(g, store, qs, L, ks)
            sync = getattr(g, f"search_batch_{kind}")
            fp = g.paged_search(qs[:50], 20)
            got = []
            with begin(g, store, qs, L) as s:
                for k in ks:
                    got.append((k,) + s.next_page(k))
                    sync(qs[100:], 10, 60)
                    getattr(g, f"search_batch_{kind}_async")(1, qs[:200], 10, 50)
                    g.wait(1)
                    fp.next_page(5)
            fp.close()
            same_pages(got, want)


@pytest.mark.gpu
def test_invalidation_by_store_writes_and_destroy():
    case = built(1000, 16, np.float32, O.L2, 64, seed=21)
    qs = case[5]
    pq, sq, mm = pq_store(case, 4), sq_store(case, 8), MMStore(case[0], 8, None, O.L2)

    def fails_changed(s):
        with pytest.raises(dab.DabError) as e:
            s.next_page(5)
        assert e.value.code == 1 and "store was written" in str(e.value), str(e.value)

    with gpu_index(case, pq) as g:
        sq.upload(g)
        mm.upload(g)
        writes = {"pq": [lambda: pq.upload(g), g.pq_encode_all],
                  "sq": [lambda: sq.upload(g), g.sq_encode_all],
                  "minmax": [lambda: mm.upload(g), g.minmax_encode_all]}
        stores = {"pq": pq, "sq": sq, "minmax": mm}
        for kind, store in stores.items():
            for write in writes[kind]:
                s = begin(g, store, qs, 20)
                assert s.next_page(5)[2].all()
                # writes to the other stores leave it valid
                for other, ws in writes.items():
                    if other != kind:
                        ws[0]()
                assert s.next_page(5)[2].all()
                write()
                fails_changed(s)
                s.close()
        # a full-precision session survives every store write
        fp = g.paged_search(qs, 20)
        fp.next_page(5)
        for ws in writes.values():
            for w in ws:
                w()
        assert fp.next_page(5)[2].all()
        fp.close()
        open_sessions = [begin(g, store, qs, 20) for store in stores.values()]
        for s in open_sessions:
            s.next_page(3)
        g.upload_graph(case[1])  # the index changed: every session fails with the full-precision rule
        for s in open_sessions:
            with pytest.raises(dab.DabError) as e:
                s.next_page(5)
            assert e.value.code == 1 and "index changed" in str(e.value)
        still_open = [begin(g, store, qs, 20) for store in stores.values()]
    # still open when the index closed: dab_destroy released them
    for s in still_open:
        with pytest.raises(dab.DabError):
            s.next_page(5)


@pytest.mark.gpu
def test_begin_time_errors():
    case = built(600, 16, np.float32, O.L2, 16, seed=31)
    qs = case[5]
    lib = dab.lib()

    def fails(code, fn, *args):
        with pytest.raises(dab.DabError) as e:
            fn(*args)
        assert e.value.code == code, str(e.value)
        return str(e.value)

    with dab.GpuIndex(dab.DType.f32, O.L2, 16, case[2], 1, case[1].shape[1] - 1) as g:
        g.upload_graph(case[1])
        # stores never uploaded: the synchronous calls' "has not been called"
        assert "dab_upload_pq has not been called" in fails(5, g.paged_search_pq, qs, 20)
        assert "dab_upload_sq has not been called" in fails(5, g.paged_search_sq, qs, 20)
        assert "dab_upload_minmax has not been called" in fails(5, g.paged_search_minmax, qs, 20)
        # set up without rows
        pq = pq_store(case, 4)
        g.upload_pq(pq.piv, pq.off)
        assert "no PQ codes" in fails(5, g.paged_search_pq, qs, 20)
        sq = sq_store(case, 8)
        g.upload_sq(8, *sq.quantizer)
        assert "no scalar-quantized rows" in fails(5, g.paged_search_sq, qs, 20)
        g.upload_minmax(8, 1.0, None)
        assert "no MinMax rows" in fails(5, g.paged_search_minmax, qs, 20)
        pq.upload(g)
        sq.upload(g)
        mm = MMStore(case[0], 8, "double_same", O.L2)
        mm.upload(g)
        for fn in (g.paged_search_pq, g.paged_search_sq, g.paged_search_minmax):
            # L + #start > 1024
            assert "> 1024" in fails(1, fn, qs, 1024)
            # k outside [1, L]
            with fn(qs, 20) as s:
                for k in (0, 21):
                    fails(1, s.next_page, k)
                assert s.next_page(20)[2].all()
        # a MinMax query holding a NaN fails begin, naming it; nothing is left open
        bad = qs.copy()
        bad[3, 4] = np.nan
        msg = fails(1, g.paged_search_minmax, bad, 20)
        assert "query 3 contains NaN after the transform (InputContainsNaN)" in msg
        assert not any(s._h.value for s in g._paged)
        for name in ("dab_paged_search_begin_pq", "dab_paged_search_begin_sq", "dab_paged_search_begin_minmax"):
            h = C.c_void_p()
            assert getattr(lib, name)(g._h, None, 5, 20, C.byref(h)) == 1 and not h.value
            assert b"NULL argument" in lib.dab_last_error()
    with dab.GpuIndex(dab.DType.f32, O.COSINE, 16, case[2], 1, case[1].shape[1] - 1) as g:
        g.upload_graph(case[1])
        sq.upload(g)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(1, g.paged_search_sq, qs, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("dims,size", GRIDS)
def test_reference_quantized_grid_check_on_the_device(dims, size):
    data, adj, n, store = grid_pq(dims, size)
    case = (data, adj, n, 1, O.L2, np.stack([np.zeros(dims, np.float32), data[n]]))
    with gpu_index(case, store) as g:
        got = device_pages(g, store, case[5], 10, (dims + 1,), until_empty=True, max_pages=1000)
    assert not got[-1][3].any()
    check_against_restatement(case, store, got, 10, range(2))
    for qi in range(2):
        pages = [[(int(i), float(d)) for i, d in zip(p[1][qi][:p[3][qi]], p[2][qi][:p[3][qi]])] for p in got]
        assert n not in {i for p in pages for i, _ in p}
        check_grid_pages(pages, groundtruth(data[:n], case[5][qi]))
