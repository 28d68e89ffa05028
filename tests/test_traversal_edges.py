"""Every graph traversal on graphs that no build makes: many start points, malformed adjacency rows, disconnected
graphs, exact ties at long lists and non-finite rows.

The library accepts any adjacency whose degrees fit max_degree: ids out of bounds (also ids >= 2^K that share the
16-bit visited tag of a real node, and UINT32_MAX), repeated ids, self-loops, edges into start points and empty rows.
The reference defines what each returns (every neighbour enters the visited set before the bounds check, the queue
drops NaN distances, start points are skipped in the output), and every kernel must return it bit for bit: ids,
distance bits, counts, cmps and hops, on every path a search can take.

CPU: a Python restatement of the reference's search_internal, queue and post-process pins the oracle on these graphs,
and a model of the quotient tags shows why ids >= 2^K must stay out of a tag table.  GPU: each case runs on
search_kernel_v3, search_kernel_v2 (global table, level 1 in flight, rows from global memory), the PQ kernels (pivots
in shared memory and the global table), SQ 8 / 4 bits and MinMax 8 bits with and without rerank, the overflow re-runs,
the synchronous device-pointer calls, and the device build with several start points."""
import functools

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
from test_gpu_parity import sq_quantizer, trained_pq
from test_minmax_search import MinMaxOracle, compress
from test_tag16_model import tag_map

FIVE = ("ids", "dists", "counts", "cmps", "hops")
EMPTY = 0xFFFFFFFF


def same(got, want, what):
    for a, b, name in zip(got, want, FIVE):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def k_bits(n_total):
    """K of the tag tables: the bits of the largest id, at least 8 (search_kernel_v2 / v3 host side)"""
    K = 8
    while (1 << K) < n_total:
        K += 1
    return K


# ---------------------------------------------------------------- the reference's search, restated

def py_search(vecs, adj, n_points, n_start, metric, query, k, L, beam=1, trace=None):
    """search_internal (graph/index.rs), NeighborPriorityQueue (neighbor/queue.rs) and the post-process that skips start
    points (inmem/provider.rs), with distances from the oracle.  `trace` (a dict) counts the edges the search met."""
    total = n_points + n_start
    q = np.ascontiguousarray(query.astype(np.float32) if vecs.dtype == np.float16 else query)  # f16 queries are widened
    dist = lambda ids: O.distance_rows(q, vecs[ids], metric, O.AVX2)
    cap, ids, ds, done, cursor = L + n_start, [], [], [], 0
    kmask = (1 << k_bits(total)) - 1
    t = trace if trace is not None else {}
    for key in ("nan", "oob", "repeat", "alias", "alias_then_scored"):
        t.setdefault(key, 0)
    aliased = set()

    def insert(i, d):
        nonlocal cursor
        if np.isnan(d):
            t["nan"] += 1
            return
        if len(ids) == cap and ds[-1] < d:  # full: rejected
            return
        at = next((j for j, x in enumerate(ds) if x >= d), len(ds))  # lower bound
        if len(ids) == cap:
            del ids[-1], ds[-1], done[-1]
        ids.insert(at, i), ds.insert(at, d), done.insert(at, False)
        cursor = min(cursor, at)

    visited = set(range(n_points, total))
    for i, d in zip(range(n_points, total), dist(np.arange(n_points, total))):
        insert(i, d)
    cmps, hops = n_start, 0
    while cursor < min(cap, len(ids)):
        nodes = []
        while len(nodes) < beam and cursor < min(cap, len(ids)):
            done[cursor] = True
            nodes.append(ids[cursor])
            cursor += 1
            while cursor < len(ids) and done[cursor]:
                cursor += 1
        fresh = []
        for u in nodes:
            for v in adj[u, 1:1 + adj[u, 0]].tolist():
                if v in visited:  # visited insert first ...
                    t["repeat"] += 1
                    continue
                visited.add(v)
                if v >= total:  # ... then is_in_bounds
                    t["oob"] += 1
                    if v > kmask and (v & kmask) < total and (v & kmask) not in visited:
                        aliased.add(v & kmask)
                        t["alias"] += 1
                    continue
                if v in aliased:
                    t["alias_then_scored"] += 1
                fresh.append(v)
        for i, d in zip(fresh, dist(np.array(fresh, np.int64)) if fresh else []):
            insert(i, d)
        cmps += len(fresh)
        hops += len(nodes)
    out = [(i, d) for i, d in zip(ids, ds) if i < n_points][:k]
    got_ids = np.full(k, EMPTY, np.uint32)
    got_d = np.full(k, np.inf, np.float32)
    got_ids[:len(out)] = [i for i, _ in out]
    got_d[:len(out)] = [d for _, d in out]
    t["starts_in_list"] = t.get("starts_in_list", 0) + sum(i >= n_points for i in ids)
    return got_ids, got_d, len(out), cmps, hops


def py_batch(case, k, L, beam, nq=None, trace=None):
    qs = case.queries[:nq]
    rows = [py_search(case.vecs, case.adj, case.n, case.n_start, case.metric, q, k, L, beam, trace) for q in qs]
    return tuple(np.array([r[j] for r in rows]).astype(dt)
                 for j, dt in enumerate((np.uint32, np.float32, np.uint32, np.uint32, np.uint32)))


# ---------------------------------------------------------------- the cases

class Case:
    def __init__(self, vecs, adj, n, n_start, metric, queries):
        self.vecs, self.adj, self.n, self.n_start, self.metric = vecs, np.ascontiguousarray(adj, np.uint32), n, n_start, metric
        self.queries = np.ascontiguousarray(queries)
        self.max_degree = self.adj.shape[1] - 1
        assert self.adj[:, 0].max() <= self.max_degree
        self.oracle = O.Index(vecs, self.adj, n, n_start, metric)

    @property
    def total(self):
        return self.n + self.n_start

    def want(self, k, L, beam):
        return self.oracle.search_batch(self.queries, k, L, beam=beam, threads=4)


def clustered(rng, n, d, n_centers=16, spread=0.3):
    centers = rng.normal(size=(n_centers, d)).astype(np.float32)
    return (centers[rng.integers(0, n_centers, n)] + spread * rng.normal(size=(n, d))).astype(np.float32)


COPIES = (0, 31, 64)  # start rows that are exact copies of base rows, in three groups of 32


def start_rows(rng, base, n_start, near):
    """start rows close to `near`, so that the start points fill short lists, except those at COPIES: exact copies of
    base rows (a start point and a real point tie)"""
    s = near[rng.integers(0, near.shape[0], n_start)] + np.float32(0.02) * rng.normal(size=(n_start, base.shape[1])).astype(np.float32)
    copies = [c for c in COPIES if c < n_start]
    s[copies] = base[rng.integers(0, base.shape[0], len(copies))]
    return s.astype(base.dtype)


def many_starts(n, d, n_start, nq, seed, R=16):
    rng = np.random.default_rng(seed)
    base = clustered(rng, n, d)
    near = base[:1]
    vecs = np.concatenate([base, start_rows(rng, base, n_start, near)])
    adj = O.build_graph(vecs, n, n_start, O.L2, R, int(R * 1.3), 30)
    queries = np.concatenate([near[np.zeros(nq // 2, np.int64)], base[rng.integers(0, n, nq - nq // 2)]])
    queries = queries + np.float32(0.05) * rng.normal(size=queries.shape).astype(np.float32)
    return Case(vecs, adj, n, n_start, O.L2, queries.astype(np.float32))


def malformed(adj, n, n_start, max_degree, seed):
    """rows of width max_degree rewritten by hand from a built graph: each neighbour v may be preceded by v + 2^K
    (the same bucket and tag as v), an id in [n_total, 2^K), UINT32_MAX, the node itself or a start point, and followed
    by a repeat of itself; every fifth row is filled to exactly max_degree, every 23rd row is empty and so is the
    second start point's"""
    rng = np.random.default_rng(seed)
    total = n + n_start
    K = k_bits(total)
    assert total + 64 < (1 << K)
    out = np.zeros((total, max_degree + 1), np.uint32)
    for u in range(total):
        row = []
        for v in adj[u, 1:1 + adj[u, 0]].tolist():
            r = rng.integers(0, 8)
            extra = {0: [v + (1 << K)], 1: [total + int(rng.integers(0, 64))], 2: [EMPTY], 3: [u], 4: [n + int(rng.integers(0, n_start))],
                     5: [v + (3 << K)]}.get(int(r), [])
            row += extra + [v] + ([v] if r == 6 else [])
        if u % 5 == 0:
            while len(row) < max_degree:
                row.append(int(rng.integers(0, total)))
        row = row[:max_degree]
        if u % 23 == 0 or (n_start > 1 and u == n + 1):
            row = []
        out[u, 0] = len(row)
        out[u, 1:1 + len(row)] = row
    return out


def malformed_case(n, d, n_start, max_degree, nq, seed):
    c = many_starts(n, d, n_start, nq, seed, R=12)
    return Case(c.vecs, malformed(c.adj, n, n_start, max_degree, seed), n, n_start, O.L2, c.queries)


def aliasing_case(n, d, nq, seed, dt=np.float32):
    """every neighbour v of every row is preceded by v + 2^K: the ids >= 2^K are out of bounds, but a tag table that
    took them would hold v's tag before v is scored"""
    rng = np.random.default_rng(seed)
    base = clustered(rng, n, d).astype(dt)
    vecs = np.concatenate([base, base[:1]])
    adj = O.build_graph(vecs, n, 1, O.L2, 12, 15, 30)
    K = k_bits(n + 1)
    out = np.zeros((n + 1, 31), np.uint32)
    for u in range(n + 1):
        nb = adj[u, 1:1 + adj[u, 0]].astype(np.uint64)
        row = np.stack([nb + (1 << K), nb], 1).reshape(-1)
        out[u, 0] = len(row)
        out[u, 1:1 + len(row)] = row
    queries = (base[rng.integers(0, n, nq)].astype(np.float32) + 0.05 * rng.normal(size=(nq, d)).astype(np.float32)).astype(dt)
    return Case(vecs, out, n, 1, O.L2, queries)


def disconnected(n, d, n_start, reach, nq, seed):
    """a built graph whose start points reach only `reach` base points (the rest is a separate component)"""
    c = many_starts(n, d, n_start, nq, seed)
    adj = c.adj.copy()
    small = list(range(reach)) + list(range(n, n + n_start))
    for j, u in enumerate(small):
        row = [small[(j + i) % len(small)] for i in range(1, min(len(small), adj.shape[1]))]  # a ring: all reachable
        adj[u, 0] = len(row)
        adj[u, 1:] = 0
        adj[u, 1:1 + len(row)] = row
    return Case(c.vecs, adj, n, n_start, O.L2, c.queries)


def grid(n, d, n_start, nq, seed):
    """integer coordinates in {0, 1, 2} and every tenth row duplicated: distances tie exactly all along the list"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 3, size=(n, d)).astype(np.float32)
    base[1::10] = base[0:-1:10]
    vecs = np.concatenate([base, base[rng.integers(0, n, n_start)]])
    adj = O.build_graph(vecs, n, n_start, O.L2, 16, 20, 30)
    queries = rng.integers(0, 3, size=(nq, d)).astype(np.float32)
    return Case(vecs, adj, n, n_start, O.L2, queries)


def non_finite(n, d, dt, metric, nq, seed, nan=True):
    """a graph built over finite rows, then every 7th row given ±inf entries (and every 11th NaN ones, f32): under L2
    inf - inf is NaN, under InnerProduct 0 * inf; the queue drops NaN candidates, which still count in cmps"""
    rng = np.random.default_rng(seed)
    base = clustered(rng, n, d)
    if metric == O.INNER_PRODUCT:
        base[:, ::5] = 0  # 0 * inf
    vecs = np.concatenate([base, base[:1]]).astype(dt)
    adj = O.build_graph(vecs, n, 1, metric, 16, 20, 30)
    bad = vecs.copy()
    bad[::7, 3] = np.inf
    bad[3::7, 5] = -np.inf
    bad[::14, 0::5] = np.inf
    if nan:
        bad[::11, 2] = np.nan
    bad[n] = vecs[n]  # a finite start point
    queries = base[rng.integers(0, n, nq)] + np.float32(0.05) * rng.normal(size=(nq, d)).astype(np.float32)
    queries[::9, 3] = np.inf
    return Case(bad, adj, n, 1, metric, queries.astype(dt)), vecs


# ---------------------------------------------------------------- CPU: the oracle on these graphs

CPU_KLB = [(10, 3, 1), (10, 30, 2), (5, 60, 4)]


def oracle_equals_restatement(case, klbs, nq=40):
    trace = {}
    for k, L, beam in klbs:
        want = case.oracle.search_batch(case.queries[:nq], k, L, beam=beam)
        same(py_batch(case, k, L, beam, nq, trace), want, (k, L, beam))
    return trace


@pytest.mark.parametrize("n_start", [2, 33, 70])
def test_oracle_with_many_start_points(n_start):
    case = many_starts(400, 8, n_start, 40, n_start)
    t = oracle_equals_restatement(case, CPU_KLB)
    assert t["starts_in_list"] > 0
    assert (case.oracle.search_batch(case.queries[:40], 10, 3)[2] < 10).any(), "start points fill a short list"


@pytest.mark.parametrize("max_degree", [1, 7, 40])
def test_oracle_on_malformed_rows(max_degree):
    case = malformed_case(400, 8, 3, max_degree, 40, max_degree)
    t = oracle_equals_restatement(case, CPU_KLB)
    assert t["repeat"] > 0 and t["oob"] > 0
    if max_degree > 1:
        assert t["alias_then_scored"] > 0, "an aliasing id precedes its node, which is then scored"


def test_oracle_on_aliasing_ids():
    t = oracle_equals_restatement(aliasing_case(400, 8, 40, 1), CPU_KLB)
    assert t["alias_then_scored"] > 0


@pytest.mark.parametrize("reach", [4, 20])
def test_oracle_on_a_disconnected_graph(reach):
    case = disconnected(300, 8, 2, reach, 40, reach)
    oracle_equals_restatement(case, CPU_KLB)
    ids, dists, counts = case.oracle.search_batch(case.queries, 10, 30)[:3]
    assert (counts == min(reach, 10)).all()
    assert (ids[:, reach:] == EMPTY).all() and np.isposinf(dists[:, reach:]).all()


def test_oracle_on_exact_ties():
    case = grid(400, 8, 3, 40, 3)
    oracle_equals_restatement(case, [(10, 30, 1), (10, 60, 2), (10, 300, 1)])
    d = case.oracle.search_batch(case.queries[:40], 10, 30)[1]
    assert (d[:, 1:] == d[:, :-1]).any(), "tied distances inside the results"


@pytest.mark.parametrize("dt,metric", [(np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.L2), (np.float16, O.INNER_PRODUCT)])
def test_oracle_on_non_finite_rows(dt, metric):
    case, _ = non_finite(400, 16, dt, metric, 40, 7, nan=dt == np.float32)
    t = oracle_equals_restatement(case, CPU_KLB)
    assert t["nan"] > 0, "NaN candidates are dropped"


def test_tag16_aliases_ids_beyond_2_to_the_k():
    """v and v + 2^K get the same bucket and tag, while ids below 2^K never collide: a tag table must not take ids
    beyond 2^K (none of them is in bounds)."""
    for K, nbk in ((12, 128), (12, 16), (20, 283)):
        kmask, magic, shift = tag_map(K, nbk)

        def key(ids):
            h = (ids.astype(np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF) & np.uint64(kmask)
            tag = (h * np.uint64(magic)) >> np.uint64(shift)
            return h - tag * np.uint64(nbk), tag

        v = np.arange(1 << K, dtype=np.uint64)
        b, t = key(v)
        assert len(np.unique(b * np.uint64(1 << 14) + t)) == 1 << K
        for alias in (v + np.uint64(1 << K), v + np.uint64(5 << K), (v | np.uint64(0xFFFFFFFF ^ kmask))):
            ba, ta = key(alias & np.uint64(0xFFFFFFFF))
            assert np.array_equal(ba, b) and np.array_equal(ta, t)


# ---------------------------------------------------------------- GPU harness

def index(case, quant):
    """the case's index with its rows, graph and PQ codes"""
    g = dab.GpuIndex(O.dtype_code(case.vecs), case.metric, case.vecs.shape[1], case.n, case.n_start, case.max_degree)
    g.upload_vectors(case.vecs)
    g.upload_graph(case.adj)
    g.upload_pq(quant.piv, quant.off, quant.codes)
    return g


class Quantized:
    """PQ codes, SQ 8 / 4-bit rows and MinMax 8-bit rows of a case (from `clean` rows) and their oracles"""

    def __init__(self, case, clean=None, chunks=16):
        clean = case.vecs if clean is None else clean
        rng = np.random.default_rng(11)
        d = case.vecs.shape[1]
        self.piv, self.off = trained_pq(rng, clean[:case.n], chunks)
        self.codes = np.zeros((case.total, chunks), np.uint8)
        for i in range(case.total):
            assert O.lib().orc_pq_encode(O.ptr(self.piv), 256, d, O.ptr(self.off), chunks, O.ptr(clean[i]), O.ptr(self.codes[i])) == 0
        self.pq = O.Index(case.vecs, case.adj, case.n, case.n_start, case.metric, pq=(self.piv, self.off, self.codes))
        self.sq_quant = sq_quantizer(clean, case.metric)
        self.sq = {}
        for nbits in (8, 4):
            rows = O.sq_encode_rows(clean, self.sq_quant[0], self.sq_quant[1], nbits)
            self.sq[nbits] = (rows, O.Index(case.vecs, case.adj, case.n, case.n_start, case.metric, sq=(rows, nbits, *self.sq_quant)))
        self.mm_rows = compress(clean, None, 8)
        self.mm_queries = compress(case.queries, None, 8)
        self.mm = MinMaxOracle(case.vecs, case.adj, case.n, case.n_start, case.metric, self.mm_rows, 8)


@functools.lru_cache(maxsize=None)
def oracle_runs(case, quant, k, L, beam):
    """(path, rerank) -> the oracle's five outputs"""
    q = case.queries
    out = {("fp", False): case.want(k, L, beam)}
    if quant is not None:
        for r in (False, True):
            run = quant.pq.search_batch_rerank if r else quant.pq.search_batch
            out["pq", r] = run(q, k, L, beam=beam, threads=4)
            for nbits, (_, o) in quant.sq.items():
                run = o.search_batch_rerank if r else o.search_batch
                out[f"sq{nbits}", r] = run(q, k, L, beam=beam, threads=4)
            out["mm", r] = quant.mm.search(q, quant.mm_queries, k, L, beam=beam, rerank=r)
    return out


def run_paths(monkeypatch, case, klbs, quant=None, env_variants=("", "global_lut", "overflow")):
    """every applicable path against the oracle; `env_variants` picks the index configurations (the DAB_TEST_*
    variables are read when the index is created)"""
    results = {}
    for variant in env_variants:
        monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
        monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
        if variant == "global_lut":
            if quant is None:
                continue
            monkeypatch.setenv("DAB_TEST_PQ_GLOBAL_LUT", "1")
        elif variant == "overflow":
            monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
        with dab.GpuIndex(O.dtype_code(case.vecs), case.metric, case.vecs.shape[1], case.n, case.n_start, case.max_degree) as g:
            g.upload_vectors(case.vecs)
            g.upload_graph(case.adj)
            if quant is not None:
                g.upload_pq(quant.piv, quant.off, quant.codes)
            for k, L, beam in klbs:
                want = oracle_runs(case, quant, k, L, beam)
                results[k, L, beam] = want
                what = (variant, k, L, beam)
                if variant != "global_lut":
                    same(g.search_batch(case.queries, k, L, beam), want["fp", False], what + ("fp sync",))
                    out = g.search_batch_async(0, case.queries, k, L, beam)
                    g.wait(0)
                    same(out, want["fp", False], what + ("fp in flight",))
                if quant is None or L + case.n_start > 1024:
                    continue
                for r in (False, True):
                    same(g.search_batch_pq(case.queries, k, L, beam, rerank=r), want["pq", r], what + ("pq", r))
                    if variant == "global_lut":
                        continue
                    for nbits, (rows, _) in quant.sq.items():
                        g.upload_sq(nbits, *quant.sq_quant, rows=rows)
                        same(g.search_batch_sq(case.queries, k, L, beam, rerank=r), want[f"sq{nbits}", r], what + ("sq", nbits, r))
                    g.upload_minmax(8, 1.0, None, rows=quant.mm_rows)
                    same(g.search_batch_minmax(case.queries, k, L, beam, rerank=r), want["mm", r], what + ("minmax", r))
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
    monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
    return results


# ---------------------------------------------------------------- GPU cases

@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 31, 32, 33, 70])
def test_many_start_points(monkeypatch, n_start):
    """start points in groups of 32 (a second and third group from 33 on), some tied with base rows, the others close
    to half of the queries: short lists hold mostly start points, so both output steps return fewer than k results.
    L + start points on both sides of 24 (v3 / v2) and 256 (tiled v2 / rows from global memory)."""
    case = many_starts(3000, 64, n_start, 120, 100 + n_start)
    quant = Quantized(case)
    klbs = [(10, 3, 1), (10, 24 - n_start, 1), (10, 25 - n_start, 2), (10, 60, 4), (10, 256 - n_start, 1), (10, 257 - n_start, 1)]
    klbs = [x for x in klbs if x[1] >= 1]
    res = run_paths(monkeypatch, case, klbs, quant)
    assert (res[10, 3, 1]["fp", False][2] < 10).any() and (res[10, 3, 1]["pq", True][2] < 10).any(), "fewer than k results"
    t = {}
    py_batch(case, 10, 60, 4, 8, t)
    assert t["starts_in_list"] > 0


@pytest.mark.gpu
def test_hundreds_of_start_points_and_the_quantized_list_limit(monkeypatch):
    """300 start points (ten groups of 32) with L = 5: L + start points > 256 on v2; the quantized traversals take
    L + start points = 1024 and reject 1025 with a clean error."""
    case = many_starts(3000, 64, 300, 64, 300)
    quant = Quantized(case)
    res = run_paths(monkeypatch, case, [(10, 5, 1), (10, 724, 1)], quant, env_variants=("",))
    assert (res[10, 5, 1]["fp", False][2] < 10).any()
    with dab.GpuIndex(dab.DType.f32, O.L2, 64, case.n, case.n_start, case.max_degree) as g:
        g.upload_vectors(case.vecs)
        g.upload_graph(case.adj)
        g.upload_pq(quant.piv, quant.off, quant.codes)
        g.upload_sq(8, *quant.sq_quant, rows=quant.sq[8][0])
        g.upload_minmax(8, 1.0, None, rows=quant.mm_rows)
        for fn in (g.search_batch_pq, g.search_batch_sq, g.search_batch_minmax):
            with pytest.raises(dab.DabError, match="1024"):
                fn(case.queries, 10, 725)
        same(g.search_batch(case.queries, 10, 725), case.want(10, 725, 1), "fp, L + start points = 1025")


@pytest.mark.gpu
@pytest.mark.parametrize("max_degree", [1, 7, 95, 96, 97, 200])
def test_malformed_adjacency_rows(monkeypatch, max_degree):
    """repeated ids (also across the rows of one beam), self-loops, edges into start points, ids in [n_total, 2^K),
    ids >= 2^K that alias a real node, UINT32_MAX, empty rows (a start point among them) and rows at exactly
    max_degree, on both sides of the 96-word adjacency buffer.  At max_degree 96 the synchronous device-pointer calls
    must equal the host calls."""
    case = malformed_case(3000, 64, 3, max_degree, 120, max_degree)
    assert (case.adj[:, 0] == max_degree).any() and (case.adj[:, 0] == 0).any() and case.adj[case.n + 1, 0] == 0
    quant = Quantized(case)
    run_paths(monkeypatch, case, [(10, 20, 1), (10, 60, 2), (10, 100, 4), (10, 300, 1)], quant)
    t = {}
    py_batch(case, 10, 60, 2, 16, t)
    if max_degree > 1:
        assert t["repeat"] > 0 and t["oob"] > 0 and t["alias_then_scored"] > 0
    if max_degree == 96:
        device_flavours(case, quant)


def device_flavours(case, quant):
    import torch
    nq, k, L = case.queries.shape[0], 10, 60
    d_q = torch.from_numpy(case.queries.view(np.uint8).copy()).cuda()
    bufs = (torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
            *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
    ptrs = [b.data_ptr() for b in bufs]
    with index(case, quant) as g:
        g.upload_sq(8, *quant.sq_quant, rows=quant.sq[8][0])
        calls = [(lambda: g.search_batch_device(d_q.data_ptr(), nq, k, L, 2, *ptrs), g.search_batch(case.queries, k, L, 2), "fp")]
        for r in (False, True):
            calls.append((lambda r=r: g.search_batch_pq_device(d_q.data_ptr(), nq, k, L, 2, *ptrs, rerank=r),
                          g.search_batch_pq(case.queries, k, L, 2, rerank=r), ("pq", r)))
            calls.append((lambda r=r: g.search_batch_sq_device(d_q.data_ptr(), nq, k, L, 2, *ptrs, rerank=r),
                          g.search_batch_sq(case.queries, k, L, 2, rerank=r), ("sq", r)))
        for call, want, what in calls:
            for b in bufs:
                b.fill_(-1)
            torch.cuda.synchronize()
            call()
            torch.cuda.synchronize()
            same([b.cpu().numpy() for b in bufs], want, ("device", what))


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [64, 100])
def test_aliasing_ids_in_flight(monkeypatch, dim):
    """v + 2^K before v in every row: level 1 of search_kernel_v2's visited set (batches in flight; register rows at
    64-d, staged rows at 100-d) must not take the out-of-bounds id, or v would look visited and never be scored."""
    case = aliasing_case(3000, dim, 160, dim)
    t = {}
    py_batch(case, 10, 60, 1, 16, t)
    assert t["alias_then_scored"] > 0
    run_paths(monkeypatch, case, [(10, 20, 1), (10, 60, 1), (10, 100, 2), (10, 200, 4)], env_variants=("", "overflow"))


@pytest.mark.gpu
@pytest.mark.parametrize("reach", [6, 40])
def test_disconnected_graph(monkeypatch, reach):
    """the start points reach `reach` base points (fewer than k, or fewer than L): every path pads with UINT32_MAX /
    +inf."""
    case = disconnected(3000, 64, 2, reach, 120, reach)
    quant = Quantized(case)
    res = run_paths(monkeypatch, case, [(10, 20, 1), (10, 60, 2), (50, 100, 1), (10, 300, 1)], quant)
    for (k, L, beam), runs in res.items():
        for path, (ids, dists, counts, _, _) in runs.items():
            assert (counts == min(reach, k)).all(), (path, k, L)
            assert (ids[:, reach:] == EMPTY).all() and np.isposinf(dists[:, reach:]).all(), (path, k, L)


@pytest.mark.gpu
def test_exact_ties_at_long_lists(monkeypatch):
    """integer coordinates and duplicated rows at L >= 25: v2 synchronously, in flight and with L + start points > 256,
    and the quantized traversals."""
    case = grid(3000, 32, 2, 120, 9)
    quant = Quantized(case, chunks=8)
    res = run_paths(monkeypatch, case, [(10, 30, 1), (10, 100, 2), (20, 200, 4), (10, 300, 1)], quant)
    d = res[10, 30, 1]["fp", False][1]
    assert (d[:, 1:] == d[:, :-1]).any(), "tied distances inside the results"


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric,nan", [(np.float32, O.L2, True), (np.float32, O.INNER_PRODUCT, True), (np.float16, O.L2, False),
                                           (np.float16, O.INNER_PRODUCT, False), (np.float32, O.L2, False)])
def test_non_finite_rows(monkeypatch, dt, metric, nan):
    """NaN and ±inf entries in the rows (full precision): NaN distances are dropped by the queue and counted in cmps.
    With ±inf alone the PQ traversal (codes of the finite rows) and its full-precision rerank run too."""
    case, clean = non_finite(3000, 64, dt, metric, 120, 13 + metric, nan=nan)
    t = {}
    py_batch(case, 10, 60, 1, 16, t)
    assert t["nan"] > 0
    klbs = [(10, 20, 1), (10, 60, 2), (10, 300, 1)]
    run_paths(monkeypatch, case, klbs, env_variants=("", "overflow"))
    if dt == np.float32 and not nan:
        # finite queries only: an inf query entry against an inf row gives NaN rerank distances, whose order the
        # reference leaves unspecified
        fin = case.queries[np.isfinite(case.queries).all(1)]
        quant = Quantized(case, clean=clean)
        with index(case, quant) as g:
            for k, L, beam in klbs:
                for r in (False, True):
                    want = (quant.pq.search_batch_rerank if r else quant.pq.search_batch)(fin, k, L, beam=beam, threads=4)
                    same(g.search_batch_pq(fin, k, L, beam, rerank=r), want, ("pq", k, L, r))


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [2, 33])
@pytest.mark.parametrize("bs", [1, 0])
def test_device_build_with_several_start_points(n_start, bs):
    """dab_build with 2 and 33 start points, one insert at a time and at the default schedule: the adjacency equals the
    oracle's build bit for bit."""
    rng = np.random.default_rng(n_start + bs)
    n, d, R, Lb = 1500, 32, 16, 30
    base = clustered(rng, n, d)
    vecs = np.concatenate([base, start_rows(rng, base, n_start, base[:8])])
    maxdeg = int(R * 1.3)
    want = O.build_graph(vecs, n, n_start, O.L2, R, maxdeg, Lb) if bs == 1 else \
        O.build_graph_batched(vecs, n, n_start, O.L2, R, maxdeg, Lb, batch_size=bs)
    with dab.GpuIndex(dab.DType.f32, O.L2, d, n, n_start, maxdeg) as g:
        g.upload_vectors(vecs)
        g.build(R, Lb, 1.2, batch_size=bs)
        got = g.download_graph()
    assert np.array_equal(got[:, 0], want[:, 0]), "degrees differ"
    for i in range(n + n_start):
        assert np.array_equal(got[i, 1:1 + got[i, 0]], want[i, 1:1 + want[i, 0]]), i
