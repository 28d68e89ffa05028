"""Every search and graph update at the id widths of the 1M - 40M workloads (K, the bits of the largest id, up to 26).

A compact case (a few thousand points: the generators of test_traversal_edges and test_paged_search) is embedded into an
index of n_total ids by a monotone map: live id j becomes pos[j], a sorted random subset of [0, N) that holds every
boundary id below N (BOUNDARY and N - 1), start point j becomes N + j, and every other id is a filler row of degree 0
that no list names.  The map keeps the order of the ids and of every adjacency row, so every rule that orders by id or
by insertion (queue ties, start points as the largest ids, prune and consolidate order) is unchanged, and

    device(embedded) == map(oracle(compact))

for ids, distance bits, counts, cmps, hops, range offsets, pages and the adjacency after every update.  The CPU test
establishes this on the oracle itself; the GPU tests run at

  A  2^18, 2^18 + 1   search_kernel_v2's level 1 with the tests' 16-bucket table: on at K = 18 (largest tags), off at 19
  B  2^21, 2^21 + 1   level 1 with the 128-bucket table and the register-row path reading 268 MB of rows with the
                      evict-first policy, then staged rows without level 1; float cosine and u8 rows at 2^21 + 1
  C  2^23, 2^23 + 1   search_kernel_v3 with its smallest (512-bucket) table, K + s = 32; then v2 alone; i8 + PQ at K = 24
  D  2^25 + 1         K = 26: ids past 2^24, the start point's row and adjacency row at byte offset 2^32

Filler rows lie far from every query, except a few planted near-duplicates of probe queries that the exhaustive scans
must find.  Only one large index is alive at a time."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import diskann_b200 as dab
import diverse_oracle as V
import filtered_oracle as F
import inplace_delete_oracle as D
import insert_oracle as I
import oracle_lib as O
import range_oracle as R
from test_delete_consolidate import consolidate
from test_graph_stats import count_reachable, degree_stats, prune_range
from test_minmax_search import compress
from test_paged_search import PyPaged, built
from test_traversal_edges import EMPTY, Case, Quantized, grid, k_bits, many_starts, non_finite, oracle_runs, same

BOUNDARY = (0, 2**14 - 1, 2**18 - 1, 2**18, 2**21 - 1, 2**21, 2**23 - 1, 2**23, 2**24 - 1, 2**24, 2**24 + 1)
POOL = 1024  # distinct filler rows, repeated over the filler ids
PRUNED, LB = 16, 40  # pruned degree and build list of the update tests


def boundary_ids(N):
    return sorted({b for b in BOUNDARY if b < N} | {N - 1})


def hole_ids(N):
    """the ids the update tests insert into: compact ids of degree 0 that map to N - 1 and to 2^24 (the largest of 2^21,
    2^18, 2^14 - 1 below N - 1 in smaller indexes)"""
    return sorted({next(b for b in (2**24, 2**21, 2**18, 2**14 - 1) if b < N - 1), N - 1})


def widen(case, max_degree):
    adj = np.zeros((case.total, max_degree + 1), np.uint32)
    adj[:, :case.adj.shape[1]] = case.adj
    return Case(case.vecs, adj, case.n, case.n_start, case.metric, case.queries)


def as_case(t):
    """a (vecs, adj, n, n_start, metric, queries) tuple of test_paged_search.built"""
    return Case(*t)


def pool_rows(rng, dt, metric, n, d):
    """filler rows far from the data and the queries (small ones under inner product, where they cannot win)"""
    if dt == np.int8:
        return rng.integers(60, 128, (n, d)).astype(dt)
    if dt == np.uint8:
        return rng.integers(230, 256, (n, d)).astype(dt)
    if metric == O.L2:
        return (40 + rng.normal(size=(n, d))).astype(dt)
    return (0.05 * rng.normal(size=(n, d))).astype(dt)


def probes(rng, dt, metric, n, d):
    """(queries, planted rows): each planted row is the nearest row of its query by a wide margin"""
    if dt == np.int8:
        q = rng.integers(-127, -100, (n, d)).astype(dt)
        return q, q.copy()
    if dt == np.uint8:
        q = rng.integers(0, 20, (n, d)).astype(dt)
        return q, q.copy()
    if metric == O.L2:
        q = (-40 + rng.normal(size=(n, d))).astype(dt)
        return q, (q.astype(np.float32) + 1e-3 * rng.normal(size=(n, d))).astype(dt)
    q = rng.normal(size=(n, d)).astype(dt)
    return q, (8 * q.astype(np.float32)).astype(dt)


class Embedded:
    """The compact case (with degree-0 rows at the ranks of `holes`) and its embedding into n_total ids."""

    def __init__(self, base, n_total, seed, holes=()):
        rng = np.random.default_rng(seed)
        ns, d, dt = base.n_start, base.vecs.shape[1], base.vecs.dtype
        N = n_total - ns
        self.N, self.n_total, self.metric = N, n_total, base.metric
        m = base.n + len(holes)
        must = np.array(boundary_ids(N), np.int64)
        extra = np.setdiff1d(rng.choice(N, m + len(must) + 16, replace=False), must)
        self.pos = np.sort(np.concatenate([must, rng.permutation(extra)[:m - len(must)]]))
        assert len(self.pos) == m and len(np.unique(self.pos)) == m
        hole_rank = np.searchsorted(self.pos, holes)
        assert np.array_equal(self.pos[hole_rank], holes)

        # the compact case: base's points at the other ranks, degree-0 rows at the holes
        self.pool = pool_rows(rng, dt, base.metric, POOL, d)
        remap = np.concatenate([np.setdiff1d(np.arange(m), hole_rank), m + np.arange(ns)]).astype(np.uint32)
        vecs = np.zeros((m + ns, d), dt)
        vecs[remap] = base.vecs
        vecs[hole_rank] = self.pool[:len(holes)]
        adj = np.zeros((m + ns, base.adj.shape[1]), np.uint32)
        adj[remap, 0] = base.adj[:, 0]
        assert all((base.adj[u, 1:1 + base.adj[u, 0]] < base.total).all() for u in range(base.total))
        adj[remap, 1:] = remap[base.adj[:, 1:]]
        # queries at every live boundary id (the last n_near queries), so that each of them is found
        self.near_ids = np.array([b for b in must if b not in holes], np.uint32)
        near = vecs[np.searchsorted(self.pos, self.near_ids)].astype(np.float32)
        near[~np.isfinite(near)] = 0  # rows of the non-finite case
        if dt in (np.float32, np.float16):
            near = near + np.float32(0.01) * rng.normal(size=near.shape).astype(np.float32)
        queries = np.concatenate([base.queries, near.astype(dt)])
        self.n_near = len(near)
        self.compact = Case(vecs, adj, m, ns, base.metric, queries)
        self.holes = np.array(holes, np.uint32)
        self.hole_rank = hole_rank.astype(np.uint32)
        self.lut = np.concatenate([self.pos, N + np.arange(ns)]).astype(np.uint32)

        # the first filler ids above 2^21 and 2^24 + 1 and the last one below N hold planted near-duplicates of probe
        # queries (at D the last is just below byte offset 2^32)
        live = set(self.pos.tolist())
        plants = []
        for t, step in ((2**21, 1), (2**24 + 2, 1), (N - 1, -1)):
            c = min(t, N - 1)
            while c in live or c in plants:
                c += step
            if c < N:
                plants.append(c)
        self.plant_ids = np.array(plants, np.uint32)
        self.probe_queries, self.plant_rows = probes(rng, dt, base.metric, len(plants), d)

        # the embedded arrays
        self.vecs = self.scatter(vecs, self.pool, self.plant_rows)
        self.adj = np.zeros((n_total, adj.shape[1]), np.uint32)
        self.adj[self.lut] = self.map_adj(adj)
        self.max_degree = adj.shape[1] - 1

    # ---- the map
    def scatter(self, compact_rows, pool, plant_rows=None):
        """rows of every embedded id: the compact rows at their ids, pool rows at the fillers"""
        out = pool[np.arange(self.n_total) % len(pool)]
        out[self.lut] = compact_rows
        if plant_rows is not None:
            out[self.plant_ids] = plant_rows
        return out

    def ids(self, ids):
        ids = np.asarray(ids, np.uint32)
        assert ((ids < len(self.lut)) | (ids == EMPTY)).all(), "a compact result holds an id outside the compact index"
        return np.where(ids == EMPTY, EMPTY, self.lut[np.minimum(ids, len(self.lut) - 1)]).astype(np.uint32)

    def out(self, res):
        """a k-NN result (ids, dists, counts, cmps, hops) with its ids mapped"""
        return (self.ids(res[0]),) + tuple(res[1:])

    def map_adj(self, adj):
        out = self.lut[adj]
        out[:, 0] = adj[:, 0]
        return out

    def full_adj(self, adj):
        out = np.zeros((self.n_total, adj.shape[1]), np.uint32)
        out[self.lut] = self.map_adj(adj)
        return out

    @property
    def queries(self):
        return self.compact.queries

    def oracle(self):
        return O.Index(self.vecs, self.adj, self.N, self.compact.n_start, self.metric)


# ---------------------------------------------------------------- CPU: the oracle is invariant under the embedding

def same_range(got, want, what):
    for a, b, name in zip(got, want, ("offsets", "ids", "dists", "cmps", "hops", "second")):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), (what, name)


def search_attrs(emb, seed):
    """attribute values / presence (diverse search) and label sets (filtered search) of the compact ids"""
    rng = np.random.default_rng(seed)
    total = emb.compact.total
    values = rng.integers(0, 6, total).astype(np.uint32)
    present = (rng.random(total) < 0.9).astype(np.uint8)
    labels = rng.integers(0, 16, total).astype(np.uint64)
    masks = (np.uint64(1) << rng.integers(0, 4, len(emb.queries)).astype(np.uint64)).astype(np.uint64)
    return values, present, labels, masks


def radius_of(case):
    """a radius that holds a few points of most queries"""
    return float(np.median(case.want(10, 40, 1)[1][:, 4]))


@pytest.mark.parametrize("kind", ["many_starts", "grid"])
@pytest.mark.parametrize("n_total", [2**18, 2**18 + 1, 2**21, 2**21 + 1])
def test_oracle_is_invariant_under_the_embedding(n_total, kind):
    """oracle(embedded) == map(oracle(compact)) for every operation family the GPU tests compare through the map, on
    clustered rows with three start points and on integer rows whose distances tie exactly"""
    N = n_total - 3
    base = many_starts(600, 16, 3, 24, n_total & 7) if kind == "many_starts" else grid(600, 16, 3, 24, n_total & 7)
    emb = Embedded(base, n_total, n_total, holes=hole_ids(N))
    c, big = emb.compact, emb.oracle()
    assert k_bits(n_total) == {2**18: 18, 2**18 + 1: 19, 2**21: 21, 2**21 + 1: 22}[n_total]
    q = emb.queries
    for k, L, beam in [(10, 21, 1), (10, 60, 4), (10, 300, 1)]:
        same(big.search_batch(q, k, L, beam=beam), emb.out(c.want(k, L, beam)), ("knn", k, L, beam))
    rad = radius_of(c)
    want = R.range_search(c.oracle, q, 40, rad)
    assert want[0][-1] > len(q)
    same_range(R.range_search(big, q, 40, rad), (want[0], emb.ids(want[1])) + want[2:], "range")
    values, present, labels, masks = search_attrs(emb, 5)
    want = V.search_batch(c.oracle, q, 10, 40, 2, values, present)
    got = V.search_batch(big, q, 10, 40, 2, emb.scatter(values, np.zeros(1, np.uint32)), emb.scatter(present, np.zeros(1, np.uint8)))
    same(got[:5], emb.out(want[:5]), "diverse")
    want = F.search_batch(c.oracle, q, 10, 30, labels, masks, adaptive_l=(20, 3.0))
    got = F.search_batch(big, q, 10, 30, emb.scatter(labels, np.zeros(1, np.uint64)), masks, adaptive_l=(20, 3.0))
    same(got, emb.out(want), "filtered")
    for qi in range(4):
        a = PyPaged(c.vecs, c.adj, c.n, c.n_start, c.metric, q[qi], 30)
        b = PyPaged(emb.vecs, emb.adj, emb.N, c.n_start, c.metric, q[qi], 30)
        for _ in range(4):
            pa, pb = a.next_page(7), b.next_page(7)
            assert [(int(emb.lut[i]), d) for i, d in pa] == [(int(i), d) for i, d in pb] and (a.cmps, a.hops) == (b.cmps, b.hops)

    # the updates
    ns, total = c.n_start, c.total
    dead = np.setdiff1d(np.searchsorted(emb.pos, boundary_ids(emb.N)), emb.hole_rank)[:6]
    deleted = np.zeros(total, bool)
    deleted[dead] = True
    big_deleted = np.zeros(n_total, bool)
    big_deleted[emb.lut[dead]] = True
    want, wn = consolidate(c.vecs, c.adj, c.n, ns, c.metric, deleted, 12)
    # consolidate_vector leaves a degree-0 row that is not deleted alone: the filler ids are skipped
    got, gn = consolidate(emb.vecs, emb.adj, emb.N, ns, c.metric, big_deleted, 12, order=emb.lut)
    assert wn == gn > 0 and np.array_equal(got, emb.full_adj(want)), "consolidate"

    rng = np.random.default_rng(1)
    fresh = (c.vecs[rng.integers(0, c.n, len(emb.holes))].astype(np.float32) + 0.05).astype(c.vecs.dtype)
    cv, bv = c.vecs.copy(), emb.vecs.copy()
    cv[emb.hole_rank], bv[emb.holes] = fresh, fresh
    want = I.insert_batched(cv, c.adj, emb.hole_rank, c.n, ns, c.metric, PRUNED, c.max_degree, LB)
    got = I.insert_batched(bv, emb.adj, emb.holes, emb.N, ns, c.metric, PRUNED, c.max_degree, LB)
    assert np.array_equal(got, emb.full_adj(want)), "insert"

    ids = rng.choice(np.setdiff1d(np.arange(c.n), emb.hole_rank), 30, replace=False)
    for method in (D.VISITED_AND_TOPK, D.TWO_HOP_AND_ONE_HOP, D.ONE_HOP):
        wa, ww = D.inplace_delete(c.vecs, c.adj, D.deleted_words(total, dead), ids, c.n, ns, c.metric, method, 3, 12, batch_size=7)
        ga, gw = D.inplace_delete(emb.vecs, emb.adj, D.deleted_words(n_total, emb.lut[dead]), emb.lut[ids], emb.N, ns, c.metric, method,
                                  3, 12, batch_size=7)
        assert np.array_equal(ga, emb.full_adj(wa)), ("inplace_delete", method)
        assert np.array_equal(D.deleted_ids(gw, n_total), emb.lut[D.deleted_ids(ww, total)]), ("inplace_delete", method)
    words = D.deleted_words(total, np.concatenate([dead, ids]))
    big_words = D.deleted_words(n_total, emb.lut[np.concatenate([dead, ids])])
    want, wn = D.drop_deleted_neighbors(wa, words, c.n, ns, 12)
    got, gn = D.drop_deleted_neighbors(ga, big_words, emb.N, ns, 12)
    assert wn == gn and np.array_equal(got, emb.full_adj(want)), "drop_deleted_neighbors"
    want, wn = prune_range(c.vecs, c.adj, c.n, ns, c.metric, np.arange(total), 8)
    got, gn = prune_range(emb.vecs, emb.adj, emb.N, ns, c.metric, emb.lut, 8)
    assert wn == gn and np.array_equal(got, emb.full_adj(want)), "prune_range"


# ---------------------------------------------------------------- GPU

SIZES = {  # base case (generator, dtype, metric, dim, start points), K and what runs beyond the searches; sizes with the
    # same `seed` embed the same compact case
    "A0": dict(n_total=2**18, K=18, case=("starts", np.float32, O.L2, 32, 3), log2=8),
    "A1": dict(n_total=2**18 + 1, K=19, case=("starts", np.float32, O.L2, 32, 3), log2=8),
    "B0": dict(n_total=2**21, K=21, case=("grid", np.float32, O.L2, 32, 2)),
    "B1": dict(n_total=2**21 + 1, K=22, case=("grid", np.float32, O.L2, 32, 2), updates=True),
    "B1cos": dict(n_total=2**21 + 1, K=22, case=("built", np.float32, O.COSINE, 32, 1)),
    "B1u8": dict(n_total=2**21 + 1, K=22, case=("built", np.uint8, O.L2, 32, 1)),
    "B1nf": dict(n_total=2**21 + 1, K=22, case=("non_finite", np.float32, O.L2, 32, 1), fp_only=True),
    "C0": dict(n_total=2**23, K=23, case=("built", np.float16, O.INNER_PRODUCT, 16, 1), seed=6, scans=True),
    "C0nf": dict(n_total=2**23, K=23, case=("non_finite", np.float16, O.INNER_PRODUCT, 16, 1), fp_only=True),
    "C1": dict(n_total=2**23 + 1, K=24, case=("built", np.float16, O.INNER_PRODUCT, 16, 1), seed=6, scans=True),
    "C1i8": dict(n_total=2**23 + 1, K=24, case=("built", np.int8, O.L2, 16, 1), scans=True),
    "D": dict(n_total=2**25 + 1, K=26, case=("starts", np.float32, O.L2, 32, 1), max_degree=31, updates=True, scans=True),
}


def base_case(name):
    kind, dt, metric, d, ns = SIZES[name]["case"]
    seed = SIZES[name].get("seed", list(SIZES).index(name))
    if kind == "starts":
        c = many_starts(3000, d, ns, 64, seed)
    elif kind == "grid":
        c = grid(3000, d, ns, 64, seed)
    elif kind == "non_finite":  # ±inf entries, and NaN ones in f32 rows
        c = non_finite(3000, d, dt, metric, 64, seed, nan=dt == np.float32)[0]
    else:
        c = as_case(built(3000, d, dt, metric, 64, seed))
    return widen(c, SIZES[name]["max_degree"]) if "max_degree" in SIZES[name] else c


@functools.lru_cache(maxsize=1)  # one large embedding alive at a time
def embedded(name):
    s = SIZES[name]
    base = base_case(name)
    holes = hole_ids(s["n_total"] - base.n_start) if s.get("updates") else ()
    emb = Embedded(base, s["n_total"], 1000 + list(SIZES).index(name), holes)
    assert k_bits(emb.n_total) == s["K"]
    c = emb.compact
    if s.get("fp_only"):
        return emb, None
    quant = Quantized(c, clean=c.vecs.astype(np.float32), chunks=8)
    if c.metric == O.COSINE:
        quant.sq = {}  # the scalar-quantized store has no Cosine (SQStore::distance_computer)
    return emb, quant


@pytest.fixture(scope="module")
def wide():
    yield embedded
    embedded.cache_clear()


def pq_encode_rows(quant, rows):
    rows = np.ascontiguousarray(rows, np.float32)
    out = np.zeros((len(rows), len(quant.off) - 1), np.uint8)
    for i in range(len(rows)):
        assert O.lib().orc_pq_encode(O.ptr(quant.piv), 256, rows.shape[1], O.ptr(quant.off), out.shape[1], O.ptr(rows[i]), O.ptr(out[i])) == 0
    return out


def store_rows(emb, quant, store):
    """the embedded index's PQ codes, SQ rows ("sq8", "sq4") or MinMax rows: the compact rows at their ids, the
    encoded pool and planted rows at the fillers"""
    enc = {"pq": lambda r: pq_encode_rows(quant, r),
           "sq8": lambda r: O.sq_encode_rows(r, quant.sq_quant[0], quant.sq_quant[1], 8),
           "sq4": lambda r: O.sq_encode_rows(r, quant.sq_quant[0], quant.sq_quant[1], 4),
           "mm": lambda r: compress(r, None, 8)}[store]
    compact = {"pq": quant.codes, "mm": quant.mm_rows}.get(store)
    if compact is None:
        compact = quant.sq[int(store[2:])][0]
    f32 = lambda r: np.ascontiguousarray(r, np.float32)
    return emb.scatter(compact, enc(f32(emb.pool)), enc(f32(emb.plant_rows)))


def gpu_index(vecs, adj, n, n_start, metric):
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, adj.shape[1] - 1)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


def indexes(emb):
    """(embedded index, compact index)"""
    c = emb.compact
    return gpu_index(emb.vecs, emb.adj, emb.N, c.n_start, c.metric), gpu_index(c.vecs, c.adj, c.n, c.n_start, c.metric)


def upload_store(g, gc, emb, quant, store):
    if store == "pq":
        g.upload_pq(quant.piv, quant.off, store_rows(emb, quant, "pq"))
        gc.upload_pq(quant.piv, quant.off, quant.codes)
    elif store.startswith("sq"):
        nbits = int(store[2:])
        g.upload_sq(nbits, *quant.sq_quant, rows=store_rows(emb, quant, store))
        gc.upload_sq(nbits, *quant.sq_quant, rows=quant.sq[nbits][0])
    else:
        g.upload_minmax(8, 1.0, None, rows=store_rows(emb, quant, "mm"))
        gc.upload_minmax(8, 1.0, None, rows=quant.mm_rows)


def device_buffers(nq, k):
    import torch
    return (torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
            *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))


def device_call(call, nq, k):
    import torch
    bufs = device_buffers(nq, k)
    for b in bufs:
        b.fill_(-1)
    torch.cuda.synchronize()
    call(*[b.data_ptr() for b in bufs])
    torch.cuda.synchronize()
    return [b.cpu().numpy() for b in bufs]


def check_pages(emb, s_emb, s_c, want_fp, what):
    """three pages of a paged session on the embedded index against the compact one, and (full precision) the
    restatement's pages of the first queries"""
    for page in range(3):
        got, ref = s_emb.next_page(10), s_c.next_page(10)
        same(got, emb.out(ref), (what, "page", page))
        for qi, py in enumerate(want_fp):
            p = py.next_page(10)
            assert [int(x) for x in got[0][qi][:len(p)]] == [int(emb.lut[i]) for i, _ in p], (what, page, qi)
            assert int(got[2][qi]) == len(p) and (int(got[3][qi]), int(got[4][qi])) == (py.cmps, py.hops), (what, page, qi)


def check_range(emb, got, want, what):
    same_range(got, (want[0], emb.ids(want[1])) + tuple(want[2:]), what)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", list(SIZES))
def test_searches(monkeypatch, wide, name):
    """every search of the library at the size against map(oracle(compact)), or map(device(compact)) where the oracle
    is the one the compact tests already pin: k-NN synchronously, in flight and over device pointers, the PQ traversal
    with both LUT kernels, SQ 8 / 4 bits and MinMax 8 bits with and without rerank, paged, range, diverse and filtered
    search"""
    import torch
    spec = SIZES[name]
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
    if spec.get("log2"):
        monkeypatch.setenv("DAB_TEST_VISITED_LOG2", str(spec["log2"]))
    else:
        monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
    emb, quant = wide(name)
    c = emb.compact
    q, nq, ns = c.queries, len(c.queries), c.n_start
    assert k_bits(emb.n_total) == spec["K"]
    klbs = [(10, 24 - ns, 1), (10, 24 - ns, 4), (10, 100, 1), (10, 100, 4), (10, 300, 1), (10, 300, 4)]
    qklbs = [(10, 24 - ns, 1), (10, 100, 4), (10, 300, 1)]
    free0 = torch.cuda.mem_get_info()[0]
    found = []
    g, gc = indexes(emb)
    with g, gc:
        for k, L, beam in klbs:
            want = emb.out(oracle_runs(c, quant, k, L, beam)["fp", False])
            got = g.search_batch(q, k, L, beam)
            same(got, want, (name, k, L, beam, "fp sync"))
            found.append(got[0])
            out = g.search_batch_async(0, q, k, L, beam)
            g.wait(0)
            same(out, want, (name, k, L, beam, "fp in flight"))
        d_q = torch.from_numpy(q.view(np.uint8).copy()).cuda()
        want = emb.out(oracle_runs(c, quant, 10, 100, 4)["fp", False])
        same(device_call(lambda *b: g.search_batch_device(d_q.data_ptr(), nq, 10, 100, 4, *b), nq, 10), want, (name, "fp device"))
        if quant is None:  # non-finite rows: the full-precision k-NN traversals, as test_traversal_edges runs them
            return

        rad = radius_of(c)
        check_range(emb, g.range_search(q, 40, rad), R.range_search(c.oracle, q, 40, rad), (name, "range fp"))
        values, present, labels, masks = search_attrs(emb, 7)
        g.upload_attributes(emb.scatter(values, np.zeros(1, np.uint32)), emb.scatter(present, np.zeros(1, np.uint8)))
        gc.upload_attributes(values, present)
        same(g.search_batch_diverse(q, 10, 60, 2, 2), emb.out(V.search_batch(c.oracle, q, 10, 60, 2, values, present, beam=2)[:5]),
             (name, "diverse fp"))
        g.upload_labels(emb.scatter(labels, np.zeros(1, np.uint64)))
        gc.upload_labels(labels)
        same(g.search_batch_filtered(q, masks, 10, 40, adaptive_l=(20, 3.0)),
             emb.out(F.search_batch(c.oracle, q, 10, 40, labels, masks, adaptive_l=(20, 3.0))), (name, "filtered fp"))
        py = [PyPaged(c.vecs, c.adj, c.n, ns, c.metric, q[i], 40) for i in range(8)]
        with g.paged_search(q, 40) as s, gc.paged_search(q, 40) as sc:
            check_pages(emb, s, sc, py, (name, "paged fp"))

        for store in ["pq"] + [f"sq{b}" for b in quant.sq] + ["mm"]:
            upload_store(g, gc, emb, quant, store)
            key = {"pq": "pq", "mm": "mm"}.get(store, store)
            run = {"pq": g.search_batch_pq, "mm": g.search_batch_minmax}.get(store, g.search_batch_sq)
            for k, L, beam in qklbs:
                for r in (False, True):
                    want = emb.out(oracle_runs(c, quant, k, L, beam)[key, r])
                    same(run(q, k, L, beam, rerank=r), want, (name, k, L, beam, store, r))
            tag = {"pq": "pq", "mm": "minmax"}.get(store, "sq")
            for r in (False, True):
                what = (name, store, r)
                check_range(emb, getattr(g, f"range_search_{tag}")(q, 40, rad, rerank=r),
                            getattr(gc, f"range_search_{tag}")(q, 40, rad, rerank=r), what + ("range",))
                same(getattr(g, f"search_batch_diverse_{tag}")(q, 10, 60, 2, 2, rerank=r),
                     emb.out(getattr(gc, f"search_batch_diverse_{tag}")(q, 10, 60, 2, 2, rerank=r)), what + ("diverse",))
                same(getattr(g, f"search_batch_filtered_{tag}")(q, masks, 10, 40, adaptive_l=(20, 3.0), rerank=r),
                     emb.out(getattr(gc, f"search_batch_filtered_{tag}")(q, masks, 10, 40, adaptive_l=(20, 3.0), rerank=r)),
                     what + ("filtered",))
            if store == "pq":
                want = emb.out(oracle_runs(c, quant, 10, 100, 4)["pq", True])
                same(device_call(lambda *b: g.search_batch_pq_device(d_q.data_ptr(), nq, 10, 100, 4, *b, rerank=True), nq, 10), want,
                     (name, "pq device"))
                with g.paged_search_pq(q, 40) as s, gc.paged_search_pq(q, 40) as sc:
                    check_pages(emb, s, sc, [], (name, "paged pq"))
        used = free0 - torch.cuda.mem_get_info()[0]
    print(f"\n{name}: n_total {emb.n_total}, device memory in use {used / 2**30:.2f} GiB")
    assert used < 12 * 2**30

    # the PQ traversal with the per-warp table in global memory
    monkeypatch.setenv("DAB_TEST_PQ_GLOBAL_LUT", "1")
    with gpu_index(emb.vecs, emb.adj, emb.N, ns, c.metric) as g:
        g.upload_pq(quant.piv, quant.off, store_rows(emb, quant, "pq"))
        for k, L, beam in qklbs:
            for r in (False, True):
                same(g.search_batch_pq(q, k, L, beam, rerank=r), emb.out(oracle_runs(c, quant, k, L, beam)["pq", r]),
                     (name, k, L, beam, "pq global lut", r))
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT")

    found = np.concatenate([f.ravel() for f in found])
    found = found[found != EMPTY]
    live_bounds = [b for b in boundary_ids(emb.N) if b not in set(emb.holes.tolist())]
    if c.metric == O.L2:  # a query next to each boundary id's row finds it (under inner product, other rows win)
        assert set(live_bounds) <= set(found.tolist()), sorted(set(live_bounds) - set(found.tolist()))
    if emb.N > 2**24:
        assert (found > 2**24).any()


def check_graph(g, emb, want, what, chunk=1 << 22):
    """the embedded index's whole adjacency == map(want), the compact adjacency: every filler row still empty"""
    expect = emb.map_adj(want)
    for first in range(0, emb.n_total, chunk):
        cnt = min(chunk, emb.n_total - first)
        got = g.download_graph(first, cnt)
        ref = np.zeros_like(got)
        sel = (emb.lut >= first) & (emb.lut < first + cnt)
        ref[emb.lut[sel] - first] = expect[sel]
        assert np.array_equal(got, ref), (what, first)


def host_degree_stats(g, emb, chunk=1 << 22):
    """get_degree_stats over every id, counted on the downloaded graph"""
    mx, mn, tot, lt2 = 0, None, 0, 0
    for first in range(0, emb.n_total, chunk):
        deg = g.download_graph(first, min(chunk, emb.n_total - first))[:, 0].astype(np.int64)
        mx, tot, lt2 = max(mx, int(deg.max())), tot + int(deg.sum()), lt2 + int((deg < 2).sum())
        mn = int(deg.min()) if mn is None else min(mn, int(deg.min()))
    return mx, np.float32(tot) / np.float32(emb.n_total), mn, lt2


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", [n for n, s in SIZES.items() if s.get("updates")])
def test_graph_updates(monkeypatch, wide, name):
    """delete (and searches over the tombstones), consolidate, release, insert into the filler-mapped ids 2^24 and N - 1,
    in-place delete with its three methods, drop_deleted_neighbors, prune_range, count_reachable and degree_stats: the
    embedded index's adjacency equals map(oracle(compact)) after every step, and the compact device index runs every step
    alongside for the searches"""
    monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
    emb, quant = wide(name)
    c = emb.compact
    q, ns, total, lut = c.queries, c.n_start, c.total, emb.lut
    assert k_bits(emb.n_total) == SIZES[name]["K"]
    rng = np.random.default_rng(3)
    holes = set(emb.hole_rank.tolist())
    dead = np.array([r for r in np.searchsorted(emb.pos, boundary_ids(emb.N)) if r not in holes], np.uint32)
    g, gc = indexes(emb)
    with g, gc:
        upload_store(g, gc, emb, quant, "pq")
        g.delete(lut[dead])
        gc.delete(dead)
        assert g.delete_status(lut[dead]).all() and not g.delete_status(emb.holes).any()
        for k, L, beam in [(10, 24 - ns, 1), (10, 100, 4), (10, 300, 1)]:
            same(g.search_batch(q, k, L, beam), emb.out(gc.search_batch(q, k, L, beam)), (name, "tombstones", k, L, beam))
            same(g.search_batch_pq(q, k, L, beam, rerank=True), emb.out(gc.search_batch_pq(q, k, L, beam, rerank=True)),
                 (name, "tombstones pq", k, L, beam))
        rad = radius_of(c)
        check_range(emb, g.range_search(q, 40, rad), gc.range_search(q, 40, rad), (name, "tombstones range"))

        deleted = np.zeros(total, bool)
        deleted[dead] = True
        adj, wn = consolidate(c.vecs, c.adj, c.n, ns, c.metric, deleted, PRUNED)
        assert wn > 0 and g.consolidate(PRUNED) == wn == gc.consolidate(PRUNED)
        check_graph(g, emb, adj, (name, "consolidate"))

        g.release(lut[dead])
        gc.release(dead)
        adj = gc.download_graph()
        assert (adj[dead, 0] == 0).all()
        check_graph(g, emb, adj, (name, "release"))

        vecs = c.vecs.copy()
        fresh = (c.vecs[rng.integers(0, c.n, len(holes))].astype(np.float32) + 0.05).astype(vecs.dtype)
        vecs[emb.hole_rank] = fresh
        adj = I.insert_batched(vecs, adj, emb.hole_rank, c.n, ns, c.metric, PRUNED, c.max_degree, LB)
        g.insert(emb.holes, fresh, PRUNED, LB)
        gc.insert(emb.hole_rank, fresh, PRUNED, LB)
        check_graph(g, emb, adj, (name, "insert"))
        got = g.search_batch(fresh, 10, 60)
        same(got, emb.out(gc.search_batch(fresh, 10, 60)), (name, "after insert"))
        assert set(emb.holes.tolist()) <= set(got[0].ravel().tolist()), "the inserted points are found"

        words = D.deleted_words(total)
        ids = rng.choice(np.setdiff1d(np.arange(c.n), emb.hole_rank), 90, replace=False).astype(np.uint32)
        for j, method in enumerate(("visited_and_topk", "two_hop_and_one_hop", "one_hop")):
            part = ids[30 * j:30 * (j + 1)]
            adj, words = D.inplace_delete(vecs, adj, words, part, c.n, ns, c.metric, j, 3, PRUNED, batch_size=7)
            g.inplace_delete(lut[part], 3, method, PRUNED, batch_size=7)
            gc.inplace_delete(part, 3, method, PRUNED, batch_size=7)
            check_graph(g, emb, adj, (name, "inplace_delete", method))
        assert np.array_equal(np.flatnonzero(g.delete_status(lut[:c.n])), D.deleted_ids(words, total))
        same(g.search_batch(q, 10, 100, 4), emb.out(gc.search_batch(q, 10, 100, 4)), (name, "after inplace_delete"))

        g.delete(lut[dead])  # soft-deleted again: their edges go too
        words = D.deleted_words(total, np.concatenate([ids, dead]))
        adj, wn = D.drop_deleted_neighbors(adj, words, c.n, ns, PRUNED)
        assert wn > 0 and g.drop_deleted_neighbors(PRUNED) == wn
        check_graph(g, emb, adj, (name, "drop_deleted_neighbors"))

        some = np.sort(rng.choice(total, 800, replace=False)).astype(np.uint32)
        adj, wn = prune_range(vecs, adj, c.n, ns, c.metric, some, 8)
        assert wn > 0 and g.prune_range(lut[some], 8) == wn
        check_graph(g, emb, adj, (name, "prune_range"))

        starts = list(range(c.n, total))
        assert g.count_reachable() == count_reachable(adj, starts)[0]
        assert g.count_reachable(lut[some[:5]]) == count_reachable(adj, some[:5])[0]
        for ids_ in (some, np.concatenate([some[:3], emb.hole_rank])):
            assert g.degree_stats(lut[ids_]) == degree_stats(adj, ids_), (name, "degree_stats")
        assert g.degree_stats() == host_degree_stats(g, emb)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", [n for n, s in SIZES.items() if s.get("scans")])
def test_encoders_and_exhaustive_scans(monkeypatch, wide, name):
    """pq_encode_all, sq_encode_all and minmax_encode_all over every row, bit-equal to the host encodes at every live id,
    every boundary id, the planted rows and 10K fillers; flat_knn (and at K <= 24 flat_knn_tc) against the oracle's
    exhaustive scan, where the planted near-duplicates just above 2^21 and 2^24 + 1 and just below N must win, and
    (L2) the queries next to the boundary ids find them"""
    monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
    emb, quant = wide(name)
    c = emb.compact
    assert k_bits(emb.n_total) == SIZES[name]["K"]
    rng = np.random.default_rng(5)
    sample = np.unique(np.concatenate([emb.lut, boundary_ids(emb.N), emb.plant_ids,
                                       rng.integers(0, emb.n_total, 10000)])).astype(np.int64)
    rows = np.ascontiguousarray(emb.vecs[sample], np.float32)
    with gpu_index(emb.vecs, emb.adj, emb.N, c.n_start, c.metric) as g:
        g.upload_pq(quant.piv, quant.off)
        g.pq_encode_all()
        assert np.array_equal(g.download_pq()[2][sample], pq_encode_rows(quant, rows)), "pq_encode_all"
        for nbits in (8, 4):
            g.upload_sq(nbits, *quant.sq_quant)
            g.sq_encode_all()
            assert np.array_equal(g.download_sq()[sample], O.sq_encode_rows(rows, quant.sq_quant[0], quant.sq_quant[1], nbits)), nbits
        g.upload_minmax(8)
        g.minmax_encode_all()
        assert np.array_equal(g.download_minmax()[sample], compress(rows, None, 8)), "minmax_encode_all"

        queries = np.concatenate([emb.probe_queries, c.queries[:8], c.queries[-emb.n_near:]])
        want_ids, want_d = O.bruteforce_knn(emb.vecs[:emb.N], queries, c.metric, 10)
        assert np.array_equal(want_ids[:len(emb.plant_ids), 0], emb.plant_ids)
        if c.metric == O.L2:
            assert np.array_equal(want_ids[-emb.n_near:, 0], emb.near_ids)
        ids, d = g.flat_knn(queries, 10)
        assert np.array_equal(ids, want_ids) and np.array_equal(d.view(np.uint32), want_d.view(np.uint32)), "flat_knn"
        if emb.n_total <= 2**24 + 1:
            ids, d = g.flat_knn_tc(queries, 10)
            assert np.array_equal(ids, want_ids) and np.array_equal(d.view(np.uint32), want_d.view(np.uint32)), "flat_knn_tc"


PROFILE = """
import json, os, sys
import numpy as np, torch
import test_wide_ids as W
out = {}
for name in sys.argv[1:]:
    if W.SIZES[name].get("log2"):
        os.environ["DAB_TEST_VISITED_LOG2"] = str(W.SIZES[name]["log2"])
    emb, _ = W.embedded(name)
    c = emb.compact
    with W.gpu_index(emb.vecs, emb.adj, emb.N, c.n_start, c.metric) as g:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            sync = g.search_batch(c.queries, 10, 24 - c.n_start)
            flight = g.search_batch_async(0, c.queries, 10, 100)
            g.wait(0)
            torch.cuda.synchronize()
    want = [emb.out(c.want(10, 24 - c.n_start, 1)), emb.out(c.want(10, 100, 1))]
    equal = all(np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))
                for got, w in zip((sync, flight), want) for a, b in zip(got, w))
    out[name] = {"kernels": sorted(e.key for e in prof.key_averages()), "equal": equal}
print(json.dumps(out))
"""


def v2_flags(kernels):
    """(L1, REG) of every search_kernel_v2 instantiation that launched"""
    out = set()
    for k in kernels:
        if "search_kernel_v2<" in k:
            args = [a.strip() for a in k.split("search_kernel_v2<", 1)[1].split(">", 1)[0].split(",")]
            out.add((args[-2] == "true", args[-1] == "true"))
    return out


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("pair", [("A0", "A1"), ("B0", "B1"), ("C0", "C1")])
def test_the_kernels_each_size_reaches(pair):
    """the k-NN calls of each boundary pair under torch.profiler (a process of its own): level 1 of search_kernel_v2 in
    flight at 2^18 with the tests' table and at 2^21 with the register rows, neither at 2^18 + 1 or 2^21 + 1, and
    search_kernel_v3 at 2^23 but not at 2^23 + 1"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    env.pop("DAB_TEST_VISITED_LOG2", None)
    p = subprocess.run([sys.executable, "-c", PROFILE, *pair], capture_output=True, text=True, timeout=1100, env=env, cwd=here)
    assert p.returncode == 0, p.stderr[-3000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    lo, hi = (out[n]["kernels"] for n in pair)
    assert out[pair[0]]["equal"] and out[pair[1]]["equal"]
    if pair[0] == "A0":
        assert (True, False) in v2_flags(lo) or (True, True) in v2_flags(lo), lo
        assert v2_flags(hi) == {(False, False)}, hi
    elif pair[0] == "B0":
        assert (True, True) in v2_flags(lo), lo
        assert v2_flags(hi) == {(False, False)}, hi
    else:
        assert any("search_kernel_v3" in k for k in lo), lo
        assert not any("search_kernel_v3" in k for k in hi), hi


def malformed_rows(emb, seed):
    """test_traversal_edges.malformed over the embedded rows, with the embedded index's K: each neighbour v may be
    preceded by v + 2^K or v + 3 * 2^K (the same bucket and tag as v), an id in [n_total, n_total + 64) below 2^K,
    UINT32_MAX, the node itself or a start point, and followed by a repeat of itself; every fifth row is filled to
    max_degree with ids of [0, n_total) (mostly fillers), every 23rd row is empty.  Only the rows of compact ids are
    rewritten (a loop over the compact case, not over n_total)."""
    rng = np.random.default_rng(seed)
    total, K, md = emb.n_total, k_bits(emb.n_total), emb.max_degree
    assert total + 64 < (1 << K) and (4 << K) <= 2**32
    starts = emb.lut[emb.compact.n:].tolist()
    adj = emb.adj.copy()
    for j, u in enumerate(emb.lut.tolist()):
        row = []
        for v in emb.adj[u, 1:1 + emb.adj[u, 0]].tolist():
            r = int(rng.integers(0, 8))
            extra = {0: [v + (1 << K)], 1: [total + int(rng.integers(0, 64))], 2: [EMPTY], 3: [u],
                     4: [starts[int(rng.integers(0, len(starts)))]], 5: [v + (3 << K)]}.get(r, [])
            row += extra + [v] + ([v] if r == 6 else [])
        if j % 5 == 0:
            row += rng.integers(0, total, max(0, md - len(row))).tolist()
        row = row[:md] if j % 23 else []
        adj[u, 0] = len(row)
        adj[u, 1:1 + len(row)] = row
        adj[u, 1 + len(row):] = 0
    return adj


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", ["B1", "C1", "D"])
def test_malformed_rows(monkeypatch, wide, name):
    """rows rewritten after the embedding with ids in [n_total, 2^K), ids v + 2^K that share v's quotient tag, UINT32_MAX,
    self-loops, edges into start points, repeats, full and empty rows, at K = 22, 24 and 26: the full-precision traversals
    (synchronous and in flight) and the PQ traversal with and without rerank equal oracle_lib.Index on the embedded
    arrays"""
    monkeypatch.delenv("DAB_TEST_VISITED_LOG2", raising=False)
    monkeypatch.delenv("DAB_TEST_PQ_GLOBAL_LUT", raising=False)
    emb, quant = wide(name)
    c = emb.compact
    q, ns, K = c.queries, c.n_start, SIZES[name]["K"]
    assert k_bits(emb.n_total) == K
    adj = malformed_rows(emb, 11)
    named = np.concatenate([adj[u, 1:1 + adj[u, 0]] for u in emb.lut.tolist()]).astype(np.uint64)
    assert ((named >= emb.n_total) & (named < 1 << K)).any() and (named >= 1 << K).any() and (named == EMPTY).any()
    codes = store_rows(emb, quant, "pq")
    fp = O.Index(emb.vecs, adj, emb.N, ns, c.metric)
    pq = O.Index(emb.vecs, adj, emb.N, ns, c.metric, pq=(quant.piv, quant.off, codes))
    with gpu_index(emb.vecs, adj, emb.N, ns, c.metric) as g:
        g.upload_pq(quant.piv, quant.off, codes)
        for k, L, beam in [(10, 24 - ns, 1), (10, 60, 2), (10, 100, 4), (10, 300, 1)]:
            want = fp.search_batch(q, k, L, beam=beam, threads=4)
            same(g.search_batch(q, k, L, beam), want, (name, k, L, beam, "fp sync"))
            out = g.search_batch_async(0, q, k, L, beam)
            g.wait(0)
            same(out, want, (name, k, L, beam, "fp in flight"))
            for r in (False, True):
                want = (pq.search_batch_rerank if r else pq.search_batch)(q, k, L, beam=beam, threads=4)
                same(g.search_batch_pq(q, k, L, beam, rerank=r), want, (name, k, L, beam, "pq", r))
