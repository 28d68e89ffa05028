"""Paged search: DiskANNIndex::paged_search + PagedSearch::next_page, each query's state resident on the device.

CPU: a Python restatement of the reference's paged session (index.rs:2075-2155, paged.rs:53-149, the resizable
NeighborPriorityQueue of queue.rs) with distances from the oracle reproduces the reference's three checked-in baselines
page by page, and on built graphs pages are disjoint, sorted, at most k long and, paged to exhaustion, return every
node reachable from the start points exactly once.
GPU: the device equals the restatement bit for bit after every page (ids, distance bits, counts, cumulative cmps and
hops) for every row type, on graphs with many start points, malformed rows and exact ties, with visited tables that
overflow in the middle of a session, with interleaved sessions, and across persistent-grid rounds."""
import bisect
import json
import os

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
from test_oracle_golden import grid as lattice
from test_traversal_edges import clustered, grid as tie_grid, malformed_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EMPTY = 0xFFFFFFFF


# ---------------------------------------------------------------- the reference's paged session, restated

class PyPaged:
    """One query's paged session.  The queue is resizable (search_param_l = L + #start, never evicts), visited starts
    as the start ids, the start points are expanded once and not queued, nothing is counted until the first page."""

    def __init__(self, vecs, adj, n_points, n_start, metric, query, L):
        self.adj, self.n_points, self.total, self.L = adj, n_points, n_points + n_start, L
        self.max_degree = adj.shape[1] - 1
        q = np.ascontiguousarray(query.astype(np.float32) if vecs.dtype == np.float16 else query)  # f16 queries are widened
        self.dist = lambda ids: O.distance_rows(q, vecs[ids], metric, O.AVX2)
        self.cap = L + n_start
        self.ids, self.ds, self.done, self.cursor = [], [], [], 0
        self.starts = set(range(n_points, self.total))
        self.visited = set(self.starts)
        self.cmps = self.hops = 0
        fresh = []
        for s in range(n_points, self.total):
            fresh += self._expand(s)
        self._insert(fresh)

    def _expand(self, u):
        out = []
        for v in self.adj[u, 1:1 + min(int(self.adj[u, 0]), self.max_degree)].tolist():
            if v in self.visited:  # visited insert first ...
                continue
            self.visited.add(v)
            if v < self.total:  # ... then is_in_bounds
                out.append(v)
        return out

    def _insert(self, fresh):
        if not fresh:
            return
        for i, d in zip(fresh, self.dist(np.array(fresh, np.int64))):
            if np.isnan(d):
                continue
            at = bisect.bisect_left(self.ds, float(d))  # first entry with distance >= d
            self.ids.insert(at, i), self.ds.insert(at, float(d)), self.done.insert(at, False)
            self.cursor = min(self.cursor, at)

    def next_page(self, k):
        if k == 0 or k > self.L:
            raise ValueError(f"k = {k} outside [1, L = {self.L}]")
        # search_internal, beam width 1: closest_notvisited hands out the entry at the cursor, visited or not
        while self.cursor < min(self.cap, len(self.ids)):
            cur = self.cursor
            self.done[cur] = True
            self.cursor += 1
            while self.cursor < len(self.ids) and self.done[self.cursor]:
                self.cursor += 1
            fresh = self._expand(self.ids[cur])
            self._insert(fresh)
            self.cmps += len(fresh)
            self.hops += 1
        # filter_search_candidates over best.iter(), then drain_best
        page, considered = [], 0
        for i, d in zip(self.ids[:min(self.cap, len(self.ids))], self.ds):
            considered += 1
            if i not in self.starts:
                page.append((i, d))
                if len(page) >= k:
                    break
        del self.ids[:considered], self.ds[:considered], self.done[:considered]
        self.cursor = 0
        return page


def padded(page, k):
    ids = np.full(k, EMPTY, np.uint32)
    ds = np.full(k, np.inf, np.float32)
    ids[:len(page)] = [i for i, _ in page]
    ds[:len(page)] = [d for _, d in page]
    return ids, ds


def bfs(adj, n_points, n_start):
    total = n_points + n_start
    seen, todo = set(range(n_points, total)), list(range(n_points, total))
    while todo:
        u = todo.pop()
        for v in adj[u, 1:1 + adj[u, 0]].tolist():
            if v < total and v not in seen:
                seen.add(v)
                todo.append(v)
    return seen - set(range(n_points, total))


def built(n, d, dt, metric, nq, seed, R=16):
    rng = np.random.default_rng(seed)
    base = clustered(rng, n, d)
    if dt == np.int8:
        base = np.clip(np.round(base * 30), -127, 127)
    elif dt == np.uint8:
        base = np.clip(np.round(base * 30 + 128), 0, 255)
    base = base.astype(dt)
    vecs = np.concatenate([base, base[:1]])
    adj = O.build_graph(vecs, n, 1, metric, R, int(R * 1.3), 30)
    qs = base[rng.integers(0, n, nq)].astype(np.float32)
    if dt in (np.float32, np.float16):
        qs = qs + np.float32(0.05) * rng.normal(size=qs.shape).astype(np.float32)
    return vecs, adj, n, 1, metric, qs.astype(dt)


# ---------------------------------------------------------------- CPU

def baselines():
    return json.load(open(os.path.join(GOLDEN, "paged_search.json")))["cases"]


def test_restatement_reproduces_the_reference_baselines():
    cases = baselines()
    assert [c["case"] for c in cases] == ["basic_paged_search", "single_page", "small_page_size"]
    for c in cases:
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        s = PyPaged(data, adj, n, 1, O.L2, np.array(c["query"], np.float32), c["search_l"])
        pages = []
        while True:
            page = s.next_page(c["page_size"])
            if not page:
                break
            pages.append([[int(i), float(d)] for i, d in page])
            if c["case"] == "single_page":
                break
        assert pages == c["pages"], c["case"]
        assert sum(len(p) for p in pages) == c["total_results"]
        if c["case"] == "single_page":  # exhausted: every later call is empty
            assert s.next_page(c["page_size"]) == [] and s.next_page(c["page_size"]) == []


@pytest.mark.parametrize("L,ks", [(20, (10, 1, 7, 20)), (50, (50,)), (8, (3,))])
def test_pages_are_disjoint_sorted_and_reach_every_reachable_node(L, ks):
    vecs, adj, n, n_start, metric, qs = built(600, 12, np.float32, O.L2, 3, seed=L)
    reach = bfs(adj, n, n_start)
    for q in qs:
        s = PyPaged(vecs, adj, n, n_start, metric, q, L)
        seen, j = [], 0
        while True:
            k = ks[j % len(ks)]
            j += 1
            page = s.next_page(k)
            if not page:
                break
            assert len(page) <= k
            assert all(a[1] <= b[1] for a, b in zip(page, page[1:]))
            seen += [i for i, _ in page]
        assert len(seen) == len(set(seen)) and set(seen) == reach
        assert s.next_page(ks[0]) == [] and s.next_page(1) == []


def test_page_size_bounds():
    vecs, adj, n, n_start, metric, qs = built(200, 8, np.float32, O.L2, 1, seed=1)
    s = PyPaged(vecs, adj, n, n_start, metric, qs[0], 10)
    for k in (0, 11):
        with pytest.raises(ValueError):
            s.next_page(k)
    assert len(s.next_page(10)) == 10


# ---------------------------------------------------------------- GPU

def device_pages(g, queries, L, ks, until_empty=False, max_pages=None):
    out = []
    with g.paged_search(queries, L) as s:
        j = 0
        while True:
            k = ks[j % len(ks)]
            j += 1
            r = s.next_page(k)
            out.append((k,) + r)
            if (until_empty and not r[2].any()) or (not until_empty and j == len(ks)) or (max_pages and j >= max_pages):
                break
    return out


def check_against_restatement(case, got, L, sample):
    vecs, adj, n, n_start, metric, qs = case
    for qi in sample:
        s = PyPaged(vecs, adj, n, n_start, metric, qs[qi], L)
        for k, ids, dists, counts, cmps, hops in got:
            page = s.next_page(k)
            wi, wd = padded(page, k)
            assert np.array_equal(ids[qi], wi), (qi, k)
            assert np.array_equal(dists[qi].view(np.uint32), wd.view(np.uint32)), (qi, k)
            assert (int(counts[qi]), int(cmps[qi]), int(hops[qi])) == (len(page), s.cmps, s.hops), (qi, k)


def gpu_index(case):
    vecs, adj, n, n_start, metric, _ = case
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, adj.shape[1] - 1)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


@pytest.mark.gpu
def test_device_reproduces_the_reference_baselines():
    for c in baselines():
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, c["grid_dims"], n, 1, adj.shape[1] - 1) as g:
            g.upload_vectors(data)
            g.upload_graph(adj)
            pages = []
            with g.paged_search(np.array([c["query"]], np.float32), c["search_l"]) as s:
                for _ in range(3 if c["case"] == "single_page" else 1000):
                    ids, dists, counts, _, _ = s.next_page(c["page_size"])
                    pages.append([[int(i), float(d)] for i, d in zip(ids[0][:counts[0]], dists[0][:counts[0]])])
                    if not counts[0]:
                        break
            assert pages[-1] == [] and pages[:-1] == c["pages"], c["case"]
            want = np.array([d for p in c["pages"] for _, d in p], np.float32)
            got = np.array([d for p in pages for _, d in p], np.float32)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


ROW_TYPES = [(np.float32, O.L2), (np.float32, O.COSINE), (np.float16, O.INNER_PRODUCT), (np.int8, O.L2), (np.uint8, O.COSINE_NORMALIZED)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", ROW_TYPES)
def test_device_equals_restatement_after_every_page(dt, metric):
    # a few thousand queries: the persistent grid takes several rounds; the restatement checks a sample
    case = built(3000, 24, dt, metric, 6000, seed=7)
    L = 40
    with gpu_index(case) as g:
        got = device_pages(g, case[5], L, (10, 1, 37, L, 10, 25))
    check_against_restatement(case, got, L, range(0, 6000, 500))


@pytest.mark.gpu
def test_device_pages_to_exhaustion():
    case = built(400, 16, np.float32, O.L2, 8, seed=3)
    L = 30
    with gpu_index(case) as g:
        got = device_pages(g, case[5], L, (10, 1, L), until_empty=True)
    assert not got[-1][3].any()
    check_against_restatement(case, got, L, range(8))
    reach = bfs(case[1], case[2], case[3])
    for qi in range(8):
        ids = np.concatenate([p[1][qi][:p[3][qi]] for p in got])
        assert len(set(ids.tolist())) == len(ids) and set(ids.tolist()) == reach


@pytest.mark.gpu
@pytest.mark.parametrize("n_start", [1, 7, 300])
def test_many_start_points(n_start):
    c = tie_grid(1500, 6, n_start, 64, seed=n_start)
    case = (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)
    L = 60
    with gpu_index(case) as g:
        got = device_pages(g, c.queries, L, (10, 1, 37, L, 7))
    check_against_restatement(case, got, L, range(0, 64, 4))


@pytest.mark.gpu
def test_malformed_rows_and_edges_into_start_points():
    c = malformed_case(1200, 8, 3, 20, 48, seed=5)
    case = (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)
    L = 30
    with gpu_index(case) as g:
        got = device_pages(g, c.queries, L, (10, 1, 30, 5), until_empty=True, max_pages=60)
    check_against_restatement(case, got, L, range(0, 48, 6))


@pytest.mark.gpu
def test_zero_rows_under_inner_product():
    # the inner product of a zero row is -0.0: it ties +0.0 and keeps its insertion order
    rng = np.random.default_rng(11)
    base = clustered(rng, 800, 8)
    base[::3] = 0
    vecs = np.concatenate([base, base[1:2]]).astype(np.float32)
    adj = O.build_graph(vecs, 800, 1, O.INNER_PRODUCT, 12, 15, 30)
    qs = np.concatenate([np.zeros((4, 8), np.float32), base[rng.integers(0, 800, 12)]])
    qs[4:, ::2] = 0
    case = (vecs, adj, 800, 1, O.INNER_PRODUCT, qs)
    with gpu_index(case) as g:
        got = device_pages(g, qs, 25, (10, 25, 3), until_empty=True, max_pages=80)
    check_against_restatement(case, got, 25, range(16))


@pytest.mark.gpu
def test_visited_overflow_in_the_middle_of_a_session(monkeypatch):
    case = built(2000, 16, np.float32, O.L2, 500, seed=9)
    L, ks = 50, (10, 1, 37, 50, 50, 50)
    with gpu_index(case) as g:
        want = device_pages(g, case[5], L, ks)
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")  # 256-slot tables: every query overflows, page after page
    with gpu_index(case) as g:
        got = device_pages(g, case[5], L, ks)
    for a, b in zip(got, want):
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))
    check_against_restatement(case, got, L, range(0, 500, 50))


@pytest.mark.gpu
def test_interleaved_sessions_and_invalidation():
    case = built(1000, 16, np.float32, O.L2, 64, seed=13)
    qa, qb = case[5][:40], case[5][20:]
    with gpu_index(case) as g:
        alone_a = device_pages(g, qa, 30, (10, 5, 30))
        alone_b = device_pages(g, qb, 20, (7, 20, 1))
        sa, sb = g.paged_search(qa, 30), g.paged_search(qb, 20)
        mixed_a, mixed_b = [], []
        for ka, kb in zip((10, 5, 30), (7, 20, 1)):
            mixed_b.append((kb,) + sb.next_page(kb))
            mixed_a.append((ka,) + sa.next_page(ka))
        for got, want in ((mixed_a, alone_a), (mixed_b, alone_b)):
            for a, b in zip(got, want):
                for x, y in zip(a[1:], b[1:]):
                    assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))
        for k in (0, 31):
            with pytest.raises(dab.DabError) as e:
                sa.next_page(k)
            assert e.value.code == 1
        g.upload_graph(case[1])  # the index changed: both sessions fail cleanly, a new one works
        for s in (sa, sb):
            with pytest.raises(dab.DabError) as e:
                s.next_page(5)
            assert e.value.code == 1 and "index changed" in str(e.value)
        sa.close()
        with g.paged_search(qa, 30) as s:
            assert s.next_page(10)[2].all()
    # sb was still open when the index closed: dab_destroy released it
    with pytest.raises(dab.DabError):
        sb.next_page(5)
