"""Diversity-aware search (Diverse::search, diskann/src/graph/search/diverse_search.rs:189-234), CPU side: the oracle
(oracle/diverse_search.cpp) pinned by restatements of the reference's own DiverseNeighborQueue tests
(neighbor/diverse_priority_queue.rs:338-836) and NeighborPriorityQueue remove / retain / truncate tests
(neighbor/queue.rs:1112-1473), by a Python restatement of Diverse::search on built graphs and on graphs with exact
ties (where removals fail and the local queues drift from the list), by the k-NN oracle when every id has an attribute
of its own, and by the properties of the providers' diversity search test (diskann_async.rs:2871-3074)."""
import numpy as np
import pytest

import diverse_oracle as D
import oracle_lib as O
from test_traversal_edges import grid, many_starts

EMPTY = 0xFFFFFFFF


def provider():
    """create_test_attribute_provider: ids 0..19 have attribute id / 3"""
    return {i: i // 3 for i in range(20)}


# ---------------------------------------------------------------- DiverseNeighborQueue (diverse_priority_queue.rs:338-836)

def test_new():
    q = D.DiverseQueue(10, 5, 5, provider())
    assert q.size() == 0 and q.capacity() == 10 and q.search_l() == 10 and q.diverse_results_l() == 10


def test_insert_single_attribute():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5)):
        q.insert(i, d)
    assert q.size() == 3 and q.n_local() == 1 and q.local_size(0) is not None


def test_insert_multiple_attributes():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (3, 0.8), (6, 1.2)):
        q.insert(i, d)
    assert q.size() == 3 and q.n_local() == 3
    assert all(q.local_size(a) is not None for a in (0, 1, 2))


def test_insert_maintains_order():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5)):
        q.insert(i, d)
    assert [q.get(n)[0] for n in range(3)] == [1, 0, 2]


def test_insert_local_queue_full():
    q = D.DiverseQueue(20, 20, 3, {i: 0 for i in range(10, 16)})  # diverse_results_l = 3 * 20 / 20 = 3
    for i, d in ((10, 1.0), (11, 0.8), (12, 1.2)):
        q.insert(i, d)
    assert q.size() == 3 and q.local_size(0) == 3
    q.insert(13, 0.5)
    assert q.size() == 3 and q.get(0)[0] == 13


def test_insert_inner_queue_full():
    q = D.DiverseQueue(3, 5, 5, provider())
    for i, d in ((0, 1.0), (3, 0.8), (6, 1.2)):
        q.insert(i, d)
    assert q.size() == 3
    q.insert(9, 0.5)
    assert q.size() == 3 and q.get(0)[0] == 9


def test_get():
    q = D.DiverseQueue(10, 5, 5, provider())
    q.insert(0, 1.0)
    q.insert(1, 0.5)
    assert q.get(0) == (1, 0.5) and q.get(1) == (0, 1.0)


def test_closest_notvisited():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5)):
        q.insert(i, d)
    assert q.has_notvisited_node()
    assert q.closest_notvisited() == (1, 0.5)
    assert q.has_notvisited_node()
    assert q.closest_notvisited()[0] == 0
    assert q.closest_notvisited()[0] == 2
    assert not q.has_notvisited_node() and q.closest_notvisited() is None


def test_has_notvisited_node():
    q = D.DiverseQueue(10, 5, 5, provider())
    assert not q.has_notvisited_node()
    q.insert(0, 1.0)
    assert q.has_notvisited_node()
    assert q.closest_notvisited() is not None
    assert not q.has_notvisited_node() and q.closest_notvisited() is None


def test_size():
    q = D.DiverseQueue(10, 5, 5, provider())
    assert q.size() == 0
    q.insert(0, 1.0)
    assert q.size() == 1
    q.insert(1, 0.5)
    assert q.size() == 2


def test_capacity():
    assert D.DiverseQueue(15, 5, 5, provider()).capacity() == 15


def test_search_l():
    assert D.DiverseQueue(20, 5, 5, provider()).search_l() == 20


def test_clear():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (3, 0.5), (6, 1.5)):
        q.insert(i, d)
    assert q.size() == 3 and q.n_local() == 3
    q.clear()
    assert q.size() == 0 and q.n_local() == 0


def test_iter_candidates():
    q = D.DiverseQueue(10, 5, 5, provider())
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5)):
        q.insert(i, d)
    assert [i for i, _ in q.iter()] == [1, 0, 2]


def test_inner_and_inner_mut():
    q = D.DiverseQueue(10, 5, 5, provider())
    q.insert(0, 1.0)
    assert q.size() == 1
    q.clear()
    assert q.size() == 0


def test_vector_id_with_attribute():
    """the global queue's entry carries (id, attribute): id 42 with attribute 7 is listed and opens attribute 7's queue"""
    q = D.DiverseQueue(10, 5, 5, {42: 7})
    q.insert(42, 1.0)
    assert q.get(0)[0] == 42 and q.local_size(7) == 1 and q.local_get(7, 0)[0] == 42


def test_attribute_value_provider():
    """get is None for an id never inserted, else its latest value (a later insert replaces the value)"""
    attrs = {}
    assert D.DiverseQueue(10, 5, 5, attrs).n_local() == 0
    q = D.DiverseQueue(10, 5, 5, {0: 10})
    q.insert(1, 1.0)  # no value: skipped
    q.insert(0, 1.0)
    assert q.size() == 1 and q.local_size(10) == 1
    attrs = {0: 10, 5: 20}
    attrs[0] = 15
    q = D.DiverseQueue(10, 5, 5, attrs)
    q.insert(0, 1.0)
    q.insert(5, 2.0)
    assert q.local_size(15) == 1 and q.local_size(20) == 1 and q.local_size(10) is None


def test_attribute_value_provider_default():
    q = D.DiverseQueue(10, 5, 5, {})
    q.insert(0, 1.0)
    assert q.size() == 0


def test_diverse_queue_complex_scenario():
    q = D.DiverseQueue(10, 5, 3, provider())
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5), (3, 0.8), (4, 1.2), (6, 0.7)):
        q.insert(i, d)
    assert q.size() == 6
    attrs = provider()
    attrs[17] = 0
    q2 = D.DiverseQueue(10, 5, 3, attrs)
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5), (3, 0.8), (4, 1.2), (6, 0.7)):
        q2.insert(i, d)
    q2.insert(17, 0.3)
    assert q2.get(0) == (17, np.float32(0.3))


def test_post_process():
    q = D.DiverseQueue(20, 5, 2, {i: i // 3 for i in range(9)})  # diverse_results_l = 2 * 20 / 5 = 8
    for i, d in ((0, 1.0), (1, 0.5), (2, 1.5), (3, 0.8), (4, 1.2), (5, 0.6), (6, 0.7), (7, 1.1), (8, 0.9)):
        q.insert(i, d)
    assert q.size() == 9 and q.local_size(0) == q.local_size(1) == q.local_size(2) == 3
    q.post_process()
    assert q.local_size(0) == q.local_size(1) == q.local_size(2) == 2
    assert q.size() == 6
    f = np.float32
    assert [q.local_get(0, n) for n in range(2)] == [(1, f(0.5)), (0, f(1.0))]
    assert [q.local_get(1, n) for n in range(2)] == [(5, f(0.6)), (3, f(0.8))]
    assert [q.local_get(2, n) for n in range(2)] == [(6, f(0.7)), (8, f(0.9))]
    assert [q.get(n)[0] for n in range(6)] == [1, 5, 6, 3, 8, 0]


def test_skip_neighbors_without_attributes():
    q = D.DiverseQueue(10, 5, 5, {0: 0, 1: 0, 2: 1, 4: 0})
    for i, d in ((0, 1.0), (1, 0.5), (2, 0.8), (3, 0.3), (4, 1.2)):
        q.insert(i, d)
    assert q.size() == 4, "Expected 4 items, ID 3 should be skipped"
    assert q.local_size(0) == 3 and q.local_size(1) == 1
    ids = [i for i, _ in q.iter()]
    assert 3 not in ids and ids == [1, 2, 0, 4]


def test_attribute_zero_vs_missing_attribute():
    q = D.DiverseQueue(10, 5, 5, {0: 0, 2: 0})
    for i, d in ((0, 1.0), (1, 0.5), (2, 0.8)):
        q.insert(i, d)
    assert q.size() == 2 and q.n_local() == 1 and q.local_size(0) == 2
    assert [i for i, _ in q.iter()] == [2, 0]


# ---------------------------------------------------------------- NeighborPriorityQueue remove / retain / truncate

def filled(pairs, cap=10):
    q = D.Npq(cap)
    for i, d in pairs:
        q.insert(i, d)
    return q


FIVE = ((1, 1.0), (2, 0.5), (3, 1.5), (4, 0.3), (5, 2.0))


def ids_of(q):
    return [e[0] for e in q.entries()]


def test_remove():
    q = D.Npq(10)
    assert not q.remove(1, 1.0)
    for i, d in FIVE:
        q.insert(i, d)
    assert q.size() == 5
    assert q.remove(1, 1.0) and q.size() == 4 and ids_of(q) == [4, 2, 3, 5]
    assert q.remove(4, 0.3) and q.size() == 3 and ids_of(q) == [2, 3, 5]
    assert q.remove(5, 2.0) and q.size() == 2 and ids_of(q) == [2, 3]
    assert not q.remove(99, 0.5) and q.size() == 2
    assert not q.remove(2, 99.0) and q.size() == 2
    assert q.remove(2, 0.5) and q.size() == 1
    assert q.remove(3, 1.5) and q.size() == 0
    assert not q.remove(1, 1.0)


def test_remove_with_cursor():
    q = filled(FIVE[:4])
    assert q.closest_notvisited() is not None and q.closest_notvisited() is not None
    assert q.cursor == 2
    assert q.remove(4, 0.3) and q.cursor == 1 and q.size() == 3
    assert q.remove(1, 1.0) and q.cursor == 1 and q.size() == 2
    assert ids_of(q) == [2, 3]


def test_remove_maintains_sorted_order():
    q = filled(FIVE + ((6, 0.8),))
    q.remove(3, 1.5)
    q.remove(4, 0.3)
    d = [e[1] for e in q.entries()]
    assert d == sorted(d) and ids_of(q) == [2, 6, 1, 5]


def test_remove_at_a_tie_fails():
    """the lower bound of an exactly tied distance is the later insertion: removing the earlier one fails"""
    q = filled(((1, 1.0), (2, 1.0)))
    assert ids_of(q) == [2, 1]
    assert not q.remove(1, 1.0) and q.size() == 2
    assert q.remove(2, 1.0) and q.remove(1, 1.0)


def test_insert_neighbors_with_infinity_distance():
    q = D.Npq(5)
    for i in range(2):
        q.insert(i, np.inf)
    assert q.size() == 2
    for i in range(2, 10):
        q.insert(i, np.inf)
    assert q.size() == 5


def test_normal_distances_should_push_infinity_distances_away_from_queue():
    q = D.Npq(5)
    for i in range(5):
        q.insert(i, np.inf)
    for i in range(5, 8):
        q.insert(i, float(i))
    assert ids_of(q) == [5, 6, 7, 4, 3]


def test_insert_neighbor_with_nan_distance_is_ignored():
    q = D.Npq(5)
    q.insert(0, np.nan)
    assert q.size() == 0


def test_retain():
    q = filled(FIVE + ((6, 0.8),))
    assert q.size() == 6
    q.retain(lambda i, d: d <= 1.0)
    assert ids_of(q) == [4, 2, 6, 1]
    q.retain(lambda i, d: i >= 3)
    assert ids_of(q) == [4, 6]


def test_retain_empty():
    q = D.Npq(10)
    q.retain(lambda i, d: True)
    assert q.size() == 0


def test_retain_remove_all():
    q = filled(FIVE[:3])
    q.retain(lambda i, d: False)
    assert q.size() == 0 and q.cursor == 0


def test_retain_remove_none():
    q = filled(FIVE[:3])
    q.retain(lambda i, d: True)
    assert ids_of(q) == [2, 1, 3]


def test_retain_resets_visited_state():
    q = filled(FIVE[:4])
    assert q.closest_notvisited() is not None and q.closest_notvisited() is not None
    assert q.cursor == 2
    q.retain(lambda i, d: d <= 1.0)
    assert q.size() == 3 and q.cursor == 0 and q.has_notvisited_node()
    assert q.closest_notvisited()[0] == 4 and q.cursor == 1
    assert q.closest_notvisited()[0] == 2 and q.cursor == 2
    assert q.closest_notvisited()[0] == 1 and q.cursor == 3


def test_truncate():
    q = filled(FIVE)
    q.truncate(3)
    assert ids_of(q) == [4, 2, 1]


def test_truncate_larger_size():
    q = filled(FIVE[:2])
    q.truncate(10)
    assert q.size() == 2


def test_truncate_with_cursor():
    q = filled(FIVE[:4])
    q.closest_notvisited(), q.closest_notvisited()
    assert q.cursor == 2
    q.truncate(1)
    assert q.size() == 1 and q.cursor == 0


# ---------------------------------------------------------------- Diverse::search, restated

class PyQueue:
    """NeighborPriorityQueue (queue.rs), fixed capacity; entries [id, distance, visited, payload]"""

    def __init__(self, cap):
        self.cap, self.e, self.cursor = cap, [], 0

    def lower_bound(self, d):
        return next((j for j, x in enumerate(self.e) if x[1] >= d), len(self.e))

    def full(self):
        return len(self.e) == self.cap

    def insert(self, i, d, a=None):
        if np.isnan(d) or (self.full() and self.e[-1][1] < d):
            return
        at = self.lower_bound(d) if self.e else 0
        if self.full():
            del self.e[-1]
        self.e.insert(at, [i, d, False, a])
        self.cursor = min(self.cursor, at)

    def remove(self, i, d):
        if not self.e:
            return False
        at = self.lower_bound(d)
        if at < len(self.e) and self.e[at][0] == i:
            del self.e[at]
            if at < self.cursor and self.cursor > 0:
                self.cursor -= 1
            return True
        return False

    def has_notvisited(self):
        return self.cursor < min(self.cap, len(self.e))

    def closest_notvisited(self):
        cur = self.cursor
        self.e[cur][2] = True
        self.cursor += 1
        while self.cursor < len(self.e) and self.e[self.cursor][2]:
            self.cursor += 1
        return self.e[cur][0]


class PyDiverse:
    """DiverseNeighborQueue (diverse_priority_queue.rs:90-220) over attribute lookups `attr(id)` (None: no attribute)"""

    def __init__(self, L, k, dk, attr):
        self.g, self.local, self.attr, self.dl, self.dk, self.failed = PyQueue(L), {}, attr, dk * L // k, dk, 0

    def insert(self, i, d):
        a = self.attr(i)
        if a is None:
            return
        lq = self.local.setdefault(a, PyQueue(self.dl))
        if not lq.full() and not self.g.full():
            lq.insert(i, d)
            self.g.insert(i, d, a)
        elif lq.full():
            if d < lq.e[self.dl - 1][1]:
                wi, wd = lq.e[self.dl - 1][:2]
                self.failed += not self.g.remove(wi, wd)
                lq.insert(i, d)
                self.g.insert(i, d, a)
        elif d < self.g.e[self.g.cap - 1][1]:
            gi, gd, _, ga = self.g.e[self.g.cap - 1]
            lq.insert(i, d)
            self.g.insert(i, d, a)
            if ga in self.local:
                self.failed += not self.local[ga].remove(gi, gd)

    def post_process(self):
        cut = set()
        for lq in self.local.values():
            if len(lq.e) > self.dk:
                cut |= {x[0] for x in lq.e[self.dk:]}
                del lq.e[self.dk:]
                lq.cursor = 0
        if cut:
            self.g.e = [[x[0], x[1], False, x[3]] for x in self.g.e if x[0] not in cut]
            self.g.cursor = 0


def py_diverse_search(vecs, adj, n, n_start, metric, query, k, L, dk, values, present, beam=1, deleted=None):
    total = n + n_start
    q = np.ascontiguousarray(query.astype(np.float32) if vecs.dtype == np.float16 else query)
    dist = lambda ids: O.distance_rows(q, vecs[ids], metric, O.AVX2)
    best = PyDiverse(L, k, dk, lambda i: int(values[i]) if present[i] else None)
    visited = set(range(n, total))
    for i, d in zip(range(n, total), dist(np.arange(n, total))):
        best.insert(i, d)
    cmps, hops = n_start, 0
    while best.g.has_notvisited():
        nodes = []
        while len(nodes) < beam and best.g.has_notvisited():
            nodes.append(best.g.closest_notvisited())
        fresh = []
        for u in nodes:
            for v in adj[u, 1:1 + adj[u, 0]].tolist():
                if v in visited:
                    continue
                visited.add(v)
                if v < total:
                    fresh.append(v)
        for i, d in zip(fresh, dist(np.array(fresh, np.int64)) if fresh else []):
            best.insert(i, d)
        cmps += len(fresh)
        hops += len(nodes)
    best.post_process()
    out = [(x[0], x[1]) for x in best.g.e[:L] if x[0] < n and not (deleted is not None and deleted[x[0]])][:k]
    ids = np.full(k, EMPTY, np.uint32)
    ds = np.full(k, np.inf, np.float32)
    ids[:len(out)] = [i for i, _ in out]
    ds[:len(out)] = [d for _, d in out]
    return ids, ds, len(out), cmps, hops, best.failed


def same(got, want, what):
    for a, b, name in zip(got, want, ("ids", "dists", "counts", "cmps", "hops")):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), (what, name)


def restated_equals_oracle(case, klbd, values, present, nq=30, deleted=None):
    failed = 0
    for k, L, beam, dk in klbd:
        want = D.search_batch(case.oracle, case.queries[:nq], k, L, dk, values, present, beam=beam, deleted=deleted)
        rows = [py_diverse_search(case.vecs, case.adj, case.n, case.n_start, case.metric, q, k, L, dk, values, present, beam, deleted)
                for q in case.queries[:nq]]
        got = tuple(np.array([r[j] for r in rows]).astype(dt) for j, dt in enumerate((np.uint32, np.float32, np.uint32, np.uint32, np.uint32)))
        same(got, want[:5], (k, L, beam, dk))
        assert [r[5] for r in rows] == want[5].tolist(), "failed removals"
        failed += int(want[5].sum())
    return failed


KLBD = [(10, 10, 1, 1), (10, 30, 1, 3), (5, 40, 4, 2), (10, 50, 2, 12)]


@pytest.mark.parametrize("card", [1, 3, 17])
def test_oracle_equals_restated_search_on_built_graphs(card):
    case = many_starts(500, 8, 3, 30, card)
    rng = np.random.default_rng(card)
    values = rng.integers(0, card, case.total).astype(np.uint32)
    present = (rng.random(case.total) < 0.8).astype(np.uint8)
    restated_equals_oracle(case, KLBD, values, present)
    deleted = np.zeros(case.total, bool)
    deleted[rng.integers(0, case.n, 60)] = True
    restated_equals_oracle(case, KLBD[:2], values, present, deleted=deleted)


@pytest.mark.parametrize("card", [2, 5])
def test_oracle_equals_restated_search_on_exact_ties(card):
    """on the exact-tie grid graphs removals fail at tied distances: the drift path is exercised"""
    case = grid(400, 8, 3, 30, 3)
    values = (np.arange(case.total) % card).astype(np.uint32)
    failed = restated_equals_oracle(case, [(10, 30, 1, 1), (10, 60, 2, 3), (5, 100, 1, 2)], values, np.ones(case.total, np.uint8))
    assert failed > 0, "no removal failed: the drift path was not reached"


def test_distinct_attributes_equal_knn_search():
    """every id its own attribute: no local queue ever fills or drops, so the search is k-NN search over a list of L
    (the k-NN list holds L + #start: l_search = L - #start)"""
    case = many_starts(500, 8, 3, 40, 5)
    values = np.arange(case.total, dtype=np.uint32)
    for k, L, beam in ((10, 13, 1), (10, 43, 2), (7, 103, 4)):
        got = D.search_batch(case.oracle, case.queries, k, L, 1, values, beam=beam)
        same(got[:5], case.oracle.search_batch(case.queries, k, L - case.n_start, beam=beam), (k, L, beam))


def test_start_points_without_attributes_make_no_hop():
    case = many_starts(300, 8, 2, 10, 1)
    present = np.ones(case.total, np.uint8)
    present[case.n:] = 0
    ids, _, counts, cmps, hops, _ = D.search_batch(case.oracle, case.queries, 10, 20, 1, np.zeros(case.total, np.uint32), present)
    assert (counts == 0).all() and (hops == 0).all() and (cmps == case.n_start).all() and (ids == EMPTY).all()


def test_inmemory_search_diversity_search():
    """the properties diskann_async.rs:2871-3074 asserts: 256 x 128 points labelled i % 5 + 1 (start point 1), L = 20,
    k = 10, diverse_k = 1: results sorted, at least one, each label at most once, at least two labels"""
    rng = np.random.default_rng(0)
    n, d = 256, 128
    base = rng.normal(size=(n, d)).astype(np.float32)
    vecs = np.concatenate([base, base.mean(0, keepdims=True)])
    adj = O.build_graph(vecs, n, 1, O.L2, 32, 41, 50)
    index = O.Index(vecs, adj, n, 1, O.L2)
    labels = np.concatenate([np.arange(n) % 5 + 1, [1]]).astype(np.uint32)
    queries = base[:8] + np.float32(0.01) * rng.normal(size=(8, d)).astype(np.float32)
    ids, dists, counts, _, _, _ = D.search_batch(index, queries, 10, 20, 1, labels)
    for q in range(8):
        c = int(counts[q])
        assert c >= 1
        assert (np.diff(dists[q, :c]) >= 0).all()
        got = labels[ids[q, :c]]
        assert len(set(got.tolist())) == c and c >= 2
