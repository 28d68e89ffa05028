"""Every graph update at the benchmark's graph shape: R = 64, max_degree 83, l_build 100 (bench.py WORKLOADS), held to the
oracles the smaller suites pin, bit for bit.

At R = 64 a prune writes rows of 33-64 ids and a back-edge target holds up to 83, so the lane-strided loops of
prune_pools_kernel, backedge_segments, consolidate_kernel and the in-place delete kernels run more than once per row.  The
default build schedule passes 1024 members a batch once n > 16384.  A hub can receive more in-edges in one batch than the
1024 slots of backedge_segments' pool: the pool is then sorted by (distance, arrival) and cut to 750 while it streams.
l_build past 127 runs search_kernel_v2's wider merge tiles and longer visited records, and an insert search that expands
more than 2048 nodes has its record cut.
Each case asserts that it reaches the edge it is there for, and compares every downloaded row (or the whole prune output)
with its oracle."""
import ctypes as C
import functools

import numpy as np
import pytest

import inplace_delete_oracle as D
import oracle_lib as O
from insert_oracle import insert_batched
from test_delete_consolidate import check_consolidate
from test_graph_stats import prune_range
from test_insert import build_schedule

R, MAXDEG, LB = 64, 83, 100           # bench.py: R = 64, max_degree int(1.3 R), l_build 100
BACKEDGE_SLOTS = 1024                 # launch_backedges' pool at max_degree 83: max(1024, pow2 >= 85)
CONSOLIDATE_SLOTS = 1024              # kConsolidateP
MAX_OCCLUSION = 750                   # graph/config/defaults.rs:13
INT_SCALE = 25.0                      # bench.py's i8 rows


def rec_cap(l_build):
    """the nodes an insert search records (LinkStep::alloc)"""
    return min(2048, 4 * l_build + 64)


def v2_tile(cap):
    """search_kernel_v2's merge tile for a list of cap = L + #start entries (v2_prepare_schema): QT 4 holds 128 entries,
    QT 8 holds 256, and longer lists run the chunked merge of any length (QT 0)"""
    return 4 if cap <= 128 else 8 if cap <= 256 else 0


# ---------------------------------------------------------------- data

def bench_rows(rng, n, d, kind, centers=64):
    """bench.py's make_data: centre ~ N(0, I), point = centre + 0.3 N(0, I); f16 rows unit-normalised, i8 rows scaled by
    25, rounded and clipped; u8 rows the same around 128"""
    c = rng.standard_normal((centers, d), dtype=np.float32)
    x = c[rng.integers(0, centers, n)] + np.float32(0.3) * rng.standard_normal((n, d), dtype=np.float32)
    if kind == "f16":
        x /= np.maximum(np.sqrt((x * x).sum(1, dtype=np.float32, keepdims=True)), np.float32(1e-12))
        return x.astype(np.float16)
    if kind == "i8":
        return np.clip(np.rint(x * np.float32(INT_SCALE)), -127, 127).astype(np.int8)
    if kind == "u8":
        return np.clip(np.rint(x * np.float32(INT_SCALE) + 128), 0, 255).astype(np.uint8)
    return x


def with_medoid(base):
    f = base.astype(np.float32)
    return np.concatenate([base, base[np.argmin(((f - f.mean(0)) ** 2).sum(1))][None]])


SCHEMAS = {  # name: (rows, metric, dim)
    "f32-l2-128": ("f32", O.L2, 128),
    "f32-l2-96": ("f32", O.L2, 96),
    "f16-ip-768": ("f16", O.INNER_PRODUCT, 768),
    "i8-l2-128": ("i8", O.L2, 128),
    "f32-cosine-64": ("f32", O.COSINE, 64),   # the two-accumulator float cosine schema (NA = 2)
    "u8-cosine-64": ("u8", O.COSINE, 64),
}


@functools.lru_cache(maxsize=None)
def schema_rows(name, n):
    kind, metric, d = SCHEMAS[name]
    return with_medoid(bench_rows(np.random.default_rng(list(SCHEMAS).index(name) * 100003 + n), n, d, kind)), metric


@functools.lru_cache(maxsize=None)
def oracle_build(name, n, batch_size):
    """(vecs, metric, adjacency) of the oracle's build at R = 64, shared by the tests of this module"""
    vecs, metric = schema_rows(name, n)
    if batch_size == 1:
        return vecs, metric, O.build_graph(vecs, n, 1, metric, R, MAXDEG, LB)
    return vecs, metric, O.build_graph_batched(vecs, n, 1, metric, R, MAXDEG, LB, batch_size=batch_size)


def degrees(adj):
    return adj[:, 0].astype(np.int64)


def assert_long_rows(adj, what):
    """the rows run every lane-strided loop more than once: some longer than a warp, some at max_degree"""
    deg = degrees(adj)
    assert (deg > 32).sum() > 0 and (deg == MAXDEG).sum() > 0, (what, int(deg.max()), int((deg > 32).sum()))


def check_graph(got, want, what):
    """degrees and the listed ids of every row"""
    bad = np.flatnonzero(got[:, 0] != want[:, 0])
    assert len(bad) == 0, (what, "degree", bad[:5], got[bad[:1], 0], want[bad[:1], 0])
    for i in range(want.shape[0]):
        k = int(want[i, 0])
        assert np.array_equal(got[i, 1:1 + k], want[i, 1:1 + k]), (what, i, got[i, :1 + k], want[i, :1 + k])


def assert_valid(adj, n_total):
    for i in range(n_total):
        row = adj[i, 1:1 + adj[i, 0]]
        assert adj[i, 0] <= MAXDEG and (row < n_total).all() and i not in row and len(set(row.tolist())) == len(row), i


def in_edges(adj, members, target):
    """member rows that list `target`: each is one in-edge the target received from the chunk of `members`"""
    return sum(int(target in adj[m, 1:1 + adj[m, 0]]) for m in members)


# ---------------------------------------------------------------- hubs

def unit_rows(rng, n, d):
    x = rng.standard_normal((n, d), dtype=np.float32)
    return x / np.sqrt((x * x).sum(1, keepdims=True))


@functools.lru_cache(maxsize=None)
def star(kind, n=12000, d=16, first=8192):
    """(vecs, metric, hub, adjacency over the first `first` ids, the rest in ascending order): id 0 is a hub every other
    point is closer to than to most of its neighbours; the start point is the last row.
      l2:     unit vectors, the hub at the origin;
      i8-tie: rows that permute one multiset of values, the hub at the origin: every row is exactly as far from the hub;
      ip:     unit vectors in a cone around e0 under inner product (the occluding prune), the hub 10 e0."""
    rng = np.random.default_rng({"l2": 1, "i8-tie": 2, "ip": 3}[kind])
    if kind == "l2":
        vecs, metric = unit_rows(rng, n + 1, d), O.L2
        vecs[0] = 0
    elif kind == "i8-tie":
        values = rng.integers(-30, 31, d).astype(np.int8)
        vecs, metric = np.stack([rng.permutation(values) for _ in range(n + 1)]), O.L2
        vecs[0] = 0
    else:
        x = rng.standard_normal((n + 1, d), dtype=np.float32)
        x[:, 0] = np.abs(x[:, 0]) + 2
        vecs, metric = x / np.sqrt((x * x).sum(1, keepdims=True)), O.INNER_PRODUCT
        vecs[0] = 0
        vecs[0, 0] = 10
    adj = np.zeros((n + 1, MAXDEG + 1), np.uint32)
    done = 0
    for b in build_schedule(first):
        adj = insert_batched(vecs, adj, np.arange(done, done + b), n, 1, metric, R, MAXDEG, LB, batch_size=b)
        done += b
    return vecs, metric, 0, adj, np.arange(first, n, dtype=np.uint32)


@functools.lru_cache(maxsize=None)
def star_inserted(kind):
    vecs, metric, hub, adj0, rest = star(kind)
    n = vecs.shape[0] - 1
    return insert_batched(vecs, adj0, rest, n, 1, metric, R, MAXDEG, LB, batch_size=0)


@functools.lru_cache(maxsize=None)
def one_chunk(n_start, n=3000, d=32):
    """n points inserted in one chunk into a graph that holds only its start points: every member's only candidates are
    the start points"""
    rng = np.random.default_rng(40 + n_start)
    vecs = bench_rows(rng, n + n_start, d, "f32")
    adj = insert_batched(vecs, np.zeros((n + n_start, MAXDEG + 1), np.uint32), np.arange(n), n, n_start, O.L2, R, MAXDEG, LB,
                         batch_size=0)
    return vecs, adj


# ---------------------------------------------------------------- CPU: the streamed cut

def streamed_cut(d, slots):
    """backedge_segments' pool: arrivals fill `slots`; a full pool is sorted by (distance, arrival) and cut to 750 before
    the next arrival; at the end one more sort, cut to 750.  Returns the arrival indices kept, in order."""
    keep = np.zeros(0, np.int64)
    for i in range(len(d)):
        if len(keep) == slots:
            keep = keep[np.lexsort((keep, d[keep]))][:MAX_OCCLUSION]
        keep = np.append(keep, i)
    return keep[np.lexsort((keep, d[keep]))][:MAX_OCCLUSION]


def streamed_cut_fast(d, slots):
    """streamed_cut, a slot-full block at a time"""
    keep, i = np.zeros(0, np.int64), 0
    while i < len(d):
        take = min(slots - len(keep), len(d) - i)
        keep = np.concatenate([keep, np.arange(i, i + take)])
        i += take
        if i < len(d):
            keep = keep[np.lexsort((keep, d[keep]))][:MAX_OCCLUSION]
    return keep[np.lexsort((keep, d[keep]))][:MAX_OCCLUSION]


@pytest.mark.parametrize("slots", [1024, 2048])
@pytest.mark.parametrize("values", [3, 40, 0])  # 0: distinct distances
def test_the_streamed_cut_keeps_what_one_stable_sort_keeps(slots, values):
    rng = np.random.default_rng(slots + values)
    n = 5000
    d = (rng.integers(0, values, n) if values else rng.permutation(n)).astype(np.float32)
    for m in range(1, n + 1):
        want = np.argsort(d[:m], kind="stable")[:MAX_OCCLUSION]
        assert np.array_equal(streamed_cut_fast(d[:m], slots), want), m
    for m in (slots, slots + 1, slots + 275, 2 * slots + 1, n):  # the per-arrival model at the lengths that cut
        assert np.array_equal(streamed_cut(d[:m], slots), np.argsort(d[:m], kind="stable")[:MAX_OCCLUSION]), m
    if values:  # ties straddle the cut: the 750th and the 751st entries are equally far
        s = np.sort(d)
        assert s[MAX_OCCLUSION - 1] == s[MAX_OCCLUSION]


def test_the_streamed_cut_with_ties_only_at_the_cut():
    """distinct distances except one value that spans the 750 boundary of every intermediate and the final cut"""
    rng = np.random.default_rng(7)
    for slots in (1024, 2048):
        d = rng.permutation(5000).astype(np.float32)
        d[(d > 700) & (rng.random(5000) < 0.5)] = 700  # about half of the rest tie at 700
        s = np.sort(d)
        assert s[MAX_OCCLUSION - 1] == s[MAX_OCCLUSION] == 700
        for m in range(slots - 2, 5001, 37):
            assert np.array_equal(streamed_cut_fast(d[:m], slots), np.argsort(d[:m], kind="stable")[:MAX_OCCLUSION]), (slots, m)


# ---------------------------------------------------------------- CPU: the oracle side reaches the edges

def test_the_oracle_graphs_have_rows_past_a_warp_and_at_max_degree():
    for name in ("f32-l2-128", "i8-l2-128"):
        vecs, metric, adj = oracle_build(name, 20000, 0)
        assert_long_rows(adj, name)
    assert max(build_schedule(20000)) == 1250 > BACKEDGE_SLOTS
    assert max(build_schedule(20000, 4096)) > 2 * BACKEDGE_SLOTS


@pytest.mark.parametrize("n_start", [1, 2])
def test_one_chunk_sends_every_member_to_the_start_points(n_start):
    n = 3000
    vecs, adj = one_chunk(n_start)
    members = np.arange(n)
    for m in members:  # a member's only candidates were the start points, and no back-edge reaches a member
        row = adj[m, 1:1 + adj[m, 0]]
        assert len(row) >= 1 and (row >= n).all(), m
    counts = [in_edges(adj, members, n + s) for s in range(n_start)]
    assert sum(counts) >= n and max(counts) > BACKEDGE_SLOTS + 2 * (BACKEDGE_SLOTS - MAX_OCCLUSION), counts  # cut 3 times


@pytest.mark.parametrize("kind", ["l2", "i8-tie", "ip"])
def test_the_stars_send_more_than_the_pool_to_the_hub(kind):
    vecs, metric, hub, adj0, rest = star(kind)
    adj = star_inserted(kind)
    assert in_edges(adj, rest, hub) > BACKEDGE_SLOTS, kind
    if kind == "i8-tie":  # every member is exactly as far from the hub: arrival order decides the cut
        assert len(np.unique(O.distance_rows(vecs[hub], vecs[rest], metric))) == 1


# ---------------------------------------------------------------- GPU

gpu = pytest.mark.gpu


def device_index(vecs, metric, n, n_start=1):
    import diskann_b200 as dab
    return dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, MAXDEG)


# ---- B: dab_build at the benchmark's shape

@gpu
@pytest.mark.parametrize("batch_size", [0, 4096])
@pytest.mark.parametrize("name", list(SCHEMAS))
def test_device_build_at_r64_is_the_oracle_build(name, batch_size):
    n = 20000
    vecs, metric, want = oracle_build(name, n, batch_size)
    assert_long_rows(want, name)
    assert max(build_schedule(n, batch_size)) > BACKEDGE_SLOTS
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.build(R, LB, 1.2, batch_size=batch_size)
        check_graph(g.download_graph(), want, (name, batch_size))


@gpu
def test_device_build_one_point_at_a_time_at_r64():
    n = 2000
    vecs, metric, want = oracle_build("f32-l2-96", n, 1)
    assert_long_rows(want, "batch_size 1")
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.build(R, LB, 1.2, batch_size=1)
        check_graph(g.download_graph(), want, "batch_size 1")


# ---- C: long build lists

@functools.lru_cache(maxsize=None)
def long_list_build(l_build, n=3000, d=64):
    vecs = with_medoid(bench_rows(np.random.default_rng(l_build), n, d, "f32", centers=16))
    return vecs, O.build_graph_batched(vecs, n, 1, O.L2, R, MAXDEG, l_build)


@gpu
@pytest.mark.parametrize("l_build", [200, 400, 1000])
def test_device_build_with_long_lists(l_build):
    n = 3000
    vecs, want = long_list_build(l_build)
    assert_long_rows(want, l_build)
    assert v2_tile(l_build + 1) == {200: 8, 400: 0, 1000: 0}[l_build]
    assert rec_cap(l_build) == {200: 864, 400: 1664, 1000: 2048}[l_build]
    if l_build == 1000:  # searches expand more nodes than a prune pool keeps
        hops = O.Index(vecs, want, n, 1, O.L2).search_batch(vecs[:n:10], 1, l_build, threads=8)[4]
        assert hops.max() > MAX_OCCLUSION, hops.max()
    with device_index(vecs, O.L2, n) as g:
        g.upload_vectors(vecs)
        g.build(R, l_build, 1.2)
        check_graph(g.download_graph(), want, l_build)


@gpu
def test_device_build_reports_cut_records():
    import diskann_b200 as dab
    n, l_build = 3000, 2100
    vecs, adj400 = long_list_build(400)
    assert rec_cap(l_build) == 2048
    hops = O.Index(vecs, adj400, n, 1, O.L2).search_batch(vecs[:n:10], 1, l_build, threads=8)[4]
    assert hops.max() > 2048, hops.max()  # on a graph over these points, searches outgrow the record
    with device_index(vecs, O.L2, n) as g:
        g.upload_vectors(vecs)
        with pytest.raises(dab.DabError) as e:
            g.build(R, l_build, 1.2)
        assert e.value.code == 1 and "prune pools were cut" in str(e.value) and "dab_build" in str(e.value), str(e.value)
        adj = g.download_graph()
    assert_valid(adj, n + 1)
    assert degrees(adj)[:n].min() >= 1


# ---- D: hubs past the back-edge pool

@gpu
@pytest.mark.parametrize("n_start", [1, 2])
def test_device_insert_of_one_chunk_into_the_start_points(n_start):
    n = 3000
    vecs, want = one_chunk(n_start)
    assert max(in_edges(want, np.arange(n), n + s) for s in range(n_start)) > BACKEDGE_SLOTS
    with device_index(vecs, O.L2, n, n_start) as g:
        g.upload_vectors(vecs)  # no graph: it starts empty
        g.insert(np.arange(n, dtype=np.uint32), vecs[:n], R, LB)
        check_graph(g.download_graph(), want, n_start)


@gpu
@pytest.mark.parametrize("kind", ["l2", "i8-tie", "ip"])
def test_device_insert_of_a_chunk_into_a_star(kind):
    vecs, metric, hub, adj0, rest = star(kind)
    n = vecs.shape[0] - 1
    want = star_inserted(kind)
    assert in_edges(want, rest, hub) > BACKEDGE_SLOTS
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.insert(rest, vecs[rest], R, LB)
        check_graph(g.download_graph(), want, kind)


# ---- E: the other updates on an R = 64 graph the oracle built

def graph_3000():
    return oracle_build("f32-l2-96", 3000, 0)


@gpu
@pytest.mark.parametrize("batch_size", [64, 0])
def test_device_insert_of_live_and_released_rows(batch_size):
    n = 3000
    vecs, metric, adj0 = graph_3000()
    assert_long_rows(adj0, "graph")
    rng = np.random.default_rng(batch_size + 1)
    ids = rng.choice(n, n // 10, replace=False).astype(np.uint32)
    released = ids[::2]
    new = vecs.copy()
    new[ids] = bench_rows(rng, len(ids), vecs.shape[1], "f32")
    start = adj0.copy()
    start[released, 0] = 0
    want = insert_batched(new, start, ids, n, 1, metric, R, MAXDEG, LB, batch_size=batch_size)
    assert_long_rows(want, "inserted")
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        g.delete(released)
        g.release(released)
        g.insert(ids, new[ids], R, LB, batch_size=batch_size)
        check_graph(g.download_graph(), want, batch_size)


def consolidate_pool(adj, deleted, v, n):
    """the distinct live ids consolidate_vector(v) gathers (test_delete_consolidate.consolidate_node's pool)"""
    row = lambda u: [int(x) for x in adj[u, 1:1 + adj[u, 0]]]
    dead = lambda u: u >= adj.shape[0] or (u < n and deleted[u])
    pool = {u for u in row(v) if not dead(u)}
    for u in row(v):
        if dead(u) and u < adj.shape[0]:
            pool.update(w for w in row(u) if not dead(w))
    pool.discard(v)
    return len(pool)


@gpu
@pytest.mark.parametrize("frac", [0.1, 0.5, "hub"])
def test_device_consolidate_at_r64(frac):
    n = 3000
    vecs, metric, adj0 = graph_3000()
    rng = np.random.default_rng(5)
    deleted = np.zeros(n, bool)
    if frac == "hub":  # every neighbour of a full row deleted: their lists bring more candidates than the pool holds
        v = int(np.flatnonzero(degrees(adj0)[:n] == MAXDEG)[0])
        nb = adj0[v, 1:1 + MAXDEG]
        deleted[nb[nb < n]] = True
        deleted[rng.choice(n, n // 20, replace=False)] = True
        deleted[v] = False
        assert consolidate_pool(adj0, deleted, v, n) > CONSOLIDATE_SLOTS
    else:
        deleted[rng.choice(n, int(frac * n), replace=False)] = True
    assert_long_rows(adj0, frac)
    got = check_consolidate(vecs, adj0, n, 1, metric, deleted, R)
    assert (degrees(got) > 32).any()


@gpu
@pytest.mark.parametrize("method", ["visited_and_topk", "two_hop_and_one_hop", "one_hop"])
def test_device_inplace_delete_at_r64(method):
    n = 3000
    vecs, metric, adj0 = graph_3000()
    m = {"visited_and_topk": D.VISITED_AND_TOPK, "two_hop_and_one_hop": D.TWO_HOP_AND_ONE_HOP, "one_hop": D.ONE_HOP}[method]
    rng = np.random.default_rng(m)
    for batch_size in (1, 37, 0):
        ids = rng.choice(n, n // 10, replace=False).astype(np.uint32)
        pre = ids[:30]  # already soft-deleted
        # the deleted ids' lists and the lists that name them run past one warp
        assert (degrees(adj0)[ids] > 32).any()
        assert any(adj0[u, 0] == MAXDEG and np.isin(adj0[u, 1:1 + MAXDEG], ids).any() for u in range(n + 1))
        want_adj, want_del = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1, pre), ids, n, 1, metric, m, 3, R,
                                              batch_size=batch_size)
        with device_index(vecs, metric, n) as g:
            g.upload_vectors(vecs)
            g.upload_graph(adj0)
            g.delete(pre)
            g.inplace_delete(ids, 3, method, R, batch_size=batch_size)
            got = g.download_graph()
            status = g.delete_status(np.arange(n, dtype=np.uint32))
        check_graph(got, want_adj, (method, batch_size))
        assert np.array_equal(np.flatnonzero(status).astype(np.uint32), D.deleted_ids(want_del, n + 1))


@gpu
@pytest.mark.parametrize("only_orphans", [False, True])
def test_device_drop_deleted_neighbors_at_r64(only_orphans):
    n = 3000
    vecs, metric, adj0 = graph_3000()
    rng = np.random.default_rng(11)
    ids = rng.choice(n, n // 10, replace=False)
    adj = adj0.copy()
    adj[ids[::2], 0] = 0  # half of them with their lists dropped (orphans), the rest soft-deleted only
    words = D.deleted_words(n + 1, ids)
    want, want_n = D.drop_deleted_neighbors(adj, words, n, 1, R, only_orphans)
    written = (want != adj).any(1)
    assert want_n > 0 and (degrees(adj)[written] > 32).any() and (degrees(want) < degrees(adj)).any()
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        g.delete(ids)
        got_n = g.drop_deleted_neighbors(R, only_orphans)
        check_graph(g.download_graph(), want, only_orphans)
    assert got_n == want_n


@gpu
def test_device_prune_range_to_40():
    n = 3000
    vecs, metric, adj0 = graph_3000()
    want, want_n = prune_range(vecs, adj0, n, 1, metric, range(n + 1), 40)
    assert want_n == (degrees(adj0) > 40).sum() > 0 and (degrees(want) > 32).any()
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        assert g.prune_range(None, 40) == want_n
        check_graph(g.download_graph(), want, "prune_range")


def prune_pools(rng, vecs, metric, n, n_pools, cap):
    pool_ids = np.full((n_pools, cap), 0xFFFFFFFF, np.uint32)
    pool_d = np.zeros((n_pools, cap), np.float32)
    lens = rng.integers(MAX_OCCLUSION + 1, cap + 1, n_pools).astype(np.uint32)
    lens[:4] = [0, 1, MAX_OCCLUSION, cap]
    locs = rng.integers(0, n, n_pools).astype(np.uint32)
    for p in range(n_pools):
        ids = rng.choice(n, lens[p], replace=False).astype(np.uint32)
        if lens[p] > 3:
            ids[2] = locs[p]
        pool_ids[p, :lens[p]] = ids
        pool_d[p, :lens[p]] = O.distance_rows(vecs[locs[p]], vecs[ids], metric) if lens[p] else []
    pool_d[:, ::7] = np.round(pool_d[:, ::7])  # exact ties across the sort
    return pool_ids, pool_d, lens, locs


@gpu
def test_device_robust_prune_of_pools_past_750():
    n = 3000
    vecs, metric, _ = graph_3000()
    rng = np.random.default_rng(13)
    cap, degree = 2048, R
    pool_ids, pool_d, lens, locs = prune_pools(rng, vecs, metric, n, 64, cap)
    assert (lens > MAX_OCCLUSION).sum() > 32 and lens.max() == cap
    oidx = O.Index(vecs, np.zeros((n + 1, 2), np.uint32), n, 1, metric)
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        got, counts = g.robust_prune(pool_ids, pool_d, lens, locs, degree, 1.2)
    for p in range(len(lens)):
        m = int(lens[p])
        order = np.argsort(pool_d[p, :m], kind="stable")[:MAX_OCCLUSION]
        sid, sd = np.ascontiguousarray(pool_ids[p, :m][order]), np.ascontiguousarray(pool_d[p, :m][order])
        excl = np.ascontiguousarray((sid == locs[p]).astype(np.uint8))
        pos = np.zeros(degree, np.uint32)
        found = O.lib().orc_robust_prune(C.byref(oidx.c), O.ptr(sid), O.ptr(sd), O.ptr(excl), len(sid), degree, 1.2, O.SIMD,
                                         O.ptr(pos), None)
        assert counts[p] == found, p
        assert np.array_equal(got[p, :found], sid[pos[:found]]), p
        assert (got[p, found:] == 0xFFFFFFFF).all(), p
    assert (counts > 32).any(), counts.max()


# ---- F: the pool capacity dab_robust_prune accepts

@gpu
def test_device_robust_prune_refuses_pools_past_2048():
    import diskann_b200 as dab
    n = 3000
    vecs, metric, adj0 = graph_3000()
    rng = np.random.default_rng(17)
    pool_ids, pool_d, lens, locs = prune_pools(rng, vecs, metric, n, 4, 2049)
    out = np.full((4, R), 0xABCD, np.uint32)
    counts = np.full(4, 0xABCD, np.uint32)
    with device_index(vecs, metric, n) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj0)
        rc = dab.lib().dab_robust_prune(g._h, O.ptr(pool_ids), O.ptr(pool_d), O.ptr(lens), O.ptr(locs), 4, 2049, R, 1.2,
                                        O.ptr(out), O.ptr(counts))
        assert rc == 1 and b"pool_cap in [1, 2048]" in dab.lib().dab_last_error()
        assert (out == 0xABCD).all() and (counts == 0xABCD).all()
        assert np.array_equal(g.download_graph(), adj0)
        got, got_n = g.robust_prune(pool_ids[:, :2048], pool_d[:, :2048], np.minimum(lens, 2048), locs, R, 1.2)
        assert got_n[0] == 0 and (got_n[1:] > 0).all()
