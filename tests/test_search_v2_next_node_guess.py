"""search_kernel_v2's next-node guess on the register-row path, against the oracle: bit-identical ids, distance bits,
result counts, cmps and hops.

In flight, f32 rows of 32 / 64 / 96 / 128 elements with level 1 of the visited set on: once a hop has selected its node,
the kernel guesses that the next hop expands the closest unvisited entry left, and copies that entry's adjacency row into
shared memory ahead of time.  A wrong guess may only cost time, never change what a search returns.  The graphs here
are written by hand so that the guess always fails (a new candidate beats it every hop), always holds, holds on rows
full of repeated, out-of-range and aliasing ids, and holds on rows longer than the 96-word adjacency buffer.  Level 1
also closes in the middle of a query while the global table overflows, and beam 2 runs on the same graphs.  Every case
also runs synchronously, on the staged-row path."""

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

FIELDS = ("ids", "dists", "counts", "cmps", "hops")
EMPTY = 0xFFFFFFFF


@pytest.fixture(scope="module")
def dab():
    import diskann_b200
    diskann_b200.lib()
    return diskann_b200


def k_bits(n_total):
    K = 8
    while (1 << K) < n_total:
        K += 1
    return K


def check(dab, vecs, adj, n, queries, cases):
    """in flight (the register path) and synchronously (staged rows), both against the oracle"""
    adj = np.ascontiguousarray(adj, np.uint32)
    maxdeg = adj.shape[1] - 1
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, vecs.shape[1], n, 1, maxdeg) as g:
        g.upload_vectors(vecs)
        g.upload_graph(adj)
        for (L, beam) in cases:
            want = oidx.search_batch(queries, 10, L, beam=beam, threads=4)
            out = g.search_batch_async(0, queries, 10, L, beam)
            g.wait(0)
            for a, b, name in zip(out, want, FIELDS):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), ("in flight", name, L, beam)
            got = g.search_batch(queries, 10, L, beam)
            for a, b, name in zip(got, want, FIELDS):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), ("synchronous", name, L, beam)
    return want


def line(n, dim, side=0.0):
    """n points at x = 0 .. n-1 on the first axis, `side` on the second; the start point is a copy of point 0"""
    base = np.zeros((n, dim), np.float32)
    base[:, 0] = np.arange(n)
    base[:, 1] = side
    return base


def queries_at(rng, x, dim, nq=64):
    q = np.zeros((nq, dim), np.float32)
    q[:, 0] = x + rng.integers(0, 4, nq)
    q[:, 2:] = rng.integers(-2, 3, (nq, dim - 2))
    return q


def always_fails(m, dim, rng):
    """main points 0..m-1 on a line, point i's side point m+i far off it; main i links to i+1 and its side point.  The
    query lies past the line's end, so i+1 (found by hop i) beats every entry already in the list: the guess (the best
    unvisited entry before hop i's merge, a side point) is wrong on every hop of the walk."""
    n = 2 * m
    vecs = np.concatenate([line(m, dim), line(m, dim, side=60.0), np.zeros((1, dim), np.float32)])
    adj = np.zeros((n + 1, 3), np.uint32)
    for i in range(m):
        row = ([i + 1] if i + 1 < m else []) + [m + i]
        adj[i, 0], adj[i, 1:1 + len(row)] = len(row), row
        adj[m + i, 0], adj[m + i, 1:3] = 2, [i, max(i - 1, 0)]
    adj[n, 0], adj[n, 1] = 1, 0
    return vecs, adj, n, queries_at(rng, m + 5, dim)


def always_holds(n, dim, rng, width=6, malformed=False):
    """points on a line, point i linked to i+1 .. i+width; the query lies before the line's start, so the walk expands
    0, 1, 2, ... in order and the guess (i+1, found `width` hops earlier) always holds.  `malformed`: every row also
    repeats i+1, holds i+2 + 2^K (an alias of i+2's tag that is out of bounds), an id in [n_total, 2^K), UINT32_MAX and
    the node itself"""
    total = n + 1
    K = k_bits(total)
    assert total + 8 < (1 << K)
    vecs = np.concatenate([line(n, dim), np.zeros((1, dim), np.float32)])
    rows = []
    for u in range(total):
        i = 0 if u == n else u
        nb = [v for v in range(i + 1, i + 1 + width) if v < n]
        if u == n:
            nb = [0] + nb
        if malformed and nb:
            nb = [nb[0], nb[0], nb[1] + (1 << K) if len(nb) > 1 else EMPTY, total + 3, EMPTY, u] + nb[1:]
        rows.append(nb)
    adj = np.zeros((total, max(len(r) for r in rows) + 1), np.uint32)
    for u, r in enumerate(rows):
        adj[u, 0], adj[u, 1:1 + len(r)] = len(r), r
    return vecs, adj, n, queries_at(rng, -20, dim)


@pytest.mark.parametrize("dim", [32, 64, 96, 128])
def test_guess_always_fails(dab, dim):
    rng = np.random.default_rng(dim)
    vecs, adj, n, q = always_fails(300, dim, rng)
    want = check(dab, vecs, adj, n, q, [(20, 1), (100, 1), (100, 2)])
    assert (want[4] > 300).all()  # the whole line was walked


@pytest.mark.parametrize("dim", [32, 128])
@pytest.mark.parametrize("width,malformed", [(6, False), (6, True), (120, False)])
def test_guess_always_holds(dab, dim, width, malformed):
    """width 120: rows longer than the 96-word adjacency buffer; the rest of the row is read from global memory"""
    rng = np.random.default_rng(dim + width + malformed)
    vecs, adj, n, q = always_holds(600, dim, rng, width, malformed)
    want = check(dab, vecs, adj, n, q, [(20, 1), (100, 1), (100, 2)])
    assert (want[3] > 1).all()


def built(dim, n, rng, R=24):
    centers = rng.normal(size=(32, dim)).astype(np.float32)
    base = (centers[rng.integers(0, 32, n)] + 0.3 * rng.normal(size=(n, dim))).astype(np.float32)
    vecs = np.concatenate([base, base[:1]])
    adj = O.build_graph(vecs, n, 1, O.L2, R, int(R * 1.3), 40)
    q = vecs[rng.integers(0, n, 128)] + np.float32(0.05) * rng.normal(size=(128, dim)).astype(np.float32)
    return vecs, adj, q.astype(np.float32)


@pytest.mark.parametrize("dim", [32, 64, 96, 128])
def test_built_graphs(dab, dim):
    rng = np.random.default_rng(dim + 11)
    vecs, adj, q = built(dim, 3000, rng)
    check(dab, vecs, adj, 3000, q, [(25, 1), (100, 1), (200, 1), (100, 2)])


@pytest.mark.parametrize("dim", [64, 128])
def test_level1_closes_and_the_global_table_overflows(dab, monkeypatch, dim):
    """a 512-byte level 1 closes after a few hops, ids spill to the tiny global table, which overflows and re-runs
    queries"""
    monkeypatch.setenv("DAB_TEST_VISITED_LOG2", "8")
    rng = np.random.default_rng(dim + 12)
    vecs, adj, q = built(dim, 4000, rng)
    check(dab, vecs, adj, 4000, q, [(25, 1), (100, 1), (60, 2)])
    vecs, adj, n, q = always_holds(600, dim, rng, 6, True)
    check(dab, vecs, adj, n, q, [(20, 1), (100, 1)])
