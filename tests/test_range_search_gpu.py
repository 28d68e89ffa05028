"""Range search on the device (dab_range_search[_device] and its result sets) bit for bit against the oracle's
Range::search (oracle/range_search.cpp, pinned in test_range_search.py): offsets, ids, distance bits, cmps, hops and the
second-round flag over the reference's five baselines, every row type and metric, L from 1 to several hundred, beams of
1, 4 and 64, radii from the k-NN distances (no second round up to long ones), every argument the reference accepts,
the edge graphs of test_traversal_edges.py, deletions and inserts into released ids, and the re-runs of the visited
tables, of the in_range regions and of the result arena; and the result sets' lifetime, the device form and every
refusal."""
import ctypes
import json
import os

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
import range_oracle as R
from test_gpu_parity import make_index
from test_oracle_golden import grid as lattice
from test_traversal_edges import grid, malformed_case, many_starts, non_finite

SIX = ("offsets", "ids", "dists", "cmps", "hops", "second_round")
INVALID_ARGUMENT, OUT_OF_MEMORY, NOT_READY = 1, 3, 5  # include/diskann_b200.h
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "range_search.json")


def same(got, want, what):
    for a, b, name in zip(got, want, SIX):
        a, b = np.asarray(a), np.asarray(b)
        if name == "second_round":
            a, b = a.astype(bool), b.astype(bool)
        elif a.dtype.itemsize == 4:
            a, b = a.view(np.uint32), b.view(np.uint32)
        assert a.shape == b.shape and np.array_equal(a, b), (what, name)


def gpu_index(vecs, adj, n, n_start, metric, max_degree):
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree)
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    return g


def check(g, oidx, queries, runs, deleted=None):
    """every (L, beam, radius, keyword arguments) of `runs` on the device against the oracle; returns how many queries
    took the second round"""
    second = 0
    for L, beam, radius, kw in runs:
        want = R.range_search(oidx, queries, L, radius, beam=beam, deleted=deleted, **kw)
        same(g.range_search(queries, L, radius, beam_width=beam, **kw), want, (L, beam, radius, kw))
        second += int(want[5].sum())
    return second


def radii(oidx, queries, L):
    """radii at the k-NN distances of rank 1, L/2, L - 1 and 3L of every query's list, at the median query: few
    queries reach the second round at the first two, about half at the third and most at the last"""
    want = oidx.search_batch(queries, 3 * L, 3 * L)[1]
    return [float(np.median(want[:, i])) for i in (1, L // 2, L - 1, 3 * L - 1)]


def runs_over(oidx, queries, Ls=(1, 10, 40), beams=(1, 4)):
    out = []
    for L in Ls:
        for r in radii(oidx, queries, max(L, 2)):
            for beam in beams:
                out.append((L, beam, r, {}))
    return out


@pytest.mark.gpu
def test_the_reference_baselines_on_the_device():
    for c in json.load(open(GOLDEN))["cases"]:
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        q = np.array([c["query"]], np.float32)
        with gpu_index(data, adj, n, 1, O.L2, adj.shape[1] - 1) as g:
            off, ids, dists, cmps, hops, second = g.range_search(q, c["starting_l"], c["radius"], inner_radius=c["inner_radius"],
                                                                 max_returned=c["max_returned"])
        assert int(off[1]) == c["result_count"] and cmps[0] == c["comparisons"] and hops[0] == c["hops"], c["case"]
        assert bool(second[0]) == c["range_search_second_round"], c["case"]
        if isinstance(c["results"], list):
            assert [[int(i), float(d)] for i, d in zip(ids, dists)] == c["results"], c["case"]
        same((off, ids, dists, cmps, hops, second), R.range_search(O.Index(data, adj, n, 1, O.L2), q, c["starting_l"], c["radius"],
                                                                   inner_radius=c["inner_radius"], max_returned=c["max_returned"]), c["case"])


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric,d,n,Rd,Lb", [
    (np.float32, O.L2, 128, 3000, 24, 40),
    (np.float32, O.INNER_PRODUCT, 64, 2000, 16, 30),
    (np.float32, O.COSINE, 48, 2000, 16, 30),
    (np.float32, O.COSINE_NORMALIZED, 32, 2000, 16, 30),
    (np.float16, O.L2, 64, 2000, 16, 30),
    (np.float16, O.INNER_PRODUCT, 96, 2000, 16, 30),
    (np.float16, O.COSINE, 64, 2000, 16, 30),
    (np.float16, O.COSINE_NORMALIZED, 32, 2000, 16, 30),
    (np.int8, O.L2, 128, 2000, 16, 30),
    (np.int8, O.INNER_PRODUCT, 64, 2000, 16, 30),
    (np.int8, O.COSINE, 64, 2000, 16, 30),
    (np.uint8, O.L2, 128, 2000, 16, 30),
    (np.uint8, O.INNER_PRODUCT, 40, 2000, 16, 30),
    (np.uint8, O.COSINE_NORMALIZED, 40, 2000, 16, 30),
])
def test_row_types_and_metrics(dt, metric, d, n, Rd, Lb):
    rng = np.random.default_rng(d + n)
    vecs, adj, maxdeg = make_index(rng, dt, metric, n, d, Rd, Lb)
    nq = 100
    queries = vecs[rng.integers(0, n, nq)].astype(np.float32) + 0.1 * rng.normal(size=(nq, d)).astype(np.float32)
    if dt in (np.int8, np.uint8):
        info = np.iinfo(dt)
        queries = np.clip(np.round(queries), info.min, info.max)
    queries = queries.astype(dt)
    oidx = O.Index(vecs, adj, n, 1, metric)
    with gpu_index(vecs, adj, n, 1, metric, maxdeg) as g:
        assert check(g, oidx, queries, runs_over(oidx, queries)) > 0, "no second round"


@pytest.mark.gpu
def test_lists_and_beams():
    rng = np.random.default_rng(3)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 4000, 32, 24, 40)
    queries = (vecs[rng.integers(0, 4000, 150)] + 0.1 * rng.normal(size=(150, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 4000, 1, O.L2)
    with gpu_index(vecs, adj, 4000, 1, O.L2, maxdeg) as g:
        assert check(g, oidx, queries, runs_over(oidx, queries, Ls=(1, 2, 64, 300), beams=(1, 4, 64))) > 0


@pytest.mark.gpu
def test_every_argument_the_reference_accepts():
    rng = np.random.default_rng(4)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    queries = (vecs[rng.integers(0, 3000, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 3000, 1, O.L2)
    L = 20
    r = radii(oidx, queries, L)
    runs = []
    for radius in (r[1], r[2], r[3]):
        for mr in (None, L, L + 1, L + 37):  # L + 37 cuts a phase-2 hop in the middle
            for islack in (0.0, 0.5, 1.0):
                for rslack in (1.0, 1.5, float("inf")):
                    for inner in (None, radius / 4):
                        runs.append((L, 1 + (len(runs) % 3) * 3, radius, dict(max_returned=mr, initial_slack=islack, range_slack=rslack,
                                                                              inner_radius=inner)))
    # a NaN radius: nothing is in range, and the second round runs on an empty frontier where L * initial_slack < 1;
    # radius 0 with an infinite range slack: the bound is NaN and the second round admits nothing
    runs += [(L, 1, float("nan"), dict(initial_slack=s)) for s in (0.0, 0.04, 1.0)]
    runs += [(L, 1, 0.0, dict(range_slack=float("inf"), initial_slack=0.0)), (L, 2, 0.0, dict(initial_slack=0.0))]
    runs += [(L, 1, r[2], dict(range_slack=float("nan"))), (L, 1, r[2], dict(inner_radius=float("nan")))]
    with gpu_index(vecs, adj, 3000, 1, O.L2, maxdeg) as g:
        check(g, oidx, queries, runs)
        got = g.range_search(queries, L, float("nan"), initial_slack=0.0)
        assert got[5].all() and int(got[0][-1]) == 0
        assert np.array_equal(got[4], 2 * g.search_batch(queries, L, L)[4])


@pytest.mark.gpu
def test_edge_graphs():
    cases = [many_starts(1500, 16, 2, 60, 2), many_starts(1500, 16, 70, 60, 70), grid(1200, 8, 3, 60, 3)]
    cases += [malformed_case(800, 8, 3, md, 60, md) for md in (1, 7, 40)]
    cases += [non_finite(800, 16, dt, m, 60, 7, nan=dt == np.float32)[0] for dt, m in
              ((np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.L2))]
    for case in cases:
        with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
            check(g, case.oracle, case.queries, runs_over(case.oracle, case.queries, Ls=(1, 30), beams=(1, 4)))


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    n = 3000
    queries = (vecs[rng.integers(0, n, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    gone = rng.choice(n, 300, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    runs = runs_over(oidx, queries, Ls=(10, 40))
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
        g.delete(gone)
        check(g, oidx, queries, runs + [(10, 1, runs[-1][2], dict(max_returned=25))], deleted)
        got = g.range_search(queries, 40, runs[-1][2])
        assert not np.isin(got[1], gone).any()
        g.release(gone)
        fresh = (vecs[rng.integers(0, n, 300)] + 0.2 * rng.normal(size=(300, 32))).astype(np.float32)
        g.insert(gone, fresh, 16, 30)
        vecs2 = vecs.copy()
        vecs2[gone] = fresh
        check(g, O.Index(vecs2, g.download_graph(), n, 1, O.L2), queries, runs)


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_RANGE_LIST": "3"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "1"}, {"DAB_TEST_RANGE_ARENA": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "2", "DAB_TEST_RANGE_ARENA": "5"}])
def test_reruns(monkeypatch, env):
    """tables of 256 slots, in_range regions of a few entries and an arena of a few entries: queries re-run, some
    several times, and every one is answered in full"""
    rng = np.random.default_rng(11)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    queries = (vecs[rng.integers(0, 3000, 150)] + 0.1 * rng.normal(size=(150, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 3000, 1, O.L2)
    runs = runs_over(oidx, queries, Ls=(1, 10, 40))
    for var, val in env.items():
        monkeypatch.setenv(var, val)
    with gpu_index(vecs, adj, 3000, 1, O.L2, maxdeg) as g:
        check(g, oidx, queries, runs)


@pytest.mark.gpu
def test_a_radius_over_every_point_returns_every_reachable_point():
    """the property the reference's sift range test asserts: a connected graph, a radius past every distance, every
    non-start point exactly once"""
    rng = np.random.default_rng(6)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 2500, 16, 16, 30)
    oidx = O.Index(vecs, adj, 2500, 1, O.L2)
    queries = vecs[:8] + 0.5
    with gpu_index(vecs, adj, 2500, 1, O.L2, maxdeg) as g:
        assert g.count_reachable([2500]) == 2501
        got = g.range_search(queries, 10, 1e30, beam_width=4)
        same(got, R.range_search(oidx, queries, 10, 1e30, beam=4), "whole graph")
        for q in range(8):
            ids = got[1][got[0][q]:got[0][q + 1]]
            assert len(ids) == 2500 and len(set(ids.tolist())) == 2500


@pytest.mark.gpu
def test_device_form_snapshot_and_destroy():
    import torch
    rng = np.random.default_rng(2)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 2000, 32, 16, 30)
    queries = (vecs[rng.integers(0, 2000, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 2000, 1, O.L2)
    radius = radii(oidx, queries, 20)[2]
    g = gpu_index(vecs, adj, 2000, 1, O.L2, maxdeg)
    want = g.range_search(queries, 20, radius, beam_width=2, max_returned=60)
    d_q = torch.from_numpy(queries).cuda()
    with g.range_search_device(d_q.data_ptr(), 100, 20, radius, beam_width=2, max_returned=60) as r:
        offsets, cmps, hops, second = r.offsets()
        n = r.total()
        d_ids = torch.empty(n, dtype=torch.int32, device="cuda")
        d_dists = torch.empty(n, dtype=torch.float32, device="cuda")
        r.results_device(d_ids.data_ptr(), d_dists.data_ptr())
        torch.cuda.synchronize()
        same((offsets, d_ids.cpu().numpy(), d_dists.cpu().numpy(), cmps, hops, second), want, "device form")
    # a result set is a snapshot: later writes to the index leave it as it was
    r = g.range_search_set(queries, 20, radius, beam_width=2, max_returned=60)
    g.delete(np.arange(0, 2000, 3, dtype=np.uint32))
    g.upload_vectors(np.zeros_like(vecs))
    g.upload_graph(np.zeros_like(adj))
    offsets, cmps, hops, second = r.offsets()
    same((offsets, *r.results(), cmps, hops, second), want, "snapshot")
    r2 = g.range_search_set(queries, 20, radius)
    g.close()  # dab_destroy releases both open result sets
    for s in (r, r2):
        with pytest.raises(dab.DabError):
            s.offsets()
        s.close()


@pytest.mark.gpu
def test_refusals_before_any_launch(monkeypatch):
    rng = np.random.default_rng(8)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 1500, 16, 16, 30)
    queries = (vecs[rng.integers(0, 1500, 50)] + 0.1 * rng.normal(size=(50, 16))).astype(np.float32)
    oidx = O.Index(vecs, adj, 1500, 1, O.L2)
    L_ = dab.lib()
    nan, inf = float("nan"), float("inf")
    bad = [  # (L, beam, radius, has_inner, inner, initial_slack, range_slack, max_returned, message)
        (10, 0, 1.0, 0, 0.0, 1.0, 1.0, 0, b"BeamWidthZero"), (0, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, b"LZero"),
        (10, 1, 1.0, 0, 0.0, 1.0, 1.0, 9, b"MaxReturnedLessThanInitialL"), (10, 1, 1.0, 0, 0.0, 1.5, 1.0, 0, b"StartingListSlack"),
        (10, 1, 1.0, 0, 0.0, -0.1, 1.0, 0, b"StartingListSlack"), (10, 1, 1.0, 0, 0.0, nan, 1.0, 0, b"StartingListSlack"),
        (10, 1, 1.0, 0, 0.0, 1.0, 0.5, 0, b"RangeSearchSlack"), (10, 1, 1.0, 1, 2.0, 1.0, 1.0, 0, b"InnerRadius"),
        (10, 1, -inf, 1, 0.0, 1.0, 1.0, 0, b"InnerRadius"), (10, 65, 1.0, 0, 0.0, 1.0, 1.0, 0, b"beam_width 65 > 64"),
        # the reference's order: the first failing check names the error
        (0, 0, 1.0, 1, 2.0, 2.0, 0.0, 0, b"BeamWidthZero"), (10, 1, 1.0, 1, 2.0, 2.0, 0.0, 1, b"MaxReturnedLessThanInitialL"),
    ]
    with gpu_index(vecs, adj, 1500, 1, O.L2, maxdeg) as g:
        launches = dab.launch_count()
        for L, beam, radius, hi, inner, isl, rsl, mr, what in bad:
            for fn in (L_.dab_range_search, L_.dab_range_search_device):
                out = ctypes.c_void_p()
                assert fn(g._h, O.ptr(queries), 50, L, beam, radius, hi, inner, isl, rsl, mr, ctypes.byref(out)) == INVALID_ARGUMENT, what
                assert what in L_.dab_last_error(), (what, L_.dab_last_error())
                assert not out.value
        assert dab.launch_count() == launches, "a refusal launched a kernel"
        radius = radii(oidx, queries, 10)[2]
        same(g.range_search(queries, 10, radius), R.range_search(oidx, queries, 10, radius), "after the refusals")
    # no graph yet; a query row too long for the kernel's shared memory
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, 16, 100, 1, 8) as g:
        out = ctypes.c_void_p()
        assert L_.dab_range_search(g._h, O.ptr(queries), 1, 10, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, ctypes.byref(out)) == NOT_READY
    d = 60000
    with gpu_index(np.zeros((11, d), np.float32), np.zeros((11, 9), np.uint32), 10, 1, O.L2, 8) as g:
        launches = dab.launch_count()
        with pytest.raises(dab.DabError, match="shared memory"):
            g.range_search(np.zeros((1, d), np.float32), 4, 1.0)
        assert dab.launch_count() == launches


@pytest.mark.gpu
def test_results_beyond_the_arena_limit(monkeypatch):
    """a batch whose results pass the test hook's limit fails with DAB_ERR_OUT_OF_MEMORY naming the entries it needs,
    leaves nothing behind and the index usable; one under the limit grows its arena and is answered in full"""
    rng = np.random.default_rng(9)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 2000, 16, 16, 30)
    queries = (vecs[rng.integers(0, 2000, 60)] + 0.1 * rng.normal(size=(60, 16))).astype(np.float32)
    oidx = O.Index(vecs, adj, 2000, 1, O.L2)
    big, small = radii(oidx, queries, 20)[3], radii(oidx, queries, 20)[1]
    want_big = R.range_search(oidx, queries, 20, big)
    want_small = R.range_search(oidx, queries, 20, small)
    need = int(want_big[0][-1])
    assert need > int(want_small[0][-1]) + 8
    monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(need - 1))
    monkeypatch.setenv("DAB_TEST_RANGE_ARENA", "4")
    with gpu_index(vecs, adj, 2000, 1, O.L2, maxdeg) as g:
        for _ in range(2):
            with pytest.raises(dab.DabError) as e:
                g.range_search(queries, 20, big)
            assert e.value.code == OUT_OF_MEMORY and f"{need} entries".encode() in dab.lib().dab_last_error()
        assert not g._ranges
        same(g.range_search(queries, 20, small), want_small, "under the limit")
    monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(need))
    with gpu_index(vecs, adj, 2000, 1, O.L2, maxdeg) as g:
        same(g.range_search(queries, 20, big), want_big, "at the limit")
