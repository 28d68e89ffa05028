"""Filtered range search on the device (dab_range_search_filtered[_device]) bit for bit against the oracle's
FilteredRange::search (oracle/filtered_range_search.cpp, pinned in test_filtered_range_search.py): offsets, ids,
distance bits, cmps, hops and the second-round flag over the reference's seven baselines, every row type and metric,
selectivities from every id to none in both modes, L from 1 to several hundred, beams of 1, 4 and 64, radii from the
k-NN distances, inner radii and max_returned reached in either phase, the edge graphs of test_traversal_edges.py,
deletions and inserts into released ids, and the re-runs of the visited tables, the regions and the result arena; and
the result sets' lifetime, the device form and every refusal."""
import ctypes

import numpy as np
import pytest

import diskann_b200 as dab
import filtered_range_oracle as FR
import oracle_lib as O
from test_filtered_range_search import golden_cases, labels_for, same_results
from test_gpu_parity import make_index
from test_range_search_gpu import INVALID_ARGUMENT, NOT_READY, gpu_index, radii, same
from test_traversal_edges import grid, malformed_case, many_starts, non_finite


def check(g, oidx, queries, runs, deleted=None):
    """every (L, beam, radius, labels, masks, match_all, keyword arguments) of `runs` on the device against the oracle;
    returns how many queries took the second round"""
    second, last = 0, None
    for L, beam, radius, labels, masks, match_all, kw in runs:
        if labels is not last:
            g.upload_labels(labels)
            last = labels
        want = FR.range_search(oidx, queries, L, radius, labels, masks, match_all, beam=beam, deleted=deleted, **kw)
        got = g.range_search_filtered(queries, masks, L, radius, match_all=match_all, beam_width=beam, **kw)
        same(got, want, (L, beam, radius, match_all, kw))
        second += int(want[5].sum())
    return second


def grid_runs(rng, oidx, queries, total, Ls=(1, 10, 40), beams=(1, 4), selectivities=(1.0, 0.5, 0.1, 0.01, 0.0)):
    runs = []
    for s in selectivities:
        labels = labels_for(rng, total, s)
        masks = np.where(rng.random(len(queries)) < 0.8, 1, 0b11).astype(np.uint64)  # most ANY bit 0, some ANY of two bits
        for L in Ls:
            for i, r in enumerate(radii(oidx, queries, max(L, 2))):
                runs.append((L, beams[i % len(beams)], r, labels, masks, False, {}))
        runs.append((Ls[-1], beams[-1], r, labels, np.uint64(0b11), True, {}))  # ALL of two bits
    return runs


@pytest.mark.gpu
def test_the_reference_baselines_on_the_device():
    for c, data, adj, n, labels in golden_cases():
        oidx = O.Index(data, adj, n, 1, O.L2)
        q = np.array([c["query"]], np.float32)
        kw = dict(inner_radius=c["inner_radius"], max_returned=c["max_returned"])
        with gpu_index(data, adj, n, 1, O.L2, adj.shape[1] - 1) as g:
            g.upload_labels(labels)
            got = g.range_search_filtered(q, 1, c["starting_l"], c["radius"], **kw)
        same(got, FR.range_search(oidx, q, c["starting_l"], c["radius"], labels, 1, **kw), c["case"])
        assert (int(got[0][1]), int(got[3][0]), int(got[4][0]), bool(got[5][0])) == (
            c["result_count"], c["comparisons"], c["hops"], c["range_search_second_round"]), c["case"]
        same_results(zip(got[1], got[2]), c)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric,d,n,Rd,Lb", [
    (np.float32, O.L2, 64, 3000, 24, 40),
    (np.float32, O.INNER_PRODUCT, 48, 3000, 24, 40),
    (np.float32, O.COSINE, 48, 3000, 24, 40),
    (np.float32, O.COSINE_NORMALIZED, 48, 3000, 24, 40),
    (np.float16, O.L2, 64, 3000, 24, 40),
    (np.float16, O.INNER_PRODUCT, 96, 3000, 24, 40),
    (np.int8, O.L2, 64, 2000, 16, 30),
    (np.int8, O.COSINE, 40, 2000, 16, 30),
    (np.uint8, O.L2, 128, 2000, 16, 30),
    (np.uint8, O.INNER_PRODUCT, 40, 2000, 16, 30),
])
def test_row_types_and_metrics(dt, metric, d, n, Rd, Lb):
    rng = np.random.default_rng(d + n)
    vecs, adj, maxdeg = make_index(rng, dt, metric, n, d, Rd, Lb)
    nq = 60
    queries = vecs[rng.integers(0, n, nq)].astype(np.float32) + 0.1 * rng.normal(size=(nq, d)).astype(np.float32)
    if dt in (np.int8, np.uint8):
        info = np.iinfo(dt)
        queries = np.clip(np.round(queries), info.min, info.max)
    queries = queries.astype(dt)
    oidx = O.Index(vecs, adj, n, 1, metric)
    with gpu_index(vecs, adj, n, 1, metric, maxdeg) as g:
        runs = grid_runs(rng, oidx, queries, n + 1, Ls=(10,), selectivities=(1.0, 0.3))
        assert check(g, oidx, queries, runs) > 0, "no second round"


@pytest.mark.gpu
def test_selectivity_mode_lists_and_beams():
    rng = np.random.default_rng(3)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 4000, 32, 24, 40)
    queries = (vecs[rng.integers(0, 4000, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 4000, 1, O.L2)
    with gpu_index(vecs, adj, 4000, 1, O.L2, maxdeg) as g:
        assert check(g, oidx, queries, grid_runs(rng, oidx, queries, 4001, Ls=(1, 2, 64, 300), beams=(1, 4, 64))) > 0


@pytest.mark.gpu
def test_inner_radius_and_max_returned():
    """max_returned reached in phase 1, inside a second-round hop, and not reached; inner radii; slack arguments"""
    rng = np.random.default_rng(4)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    queries = (vecs[rng.integers(0, 3000, 80)] + 0.1 * rng.normal(size=(80, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 3000, 1, O.L2)
    L = 20
    r = radii(oidx, queries, L)
    labels = labels_for(rng, 3001, 0.4)
    runs = []
    for radius in (r[2], r[3]):
        for mr in (None, L, L + 1, L + 37):
            for islack in (0.0, 0.5, 1.0):
                for rslack in (1.0, 1.5):
                    for inner in (None, radius / 4):
                        runs.append((L, 1 + (len(runs) % 3) * 3, radius, labels, 1, False,
                                     dict(max_returned=mr, initial_slack=islack, range_slack=rslack, inner_radius=inner)))
    runs += [(L, 1, float("nan"), labels, 1, False, dict(initial_slack=0.0)), (L, 1, r[2], labels, 1, False, dict(range_slack=float("inf")))]
    with gpu_index(vecs, adj, 3000, 1, O.L2, maxdeg) as g:
        check(g, oidx, queries, runs)


@pytest.mark.gpu
def test_edge_graphs():
    rng = np.random.default_rng(7)
    cases = [many_starts(1500, 16, 2, 40, 2), many_starts(1500, 16, 70, 40, 70), grid(1200, 8, 3, 40, 3)]
    cases += [malformed_case(800, 8, 3, md, 40, md) for md in (1, 7, 40)]
    cases += [non_finite(800, 16, dt, m, 40, 7, nan=dt == np.float32)[0] for dt, m in
              ((np.float32, O.L2), (np.float32, O.INNER_PRODUCT), (np.float16, O.L2))]
    for case in cases:
        with gpu_index(case.vecs, case.adj, case.n, case.n_start, case.metric, case.max_degree) as g:
            runs = grid_runs(rng, case.oracle, case.queries, case.total, Ls=(1, 30), selectivities=(1.0, 0.5, 0.0))
            # start points accepted and rejected
            check(g, case.oracle, case.queries, runs)


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    n = 3000
    queries = (vecs[rng.integers(0, n, 80)] + 0.1 * rng.normal(size=(80, 32))).astype(np.float32)
    gone = rng.choice(n, 300, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    runs = grid_runs(rng, oidx, queries, n + 1, Ls=(10, 40), selectivities=(1.0, 0.3))
    with gpu_index(vecs, adj, n, 1, O.L2, maxdeg) as g:
        g.delete(gone)
        check(g, oidx, queries, runs, deleted)
        g.release(gone)
        fresh = (vecs[rng.integers(0, n, 300)] + 0.2 * rng.normal(size=(300, 32))).astype(np.float32)
        g.insert(gone, fresh, 16, 30)
        vecs2 = vecs.copy()
        vecs2[gone] = fresh
        check(g, O.Index(vecs2, g.download_graph(), n, 1, O.L2), queries, runs)


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_RANGE_LIST": "3"}, {"DAB_TEST_RANGE_ARENA": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "2", "DAB_TEST_RANGE_ARENA": "5"}])
def test_reruns(monkeypatch, env):
    """tables of 256 slots, regions of matches (and frontiers of L more) of a few entries, an arena of a few entries:
    queries re-run, some several times, and every one is answered in full"""
    rng = np.random.default_rng(11)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 3000, 32, 16, 30)
    queries = (vecs[rng.integers(0, 3000, 100)] + 0.1 * rng.normal(size=(100, 32))).astype(np.float32)
    oidx = O.Index(vecs, adj, 3000, 1, O.L2)
    runs = grid_runs(rng, oidx, queries, 3001, Ls=(1, 10, 40), selectivities=(1.0, 0.2))
    for var, val in env.items():
        monkeypatch.setenv(var, val)
    with gpu_index(vecs, adj, 3000, 1, O.L2, maxdeg) as g:
        check(g, oidx, queries, runs)


@pytest.mark.gpu
def test_a_radius_over_every_point_returns_every_point():
    rng = np.random.default_rng(6)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 2500, 16, 16, 30)
    oidx = O.Index(vecs, adj, 2500, 1, O.L2)
    queries = vecs[:8] + 0.5
    labels = np.ones(2501, np.uint64)
    with gpu_index(vecs, adj, 2500, 1, O.L2, maxdeg) as g:
        assert g.count_reachable([2500]) == 2501
        g.upload_labels(labels)
        got = g.range_search_filtered(queries, 1, 10, 1e30, beam_width=4)
        same(got, FR.range_search(oidx, queries, 10, 1e30, labels, 1, beam=4), "whole graph")
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
    radius = radii(oidx, queries, 20)[3]
    labels = labels_for(rng, 2001, 0.3)
    masks = np.where(np.arange(100) % 3 == 0, 0b11, 1).astype(np.uint64)
    g = gpu_index(vecs, adj, 2000, 1, O.L2, maxdeg)
    g.upload_labels(labels)
    want = FR.range_search(oidx, queries, 20, radius, labels, masks, beam=2, max_returned=60)
    same(g.range_search_filtered(queries, masks, 20, radius, beam_width=2, max_returned=60), want, "host form")
    d_q = torch.from_numpy(queries).cuda()
    d_m = torch.from_numpy(masks.view(np.int64)).cuda()
    with g.range_search_filtered_device(d_q.data_ptr(), d_m.data_ptr(), 100, 20, radius, beam_width=2, max_returned=60) as r:
        offsets, cmps, hops, second = r.offsets()
        n = r.total()
        d_ids = torch.empty(n, dtype=torch.int32, device="cuda")
        d_dists = torch.empty(n, dtype=torch.float32, device="cuda")
        r.results_device(d_ids.data_ptr(), d_dists.data_ptr())
        torch.cuda.synchronize()
        same((offsets, d_ids.cpu().numpy(), d_dists.cpu().numpy(), cmps, hops, second), want, "device form")
    r = g.range_search_filtered_set(queries, masks, 20, radius, beam_width=2, max_returned=60)
    g.delete(np.arange(0, 2000, 3, dtype=np.uint32))
    g.upload_labels(np.zeros(2001, np.uint64))
    g.upload_vectors(np.zeros_like(vecs))
    g.upload_graph(np.zeros_like(adj))
    offsets, cmps, hops, second = r.offsets()
    same((offsets, *r.results(), cmps, hops, second), want, "snapshot")
    r2 = g.range_search_filtered_set(queries, masks, 20, radius)
    g.close()  # dab_destroy releases both open result sets
    for s in (r, r2):
        with pytest.raises(dab.DabError):
            s.offsets()
        s.close()


@pytest.mark.gpu
def test_refusals_before_any_launch():
    rng = np.random.default_rng(8)
    vecs, adj, maxdeg = make_index(rng, np.float32, O.L2, 1500, 16, 16, 30)
    queries = (vecs[rng.integers(0, 1500, 50)] + 0.1 * rng.normal(size=(50, 16))).astype(np.float32)
    masks = np.ones(50, np.uint64)
    oidx = O.Index(vecs, adj, 1500, 1, O.L2)
    L_ = dab.lib()
    nan, inf = float("nan"), float("inf")
    bad = [  # (L, beam, radius, has_inner, inner, initial_slack, range_slack, max_returned, message)
        (10, 0, 1.0, 0, 0.0, 1.0, 1.0, 0, b"BeamWidthZero"), (0, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, b"LZero"),
        (10, 1, 1.0, 0, 0.0, 1.0, 1.0, 9, b"MaxReturnedLessThanInitialL"), (10, 1, 1.0, 0, 0.0, 1.5, 1.0, 0, b"StartingListSlack"),
        (10, 1, 1.0, 0, 0.0, nan, 1.0, 0, b"StartingListSlack"), (10, 1, 1.0, 0, 0.0, 1.0, 0.5, 0, b"RangeSearchSlack"),
        (10, 1, 1.0, 1, 2.0, 1.0, 1.0, 0, b"InnerRadius"), (10, 1, -inf, 1, 0.0, 1.0, 1.0, 0, b"InnerRadius"),
        (10, 65, 1.0, 0, 0.0, 1.0, 1.0, 0, b"beam_width 65 > 64"), (1024, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, b"L + #start = 1025 > 1024"),
        (0, 0, 1.0, 1, 2.0, 2.0, 0.0, 0, b"BeamWidthZero"), (10, 1, 1.0, 1, 2.0, 2.0, 0.0, 1, b"MaxReturnedLessThanInitialL"),
    ]
    fns = (L_.dab_range_search_filtered, L_.dab_range_search_filtered_device)
    with gpu_index(vecs, adj, 1500, 1, O.L2, maxdeg) as g:
        launches = dab.launch_count()
        # no label table yet
        for fn in fns:
            out = ctypes.c_void_p()
            assert fn(g._h, O.ptr(queries), 50, 10, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, O.ptr(masks), 0, ctypes.byref(out)) == INVALID_ARGUMENT
            assert b"no label table" in L_.dab_last_error() and not out.value
        labels = labels_for(rng, 1501, 0.5)
        g.upload_labels(labels)
        launches = dab.launch_count()
        for L, beam, radius, hi, inner, isl, rsl, mr, what in bad:
            for fn in fns:
                out = ctypes.c_void_p()
                assert fn(g._h, O.ptr(queries), 50, L, beam, radius, hi, inner, isl, rsl, mr, O.ptr(masks), 0,
                          ctypes.byref(out)) == INVALID_ARGUMENT, what
                assert what in L_.dab_last_error(), (what, L_.dab_last_error())
                assert not out.value
        assert dab.launch_count() == launches, "a refusal launched a kernel"
        assert not g._ranges
        radius = radii(oidx, queries, 10)[2]
        same(g.range_search_filtered(queries, masks, 10, radius), FR.range_search(oidx, queries, 10, radius, labels, masks), "after")
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, 16, 100, 1, 8) as g:
        out = ctypes.c_void_p()
        assert L_.dab_range_search_filtered(g._h, O.ptr(queries), 1, 10, 1, 1.0, 0, 0.0, 1.0, 1.0, 0, O.ptr(masks), 0,
                                            ctypes.byref(out)) == NOT_READY
    d = 30000
    with gpu_index(np.zeros((11, d), np.float32), np.zeros((11, 9), np.uint32), 10, 1, O.L2, 8) as g:
        g.upload_labels(np.ones(11, np.uint64))
        launches = dab.launch_count()
        with pytest.raises(dab.DabError, match="shared memory"):
            g.range_search_filtered(np.zeros((1, d), np.float32), 1, 4, 1.0)
        assert dab.launch_count() == launches
