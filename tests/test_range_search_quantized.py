"""Range search over the PQ, SQ and MinMax stores: dab_range_search_{pq,sq,minmax}[_device].

The reference's Range::search is generic over the search strategy (range_search.rs:255-469): both phases read the
strategy's accessor, so every distance — the traversal, the in_range test and the second round's test — is the store's,
and the strategy's post-processor runs over in_range behind a DistanceFiltered buffer.  Without rerank that is the
full-precision output rule on the store's distances; with rerank (Pipeline<FilterStartPoints, Rerank>) in_range loses
its start points and deleted ids, each id gets its full-precision distance, the ids outside (inner_radius, radius] of
it are dropped and the rest are sorted by it, stably.

CPU: the oracle's table entry point (orc_range_search_table, oracle/range_table.cpp) fed the full-precision distances
equals orc_range_search bit for bit — ids, distance bits, order, counts, cmps, hops and the second-round flag — over the
reference's five baselines, row types and metrics, L from 1 to 300, beams 1, 4 and 64, every argument combination,
NaN and zero radii, edge graphs and deletions; with rerank it equals a Python restatement of the rule, exact ties, ±0
and non-finite rows included.
GPU: the device equals the oracle fed each store's exhaustive distances (test_paged_search_quantized.py pins them to
the oracle's quantized searches) bit for bit, with rerank 0 and 1, over every PQ table kind and chunk layout, every SQ
and MinMax width, metric and transform, every row type, beams 1 / 4 / 64, the argument grid, edge graphs, deletions and
re-inserted ids and the forced re-runs; the device form, snapshots, dab_destroy, every refusal before any launch and
the out-of-memory path."""
import ctypes
import functools
import json
import os

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O
import range_oracle as R
import range_table_oracle as RT
from test_diverse_search_quantized import encoded, fp_tables, store_tables
from test_gpu_parity import make_index
from test_oracle_golden import grid as lattice
from test_paged_search import built
from test_paged_search_quantized import MMStore, PQStore, SQStore, pq_store, sq_store
from test_traversal_edges import grid as tie_grid, malformed_case, many_starts, non_finite

F32 = np.float32
SIX = ("offsets", "ids", "dists", "cmps", "hops", "second_round")
INVALID_ARGUMENT, OUT_OF_MEMORY, NOT_READY = 1, 3, 5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "range_search.json")


def same(got, want, what):
    for a, b, name in zip(got, want, SIX):
        a, b = np.asarray(a), np.asarray(b)
        if name == "second_round":
            a, b = a.astype(bool), b.astype(bool)
        elif a.dtype.itemsize == 4:
            a, b = a.view(np.uint32), b.view(np.uint32)
        assert a.shape == b.shape and np.array_equal(a, b), (what, name)


def radii_of(tables, L):
    """radii at the sorted table distances of rank 1, L/2, L - 1 and 3L of every query, at the median query"""
    s = np.sort(tables, axis=1)
    return [float(np.median(s[:, min(i, s.shape[1] - 1)])) for i in (1, L // 2, L - 1, 3 * L - 1)]


def runs_over(tables, Ls=(1, 10, 40), beams=(1, 4)):
    return [(L, beam, r, {}) for L in Ls for r in radii_of(tables, max(L, 2)) for beam in beams]


# ---------------------------------------------------------------- CPU

def table_equals_search(oidx, queries, tables, runs, deleted=None):
    second = 0
    for L, beam, radius, kw in runs:
        want = R.range_search(oidx, queries, L, radius, beam=beam, deleted=deleted, **kw)
        same(RT.range_search_table(oidx, tables, None, L, radius, beam=beam, deleted=deleted, **kw), want, (L, beam, radius, kw))
        second += int(want[5].sum())
    return second


def test_table_of_full_precision_distances_reproduces_the_baselines():
    for c in json.load(open(GOLDEN))["cases"]:
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        q = np.array([c["query"]], F32)
        oidx = O.Index(data, adj, n, 1, O.L2)
        got = RT.range_search_table(oidx, fp_tables(data, O.L2, q), None, c["starting_l"], c["radius"], inner_radius=c["inner_radius"],
                                    max_returned=c["max_returned"])
        assert int(got[0][1]) == c["result_count"] and got[3][0] == c["comparisons"] and got[4][0] == c["hops"], c["case"]
        assert bool(got[5][0]) == c["range_search_second_round"], c["case"]
        if isinstance(c["results"], list):
            assert [[int(i), float(d)] for i, d in zip(got[1], got[2])] == c["results"], c["case"]
        same(got, R.range_search(oidx, q, c["starting_l"], c["radius"], inner_radius=c["inner_radius"], max_returned=c["max_returned"]),
             c["case"])


@pytest.mark.parametrize("dt,metric", [(F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.int8, O.L2),
                                       (np.uint8, O.COSINE_NORMALIZED), (np.float16, O.INNER_PRODUCT), (np.int8, O.COSINE)])
def test_table_of_full_precision_distances_is_the_range_search(dt, metric):
    rng = np.random.default_rng(7)
    vecs, adj, maxdeg = make_index(rng, dt, metric, 500, 16, 12, 24)
    queries = vecs[rng.integers(0, 500, 8)]
    oidx = O.Index(vecs, adj, 500, 1, metric)
    tables = fp_tables(vecs, metric, queries)
    table_equals_search(oidx, queries, tables, runs_over(tables, Ls=(1, 10, 40)))


@pytest.mark.parametrize("beam", [1, 4, 64])
def test_lists_and_beams(beam):
    rng = np.random.default_rng(beam)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 800, 16, 12, 24)
    queries = (vecs[rng.integers(0, 800, 6)] + 0.1 * rng.normal(size=(6, 16))).astype(F32)
    oidx = O.Index(vecs, adj, 800, 1, O.L2)
    tables = fp_tables(vecs, O.L2, queries)
    assert table_equals_search(oidx, queries, tables, runs_over(tables, Ls=(1, 2, 64, 300), beams=(beam,))) > 0


def argument_grid(r, L):
    runs = []
    for radius in (r[1], r[2], r[3]):
        for mr in (None, L, L + 1, L + 23):
            for islack in (0.0, 0.5, 1.0):
                for rslack in (1.0, 1.5, float("inf")):
                    for inner in (None, radius / 4):
                        runs.append((L, 1 + (len(runs) % 3) * 3, radius, dict(max_returned=mr, initial_slack=islack, range_slack=rslack,
                                                                              inner_radius=inner)))
    runs += [(L, 1, float("nan"), dict(initial_slack=s)) for s in (0.0, 0.05, 1.0)]
    runs += [(L, 1, 0.0, dict(range_slack=float("inf"), initial_slack=0.0)), (L, 2, 0.0, dict(initial_slack=0.0))]
    runs += [(L, 1, r[2], dict(range_slack=float("nan"))), (L, 1, r[2], dict(inner_radius=float("nan")))]
    return runs


def test_every_argument_the_reference_accepts():
    rng = np.random.default_rng(4)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 500, 16, 12, 24)
    queries = (vecs[rng.integers(0, 500, 6)] + 0.1 * rng.normal(size=(6, 16))).astype(F32)
    oidx = O.Index(vecs, adj, 500, 1, O.L2)
    tables = fp_tables(vecs, O.L2, queries)
    table_equals_search(oidx, queries, tables, argument_grid(radii_of(tables, 12), 12))


def test_edge_graphs_and_deletions():
    cases = [many_starts(300, 8, 2, 6, 2), many_starts(300, 8, 40, 6, 40), tie_grid(300, 6, 3, 6, 3)]
    cases += [malformed_case(150, 6, 3, md, 6, md) for md in (1, 7, 40)]
    cases += [non_finite(200, 8, dt, m, 6, 7, nan=dt == F32)[0] for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2))]
    for case in cases:
        tables = fp_tables(case.vecs, case.metric, case.queries)
        table_equals_search(case.oracle, case.queries, tables, runs_over(tables, Ls=(1, 12)))
        deleted = np.zeros(case.n + case.n_start, bool)
        deleted[::5] = True
        table_equals_search(case.oracle, case.queries, tables, runs_over(tables, Ls=(12,), beams=(2,)), deleted)


def rerank_rule(vecs, metric, query, in_range, radius, inner_radius):
    """Pipeline<FilterStartPoints, Rerank> behind DistanceFiltered, restated: in_range's ids (start points and deleted
    ids already out) by full-precision distance, those within (inner_radius, radius], sorted stably (-0.0 == +0.0)"""
    ids = np.asarray(in_range, np.int64)
    fp = O.distance_rows(query, vecs[ids], metric, O.AVX2) if len(ids) else np.empty(0, F32)
    with np.errstate(invalid="ignore"):
        keep = (fp <= F32(radius)) & ~((inner_radius is not None) & (fp <= F32(0.0 if inner_radius is None else inner_radius)))
    ids, fp = ids[keep], fp[keep]
    order = np.argsort(np.where(fp == 0, F32(0.0), fp), kind="stable")
    return ids[order].astype(np.uint32), fp[order]


def check_rerank_rule(oidx, vecs, metric, queries, tables, runs, deleted=None):
    for L, beam, radius, inner in runs:
        # with range_slack 1 every in_range distance is within the radius: the output without rerank and without an
        # inner radius is in_range without start points and deleted ids
        base = RT.range_search_table(oidx, tables, None, L, radius, beam=beam, deleted=deleted)
        got = RT.range_search_table(oidx, tables, queries, L, radius, beam=beam, deleted=deleted, rerank=True, inner_radius=inner)
        same((None, None, None, *got[3:]), (None, None, None, *base[3:]), (L, beam, radius, inner))
        for q in range(queries.shape[0]):
            a, b = int(base[0][q]), int(base[0][q + 1])
            w_ids, w_d = rerank_rule(vecs, metric, queries[q], base[1][a:b], radius, inner)
            c, d = int(got[0][q]), int(got[0][q + 1])
            assert np.array_equal(got[1][c:d], w_ids), (L, beam, radius, inner, q)
            assert np.array_equal(got[2][c:d].view(np.uint32), w_d.view(np.uint32)), (L, beam, radius, inner, q)


@pytest.mark.parametrize("kind", ["pq", "sq", "mm"])
def test_rerank_is_the_rule_over_each_store(kind):
    case = built(600, 16, F32, O.L2, 8, seed=5)
    vecs, adj, n, n_start, metric, qs = case
    store = pq_store(case, 4) if kind == "pq" else sq_store(case, 4) if kind == "sq" else MMStore(vecs, 4, "double_same", metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs)
    deleted = np.zeros(n + n_start, bool)
    deleted[::7] = True
    runs = [(L, beam, r, inner) for L in (10, 40) for beam in (1, 4) for r in radii_of(tables, L)[1:] for inner in (None, r / 3)]
    for dl in (None, deleted):
        check_rerank_rule(oidx, vecs, metric, qs, tables, runs, dl)


def test_rerank_rule_on_ties_signed_zeros_and_non_finite_rows():
    # exact ties all along the list
    c = tie_grid(300, 6, 3, 6, 3)
    tables = np.round(fp_tables(c.vecs, c.metric, c.queries) / 4) * 4  # coarser ties in the traversal too
    check_rerank_rule(c.oracle, c.vecs, c.metric, c.queries, tables.astype(F32), [(12, 1, 40.0, None), (30, 4, 60.0, 8.0)])
    # inner products of zero rows: -0.0, tied with +0.0 rows of the same distance
    rng = np.random.default_rng(2)
    vecs, adj, maxdeg = make_index(rng, F32, O.INNER_PRODUCT, 300, 8, 12, 24)
    vecs = vecs.copy()
    vecs[::9] = 0.0
    vecs[1::9] = -0.0
    queries = vecs[rng.integers(0, 300, 6)] + 0.1
    oidx = O.Index(vecs, adj, 300, 1, O.INNER_PRODUCT)
    tables = fp_tables(vecs, O.INNER_PRODUCT, queries)
    assert np.signbit(tables[tables == 0]).any()
    check_rerank_rule(oidx, vecs, O.INNER_PRODUCT, queries, tables, [(20, 1, 0.0, None), (20, 2, 1.0, None), (20, 1, 1.0, -1.0)])
    # ±inf and NaN rows: NaN full-precision distances never pass the radius
    for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2)):
        c = non_finite(200, 8, dt, m, 6, 7, nan=dt == F32)[0]
        tables = np.nan_to_num(fp_tables(c.vecs, c.metric, c.queries), nan=1.0, posinf=2.0, neginf=-2.0).astype(F32)
        check_rerank_rule(c.oracle, c.vecs, c.metric, c.queries, tables, [(12, 1, 1.5, None), (12, 4, 3.0, 0.5)])


# ---------------------------------------------------------------- GPU

def kind_of(store):
    return {PQStore: "pq", SQStore: "sq", MMStore: "minmax"}[type(store)]


def gpu_index(case, store, max_degree=None, vectors=True):
    vecs, adj, n, n_start, metric = case[:5]
    g = dab.GpuIndex(O.dtype_code(vecs), metric, vecs.shape[1], n, n_start, max_degree or adj.shape[1] - 1)
    if vectors:
        g.upload_vectors(vecs)
    g.upload_graph(adj)
    store.upload(g)
    return g


def check(g, store, case, runs, deleted=None, tables=None, reranks=(False, True)):
    """every (L, beam, radius, keyword arguments) of `runs`, with and without rerank, on the device against the oracle
    fed the store's distances; returns how many queries took the second round"""
    vecs, adj, n, n_start, metric, qs = case[:6]
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs) if tables is None else tables
    fn = getattr(g, f"range_search_{kind_of(store)}")
    second = 0
    for L, beam, radius, kw in runs:
        for rr in reranks:
            want = RT.range_search_table(oidx, tables, qs, L, radius, beam=beam, deleted=deleted, rerank=rr, **kw)
            same(fn(qs, L, radius, beam_width=beam, rerank=rr, **kw), want, (kind_of(store), L, beam, radius, kw, rr))
            second += int(want[5].sum())
    return second


NQ = 100


@functools.lru_cache(maxsize=None)
def gpu_case(dt, metric, d=64):
    return built(2000, d, dt, metric, NQ, seed=41 + d)


def run_store(case, store, Ls=(1, 10, 40), beams=(1, 4)):
    tables = store_tables(store, case[5])
    with gpu_index(case, store) as g:
        assert check(g, store, case, runs_over(tables, Ls, beams), tables=tables) > 0, "no second round"


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(F32, O.L2), (np.int8, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.uint8, O.COSINE_NORMALIZED)])
@pytest.mark.parametrize("chunks", [16, 8, 7])  # chunks of 4, of 8, of 9 and 10
def test_pq_equals_the_oracle(dt, metric, chunks):
    case = gpu_case(dt, metric)
    run_store(case, pq_store(case, chunks))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_sq_equals_the_oracle(nbits, metric):
    dt = {8: F32, 4: np.float16, 2: np.int8, 1: np.uint8}[nbits]
    case = gpu_case(dt, metric)
    run_store(case, sq_store(case, nbits))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_minmax_equals_the_oracle(nbits, metric):
    dt = {8: F32, 4: np.float16, 2: np.uint8, 1: np.int8}[nbits]
    case = gpu_case(dt, metric, d=48)  # 48: PaddingHadamard pads to 64
    for kind in (None, "padding_natural", "double_same"):
        run_store(case, MMStore(case[0], nbits, kind, metric), Ls=(1, 10))


def three_stores(case):
    return [pq_store(case, 8), sq_store(case, 8), MMStore(case[0], 8, "double_same", case[4])]


@pytest.mark.gpu
def test_lists_and_beams():
    case = gpu_case(F32, O.L2, d=32)
    for store in three_stores(case):
        run_store(case, store, Ls=(1, 2, 64, 300), beams=(1, 4, 64))


@pytest.mark.gpu
def test_every_argument_the_reference_accepts():
    case = gpu_case(F32, O.L2, d=32)
    for store in three_stores(case):
        tables = store_tables(store, case[5])
        with gpu_index(case, store) as g:
            check(g, store, case, argument_grid(radii_of(tables, 20), 20), tables=tables)


def as_tuple(c):
    return (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)


@pytest.mark.gpu
def test_edge_graphs():
    cases = [many_starts(1500, 16, 2, 60, 2), many_starts(1500, 16, 70, 60, 70), tie_grid(1200, 8, 3, 60, 3)]
    cases += [malformed_case(800, 8, 3, md, 60, md) for md in (1, 7, 40)]
    cases += [non_finite(800, 16, dt, m, 60, 7, nan=dt == F32)[0] for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2))]
    for c in cases:
        case = as_tuple(c)
        # the stores encode the finite rows (a PQ code has no NaN or inf) and the rerank reads the rows as they are;
        # MinMax refuses the non-finite queries of those cases
        stores = three_stores((np.nan_to_num(c.vecs, nan=0.0, posinf=4.0, neginf=-4.0), *case[1:]))
        for store in stores if np.isfinite(c.queries.astype(F32)).all() else stores[:2]:
            tables = store_tables(store, c.queries)
            with gpu_index(case, store, c.max_degree) as g:
                check(g, store, case, runs_over(tables, Ls=(1, 30)), tables=tables)


@pytest.mark.gpu
def test_deleted_and_reinserted_points():
    rng = np.random.default_rng(5)
    case = gpu_case(F32, O.L2, d=32)
    vecs, adj, n, n_start, metric, qs = case
    gone = rng.choice(n, 200, replace=False).astype(np.uint32)
    deleted = np.zeros(n + 1, bool)
    deleted[gone] = True
    fresh = (vecs[rng.integers(0, n, 200)] + 0.2 * rng.normal(size=(200, vecs.shape[1]))).astype(F32)
    vecs2 = vecs.copy()
    vecs2[gone] = fresh
    for store in three_stores(case):
        tables = store_tables(store, qs)
        runs = runs_over(tables, Ls=(10, 40))
        with gpu_index(case, store) as g:
            g.delete(gone)
            check(g, store, case, runs + [(10, 1, runs[-1][2], dict(max_returned=25))], deleted=deleted, tables=tables)
            g.release(gone)
            g.insert(gone, fresh, 16, 30)
            case2 = (vecs2, g.download_graph(), n, n_start, metric, qs)
            check(g, store, case2, runs, tables=store_tables(encoded(store, vecs2), qs))


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_RANGE_LIST": "3"}, {"DAB_TEST_RANGE_ARENA": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "2", "DAB_TEST_RANGE_ARENA": "5"}])
def test_reruns(monkeypatch, env):
    """tables of 256 slots, in_range regions of a few entries and an arena of a few entries: queries re-run, some
    several times, and every one is answered in full"""
    case = gpu_case(F32, O.L2, d=32)
    for var, val in env.items():
        monkeypatch.setenv(var, val)
    for store in three_stores(case):
        tables = store_tables(store, case[5])
        with gpu_index(case, store) as g:
            check(g, store, case, runs_over(tables, Ls=(1, 10, 40), beams=(1,)), tables=tables)


@pytest.mark.gpu
def test_device_form_snapshot_and_destroy():
    import torch
    case = gpu_case(F32, O.L2, d=32)
    qs = case[5]
    for store in three_stores(case):
        kind = kind_of(store)
        radius = radii_of(store_tables(store, qs), 20)[2]
        g = gpu_index(case, store)
        d_q = torch.from_numpy(qs).cuda()
        for rr in (False, True):
            want = getattr(g, f"range_search_{kind}")(qs, 20, radius, beam_width=2, max_returned=60, rerank=rr)
            with getattr(g, f"range_search_{kind}_device")(d_q.data_ptr(), NQ, 20, radius, beam_width=2, max_returned=60, rerank=rr) as r:
                offsets, cmps, hops, second = r.offsets()
                n = r.total()
                d_ids = torch.empty(n, dtype=torch.int32, device="cuda")
                d_dists = torch.empty(n, dtype=torch.float32, device="cuda")
                r.results_device(d_ids.data_ptr(), d_dists.data_ptr())
                torch.cuda.synchronize()
                same((offsets, d_ids.cpu().numpy(), d_dists.cpu().numpy(), cmps, hops, second), want, (kind, rr, "device form"))
        # a result set is a snapshot: later writes to the index leave it as it was
        r = g._range_quant_device(kind, d_q.data_ptr(), NQ, 20, radius, beam_width=2, max_returned=60, rerank=True)
        g.delete(np.arange(0, case[2], 3, dtype=np.uint32))
        g.upload_vectors(np.zeros_like(case[0]))
        g.upload_graph(np.zeros_like(case[1]))
        offsets, cmps, hops, second = r.offsets()
        same((offsets, *r.results(), cmps, hops, second), want, (kind, "snapshot"))
        r2 = g._range_quant_device(kind, d_q.data_ptr(), NQ, 20, radius)
        g.close()  # dab_destroy releases both open result sets
        for s in (r, r2):
            with pytest.raises(dab.DabError):
                s.offsets()
            s.close()


@pytest.mark.gpu
def test_refusals_before_any_launch():
    case = built(600, 16, F32, O.L2, 16, seed=31)
    vecs, adj, n, n_start, metric, qs = case
    L_ = dab.lib()
    nan = float("nan")

    def fails(code, fn, *args, staged=False, **kw):
        launches = dab.launch_count()
        with pytest.raises(dab.DabError) as e:
            fn(*args, **kw)
        assert e.value.code == code, str(e.value)
        # a NaN after the transform is found by the staging of the queries, before any traversal
        assert staged or dab.launch_count() == launches, ("a refused call launched a kernel", str(e.value))
        return str(e.value)

    pq, sq = pq_store(case, 4), sq_store(case, 8)
    mm = MMStore(vecs, 8, "double_same", O.L2)
    with dab.GpuIndex(dab.DType.f32, O.L2, 16, n, 1, adj.shape[1] - 1) as g:
        calls = [g.range_search_pq, g.range_search_sq, g.range_search_minmax]
        for fn in calls:
            assert "graph must be uploaded first" in fails(NOT_READY, fn, qs, 10, 1.0)
        g.upload_graph(adj)
        # stores never uploaded, or set up without rows: the k-NN calls' messages
        assert "no PQ codes" in fails(NOT_READY, g.range_search_pq, qs, 10, 1.0)
        assert "no scalar-quantized rows" in fails(NOT_READY, g.range_search_sq, qs, 10, 1.0)
        assert "no MinMax rows" in fails(NOT_READY, g.range_search_minmax, qs, 10, 1.0)
        for s in (pq, sq, mm):
            s.upload(g)
        bad = [  # (L, beam, radius, keyword arguments, message): the checks of dab_range_search in the reference's order
            (10, 0, 1.0, {}, "BeamWidthZero"), (0, 1, 1.0, {}, "LZero"), (10, 1, 1.0, dict(max_returned=9), "MaxReturnedLessThanInitialL"),
            (10, 1, 1.0, dict(initial_slack=1.5), "StartingListSlack"), (10, 1, 1.0, dict(initial_slack=nan), "StartingListSlack"),
            (10, 1, 1.0, dict(range_slack=0.5), "RangeSearchSlack"), (10, 1, 1.0, dict(inner_radius=2.0), "InnerRadius"),
            (10, 65, 1.0, {}, "beam_width 65 > 64"), (0, 0, 1.0, dict(inner_radius=2.0, initial_slack=2.0, range_slack=0.0), "BeamWidthZero"),
            (1024, 1, 1.0, {}, "L + #start must be <= 1024"),
        ]
        for fn in calls:
            for L, beam, radius, kw, what in bad:
                assert what in fails(INVALID_ARGUMENT, fn, qs, L, radius, beam_width=beam, **kw)
            # rerank without the full-precision vectors; without rerank the rows are not needed
            assert "rerank needs the full-precision vectors" in fails(NOT_READY, fn, qs, 10, 1.0, rerank=True)
            assert len(fn(qs, 10, 1.0)[0]) == 17
        # the C entry points, host and device forms: nothing is returned
        for name in ("pq", "sq", "minmax"):
            for suffix in ("", "_device"):
                out = ctypes.c_void_p()
                f = getattr(L_, f"dab_range_search_{name}{suffix}")
                assert f(g._h, O.ptr(qs), 16, 10, 0, 1.0, 0, 0.0, 1.0, 1.0, 0, 1, ctypes.byref(out)) == INVALID_ARGUMENT
                assert b"BeamWidthZero" in L_.dab_last_error() and not out.value
        # a MinMax query holding a NaN fails the call, naming it
        badq = qs.copy()
        badq[3, 4] = np.nan
        assert "query 3 contains NaN after the transform (InputContainsNaN)" in fails(INVALID_ARGUMENT, g.range_search_minmax, badq, 10, 1.0,
                                                                                     staged=True)
        g.upload_vectors(vecs)
        for s in (pq, sq, mm):  # the index is usable after every refusal
            tables = store_tables(s, qs)
            check(g, s, case, [(10, 1, radii_of(tables, 10)[2], {})], tables=tables)
    with dab.GpuIndex(dab.DType.f32, O.COSINE, 16, n, 1, adj.shape[1] - 1) as g:
        g.upload_graph(adj)
        sq.upload(g)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(INVALID_ARGUMENT, g.range_search_sq, qs, 10, 1.0)
    # a code row too long for the kernel's shared memory (checked before the store's rows)
    d = 60000
    with dab.GpuIndex(dab.DType.f32, O.L2, d, 10, 1, 8) as g:
        g.upload_graph(np.zeros((11, 9), np.uint32))
        g.upload_sq(8, np.zeros(d, F32), 1.0, 0.0)
        assert "shared memory" in fails(INVALID_ARGUMENT, g.range_search_sq, np.zeros((1, d), F32), 4, 1.0)


@pytest.mark.gpu
def test_results_beyond_the_arena_limit(monkeypatch):
    """a batch whose results, or whose rerank's sort, pass the test hook's limit fails with DAB_ERR_OUT_OF_MEMORY, leaves
    nothing behind and the index usable"""
    case = gpu_case(F32, O.L2, d=32)
    qs = case[5]
    oidx = O.Index(*case[:5])
    for store in three_stores(case):
        tables = store_tables(store, qs)
        big, small = radii_of(tables, 20)[3], radii_of(tables, 20)[1]
        want_big = RT.range_search_table(oidx, tables, qs, 20, big)
        want_small = RT.range_search_table(oidx, tables, qs, 20, small)
        need = int(want_big[0][-1])
        assert need > int(want_small[0][-1]) + 8
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(need - 1))
        monkeypatch.setenv("DAB_TEST_RANGE_ARENA", "4")
        fn = f"range_search_{kind_of(store)}"
        with gpu_index(case, store) as g:
            for rr in (False, True):
                with pytest.raises(dab.DabError) as e:
                    getattr(g, fn)(qs, 20, big, rerank=rr)
                assert e.value.code == OUT_OF_MEMORY, str(e.value)
            assert not g._ranges
            same(getattr(g, fn)(qs, 20, small), want_small, "under the limit")
        # the rerank's sort keys take twice the entries it keeps: a limit that holds the results but not the keys
        want_rr = RT.range_search_table(oidx, tables, qs, 20, big, rerank=True)
        kept = int(want_rr[0][-1])
        assert 2 * kept > need
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(2 * kept - 1))
        with gpu_index(case, store) as g:
            same(getattr(g, fn)(qs, 20, big), want_big, "at the limit")
            with pytest.raises(dab.DabError) as e:
                getattr(g, fn)(qs, 20, big, rerank=True)
            assert e.value.code == OUT_OF_MEMORY, str(e.value)
            assert not g._ranges
            same(getattr(g, fn)(qs, 20, small, rerank=True), RT.range_search_table(oidx, tables, qs, 20, small, rerank=True), "usable")
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(2 * kept))
        with gpu_index(case, store) as g:
            same(getattr(g, fn)(qs, 20, big, rerank=True), want_rr, "the sort at the limit")
        monkeypatch.delenv("DAB_TEST_RANGE_LIMIT")
        monkeypatch.delenv("DAB_TEST_RANGE_ARENA")
