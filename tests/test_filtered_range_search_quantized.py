"""Filtered range search over the PQ, SQ and MinMax stores: dab_range_search_filtered_{pq,sq,minmax}[_device].

The reference's FilteredRange::search is generic over any strategy whose accessor is a FilteredAccessor, and
graph::ext::labeled::Filtered wraps the quantized strategies with their post-processor (labeled.rs:118-129).  Both phases
read the strategy's accessor, so every distance is the store's.  Without rerank the output is the full-precision rule on
the store's distances; with rerank (Pipeline<FilterStartPoints, Rerank>) matched.take(max_returned) loses its start
points and deleted ids, each id gets its full-precision distance, the ids are sorted by it and those with d <=
inner_radius are dropped.  No outer-radius filter follows, unlike Range::search: ids above the radius, and NaN, stay.

CPU: the table oracle (tests/filtered_range_table_oracle.py: the unchanged orc_filtered_range_search over a
one-dimensional view whose distances are the table's) fed the full-precision distances equals
orc_filtered_range_search bit for bit — offsets, ids, distance bits, order, cmps, hops and the second-round flag — over
the reference's seven baselines, every row type and metric, selectivities from every id to none in both modes, L from 1
to 300, beams 1, 4 and 64, the argument grid of test_range_search_quantized.py, edge graphs and deletions; with rerank it
equals an independent restatement of the rule, exact ties, ±0, ±inf and NaN rows included, and keeps ids whose
full-precision distance lies above the radius.
GPU: the device equals the oracle fed each store's exhaustive distances bit for bit, with rerank 0 and 1, over every PQ
table kind and chunk layout, every SQ and MinMax width, metric and transform, every row type, the selectivity / mode / L /
beam / argument grid, edge graphs, deletions and re-inserted ids, the forced re-runs of visited tables, regions and the
arena; the device form, result sets across dab_destroy, every refusal in order before any launch, a MinMax NaN query and
the out-of-memory path."""
import ctypes
import functools
import json

import numpy as np
import pytest

import diskann_b200 as dab
import filtered_range_oracle as FR
import filtered_range_table_oracle as FRT
import oracle_lib as O
from test_diverse_search_quantized import encoded, fp_tables, store_tables
from test_filtered_range_search import GOLDEN, golden_labels, labels_for
from test_gpu_parity import make_index
from test_oracle_golden import grid as lattice
from test_paged_search import built
from test_paged_search_quantized import MMStore, PQStore, SQStore, pq_store, sq_store
from test_range_search_quantized import argument_grid, radii_of, same as same_bits
from test_traversal_edges import grid as tie_grid, malformed_case, many_starts, non_finite

F32 = np.float32
INVALID_ARGUMENT, OUT_OF_MEMORY, NOT_READY = 1, 3, 5
SELECTIVITIES = (1.0, 0.5, 0.1, 0.01, 0.0)


def same(got, want, what):
    """offsets, ids, distance bits, cmps, hops and second-round flags equal, every NaN distance taken as one value: a
    reranked NaN stays in the results (FilteredRange::search has no outer-radius filter), and the device computes the
    canonical NaN where x86 propagates a NaN operand's payload"""
    got, want = list(got), list(want)
    for x in (got, want):
        if x[2] is not None:
            d = np.array(x[2], F32)
            d[np.isnan(d)] = np.nan
            x[2] = d
    same_bits(got, want, what)


def masks_of(rng, nq):
    """most queries ANY of bit 0 (labels_for's share), some ANY of bits 0 and 1"""
    return np.where(rng.random(nq) < 0.8, 1, 0b11).astype(np.uint64)


def grid_runs(rng, tables, total, Ls=(1, 10, 40), beams=(1, 4), selectivities=SELECTIVITIES):
    """(L, beam, radius, labels, masks, match_all, keyword arguments): radii at the table's ranks, every selectivity, ANY
    and ALL"""
    runs = []
    nq = tables.shape[0]
    for s in selectivities:
        labels = labels_for(rng, total, s)
        masks = masks_of(rng, nq)
        for L in Ls:
            for i, r in enumerate(radii_of(tables, max(L, 2))):
                runs.append((L, beams[i % len(beams)], r, labels, masks, False, {}))
        runs.append((Ls[-1], beams[-1], r, labels, np.uint64(0b11), True, {}))  # ALL of two bits
    return runs


# ---------------------------------------------------------------- CPU

def table_equals_search(oidx, queries, tables, runs, deleted=None):
    second = 0
    for L, beam, radius, labels, masks, match_all, kw in runs:
        want = FR.range_search(oidx, queries, L, radius, labels, masks, match_all, beam=beam, deleted=deleted, **kw)
        got = FRT.range_search_table(oidx, tables, None, L, radius, labels, masks, match_all, beam=beam, deleted=deleted, **kw)
        same(got, want, (L, beam, radius, match_all, kw))
        second += int(want[5].sum())
    return second


def test_table_of_full_precision_distances_reproduces_the_baselines():
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) == 7
    for c in cases:
        data, adj, n = lattice(c["grid_dims"], c["grid_size"])
        labels = golden_labels(c["filter"], n + 1)
        q = np.array([c["query"]], F32)
        oidx = O.Index(data, adj, n, 1, O.L2)
        kw = dict(inner_radius=c["inner_radius"], max_returned=c["max_returned"])
        got = FRT.range_search_table(oidx, fp_tables(data, O.L2, q), None, c["starting_l"], c["radius"], labels, 1, **kw)
        assert (int(got[0][1]), int(got[3][0]), int(got[4][0]), bool(got[5][0])) == (
            c["result_count"], c["comparisons"], c["hops"], c["range_search_second_round"]), c["case"]
        same(got, FR.range_search(oidx, q, c["starting_l"], c["radius"], labels, 1, **kw), c["case"])


@pytest.mark.parametrize("dt", [F32, np.float16, np.int8, np.uint8])
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED])
def test_table_of_full_precision_distances_is_the_filtered_range_search(dt, metric):
    rng = np.random.default_rng(7)
    vecs, adj, maxdeg = make_index(rng, dt, metric, 400, 16, 12, 24)
    queries = vecs[rng.integers(0, 400, 6)]
    oidx = O.Index(vecs, adj, 400, 1, metric)
    tables = fp_tables(vecs, metric, queries)
    table_equals_search(oidx, queries, tables, grid_runs(rng, tables, 401, Ls=(1, 12), selectivities=(1.0, 0.3, 0.0)))


@pytest.mark.parametrize("beam", [1, 4, 64])
def test_selectivities_lists_and_beams(beam):
    rng = np.random.default_rng(beam)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 800, 16, 12, 24)
    queries = (vecs[rng.integers(0, 800, 6)] + 0.1 * rng.normal(size=(6, 16))).astype(F32)
    oidx = O.Index(vecs, adj, 800, 1, O.L2)
    tables = fp_tables(vecs, O.L2, queries)
    assert table_equals_search(oidx, queries, tables, grid_runs(rng, tables, 801, Ls=(1, 2, 64, 300), beams=(beam,))) > 0


def test_every_argument_the_reference_accepts():
    rng = np.random.default_rng(4)
    vecs, adj, maxdeg = make_index(rng, F32, O.L2, 500, 16, 12, 24)
    queries = (vecs[rng.integers(0, 500, 6)] + 0.1 * rng.normal(size=(6, 16))).astype(F32)
    oidx = O.Index(vecs, adj, 500, 1, O.L2)
    tables = fp_tables(vecs, O.L2, queries)
    labels = labels_for(rng, 501, 0.4)
    runs = [(L, beam, r, labels, masks_of(rng, 6), False, kw) for L, beam, r, kw in argument_grid(radii_of(tables, 12), 12)]
    table_equals_search(oidx, queries, tables, runs)


def edge_cases(nq):
    cases = [many_starts(300, 8, 2, nq, 2), many_starts(300, 8, 40, nq, 40), tie_grid(300, 6, 3, nq, 3)]
    cases += [malformed_case(150, 6, 3, md, nq, md) for md in (1, 7, 40)]
    cases += [non_finite(200, 8, dt, m, nq, 7, nan=dt == F32)[0] for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2))]
    return cases


def test_edge_graphs_and_deletions():
    rng = np.random.default_rng(9)
    for case in edge_cases(6):
        tables = fp_tables(case.vecs, case.metric, case.queries)
        runs = grid_runs(rng, tables, case.total, Ls=(1, 12), selectivities=(1.0, 0.5, 0.0))
        table_equals_search(case.oracle, case.queries, tables, runs)
        deleted = np.zeros(case.total, bool)
        deleted[::5] = True
        table_equals_search(case.oracle, case.queries, tables, grid_runs(rng, tables, case.total, Ls=(12,), beams=(2,)), deleted)


def rerank_rule(vecs, metric, query, matched, inner_radius):
    """Pipeline<FilterStartPoints, Rerank> under FilteredRange::search, restated: the returned matches (start points and
    deleted ids already out) by full-precision distance in a stable sort with NaN last and -0.0 == +0.0, the ids with d
    <= inner_radius dropped, nothing dropped for being above the radius"""
    ids = [int(i) for i in matched]
    fp = O.distance_rows(query, vecs[np.asarray(ids, np.int64)], metric, O.AVX2) if ids else np.empty(0, F32)
    pairs = sorted(zip(ids, fp.tolist()), key=lambda p: (p[1] != p[1], 0.0 if p[1] != p[1] else p[1]))  # stable
    out = [(i, d) for i, d in pairs if not (inner_radius is not None and d <= float(F32(inner_radius)))]
    return np.array([i for i, _ in out], np.uint32), np.array([d for _, d in out], F32)


def check_rerank_rule(oidx, vecs, metric, queries, tables, runs, deleted=None):
    """returns how many reranked results lie above the radius"""
    above = 0
    for L, beam, radius, labels, masks, inner in runs:
        # without an inner radius the output is matched.take(max_returned) without start points and deleted ids
        base = FRT.range_search_table(oidx, tables, None, L, radius, labels, masks, beam=beam, deleted=deleted)
        got = FRT.range_search_table(oidx, tables, queries, L, radius, labels, masks, beam=beam, deleted=deleted, rerank=True,
                                     inner_radius=inner)
        same((None, None, None, *got[3:]), (None, None, None, *base[3:]), (L, beam, radius, inner))
        for q in range(queries.shape[0]):
            a, b = int(base[0][q]), int(base[0][q + 1])
            w_ids, w_d = rerank_rule(vecs, metric, queries[q], base[1][a:b], inner)
            c, d = int(got[0][q]), int(got[0][q + 1])
            assert np.array_equal(got[1][c:d], w_ids), (L, beam, radius, inner, q)
            assert np.array_equal(got[2][c:d].view(np.uint32), w_d.view(np.uint32)), (L, beam, radius, inner, q)
            with np.errstate(invalid="ignore"):
                above += int((~(w_d <= F32(radius))).sum())
    return above


@pytest.mark.parametrize("kind", ["pq", "sq", "mm"])
def test_rerank_is_the_rule_over_each_store(kind):
    case = built(600, 16, F32, O.L2, 8, seed=5)
    vecs, adj, n, n_start, metric, qs = case
    store = pq_store(case, 4) if kind == "pq" else sq_store(case, 4) if kind == "sq" else MMStore(vecs, 4, "double_same", metric)
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs)
    rng = np.random.default_rng(3)
    deleted = np.zeros(n + n_start, bool)
    deleted[::7] = True
    runs = [(L, beam, r, labels_for(rng, n + n_start, s), masks_of(rng, 8), inner) for L in (10, 40) for beam in (1, 4)
            for r in radii_of(tables, L)[1:] for s in (0.5, 0.1) for inner in (None, r / 3)]
    above = sum(check_rerank_rule(oidx, vecs, metric, qs, tables, runs, dl) for dl in (None, deleted))
    assert above > 0, "no reranked distance above the radius: the missing outer filter is untested"


def test_rerank_rule_on_ties_signed_zeros_and_non_finite_rows():
    rng = np.random.default_rng(2)
    # exact ties all along the list
    c = tie_grid(300, 6, 3, 6, 3)
    tables = (np.round(fp_tables(c.vecs, c.metric, c.queries) / 4) * 4).astype(F32)  # coarser ties in the traversal too
    lab = labels_for(rng, c.total, 0.6)
    check_rerank_rule(c.oracle, c.vecs, c.metric, c.queries, tables, [(12, 1, 40.0, lab, 1, None), (30, 4, 60.0, lab, 0b11, 8.0)])
    # inner products of zero rows: -0.0, tied with +0.0 rows of the same distance
    vecs, adj, maxdeg = make_index(rng, F32, O.INNER_PRODUCT, 300, 8, 12, 24)
    vecs = vecs.copy()
    vecs[::9] = 0.0
    vecs[1::9] = -0.0
    queries = vecs[rng.integers(0, 300, 6)] + 0.1
    oidx = O.Index(vecs, adj, 300, 1, O.INNER_PRODUCT)
    tables = fp_tables(vecs, O.INNER_PRODUCT, queries)
    assert np.signbit(tables[tables == 0]).any()
    lab = labels_for(rng, 301, 0.7)
    check_rerank_rule(oidx, vecs, O.INNER_PRODUCT, queries, tables, [(20, 1, 0.0, lab, 1, None), (20, 2, 1.0, lab, 1, None),
                                                                       (20, 1, 1.0, lab, 1, -1.0)])
    # ±inf and NaN rows: the traversal sees finite store distances, the rerank the rows as they are; NaN and +inf stay,
    # NaN after every number
    nan_kept = 0
    for dt, m in ((F32, O.L2), (F32, O.INNER_PRODUCT), (np.float16, O.L2)):
        c = non_finite(200, 8, dt, m, 6, 7, nan=dt == F32)[0]
        tables = np.nan_to_num(fp_tables(c.vecs, c.metric, c.queries), nan=1.0, posinf=2.0, neginf=-2.0).astype(F32)
        lab = labels_for(rng, c.total, 0.8)
        runs = [(12, 1, 1.5, lab, 1, None), (12, 4, 3.0, lab, 1, 0.5)]
        check_rerank_rule(c.oracle, c.vecs, c.metric, c.queries, tables, runs)
        got = FRT.range_search_table(c.oracle, tables, c.queries, 12, 3.0, lab, 1, beam=4, rerank=True)
        nan_kept += int(np.isnan(got[2]).sum())
        for q in range(c.queries.shape[0]):
            d = got[2][int(got[0][q]):int(got[0][q + 1])]
            assert not np.isnan(d[:int((~np.isnan(d)).sum())]).any(), "NaN before a number"
    assert nan_kept > 0, "no NaN full-precision distance was returned"


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
    """every (L, beam, radius, labels, masks, match_all, keyword arguments) of `runs`, with and without rerank, on the
    device against the oracle fed the store's distances; returns how many queries took the second round"""
    vecs, adj, n, n_start, metric, qs = case[:6]
    oidx = O.Index(vecs, adj, n, n_start, metric)
    tables = store_tables(store, qs) if tables is None else tables
    fn = getattr(g, f"range_search_filtered_{kind_of(store)}")
    second, last = 0, None
    for L, beam, radius, labels, masks, match_all, kw in runs:
        if labels is not last:
            g.upload_labels(labels)
            last = labels
        for rr in reranks:
            want = FRT.range_search_table(oidx, tables, qs, L, radius, labels, masks, match_all, beam=beam, deleted=deleted, rerank=rr, **kw)
            got = fn(qs, masks, L, radius, match_all=match_all, beam_width=beam, rerank=rr, **kw)
            same(got, want, (kind_of(store), L, beam, radius, match_all, kw, rr))
            second += int(want[5].sum())
    return second


NQ = 100


@functools.lru_cache(maxsize=None)
def gpu_case(dt, metric, d=64):
    return built(2000, d, dt, metric, NQ, seed=43 + d)


def run_store(case, store, Ls=(1, 10, 40), beams=(1, 4), selectivities=(0.5, 0.05)):
    tables = store_tables(store, case[5])
    rng = np.random.default_rng(len(Ls) * 10 + len(selectivities))
    with gpu_index(case, store) as g:
        assert check(g, store, case, grid_runs(rng, tables, case[2] + case[3], Ls, beams, selectivities), tables=tables) > 0, "no second round"


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [(F32, O.L2), (np.int8, O.INNER_PRODUCT), (np.float16, O.COSINE), (np.uint8, O.COSINE_NORMALIZED)])
@pytest.mark.parametrize("chunks", [16, 8, 7])  # chunks of 4, of 8, of 9 and 10
def test_pq_equals_the_oracle(dt, metric, chunks):
    case = gpu_case(dt, metric)
    run_store(case, pq_store(case, chunks), Ls=(1, 10, 40) if chunks == 16 else (10,))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_sq_equals_the_oracle(nbits, metric):
    dt = {8: F32, 4: np.float16, 2: np.int8, 1: np.uint8}[nbits]
    case = gpu_case(dt, metric)
    run_store(case, sq_store(case, nbits), Ls=(10,))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED])
@pytest.mark.parametrize("nbits", [8, 4, 2, 1])
def test_minmax_equals_the_oracle(nbits, metric):
    dt = {8: F32, 4: np.float16, 2: np.uint8, 1: np.int8}[nbits]
    case = gpu_case(dt, metric, d=48)  # 48: PaddingHadamard pads to 64
    for kind in (None, "padding_natural", "double_same"):
        run_store(case, MMStore(case[0], nbits, kind, metric), Ls=(10,), selectivities=(0.3,))


def three_stores(case):
    return [pq_store(case, 8), sq_store(case, 8), MMStore(case[0], 8, "double_same", case[4])]


@pytest.mark.gpu
def test_selectivity_mode_lists_and_beams():
    case = gpu_case(F32, O.L2, d=32)
    for store in three_stores(case):
        run_store(case, store, Ls=(1, 2, 64, 300), beams=(1, 4, 64), selectivities=SELECTIVITIES)


@pytest.mark.gpu
def test_every_argument_the_reference_accepts():
    case = gpu_case(F32, O.L2, d=32)
    rng = np.random.default_rng(12)
    labels = labels_for(rng, case[2] + case[3], 0.4)
    for store in three_stores(case):
        tables = store_tables(store, case[5])
        runs = [(L, beam, r, labels, masks_of(rng, NQ), False, kw) for L, beam, r, kw in argument_grid(radii_of(tables, 20), 20)]
        with gpu_index(case, store) as g:
            check(g, store, case, runs, tables=tables)


def as_tuple(c):
    return (c.vecs, c.adj, c.n, c.n_start, c.metric, c.queries)


@pytest.mark.gpu
def test_edge_graphs():
    rng = np.random.default_rng(7)
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
                check(g, store, case, grid_runs(rng, tables, c.total, Ls=(1, 30), selectivities=(1.0, 0.5, 0.0)), tables=tables)


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
        runs = grid_runs(rng, tables, n + 1, Ls=(10, 40), selectivities=(1.0, 0.3))
        with gpu_index(case, store) as g:
            g.delete(gone)
            check(g, store, case, runs + [(10, 1, runs[-1][2], runs[-1][3], 1, False, dict(max_returned=25))], deleted=deleted, tables=tables)
            g.release(gone)
            g.insert(gone, fresh, 16, 30)
            case2 = (vecs2, g.download_graph(), n, n_start, metric, qs)
            check(g, store, case2, runs, tables=store_tables(encoded(store, vecs2), qs))


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"DAB_TEST_VISITED_LOG2": "8"}, {"DAB_TEST_RANGE_LIST": "3"}, {"DAB_TEST_RANGE_ARENA": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "1"},
                                 {"DAB_TEST_VISITED_LOG2": "8", "DAB_TEST_RANGE_LIST": "2", "DAB_TEST_RANGE_ARENA": "5"}])
def test_reruns(monkeypatch, env):
    """tables of 256 slots, regions of matches (and frontiers of L more) of a few entries, an arena of a few entries:
    queries re-run, some several times, and every one is answered in full"""
    case = gpu_case(F32, O.L2, d=32)
    for var, val in env.items():
        monkeypatch.setenv(var, val)
    for store in three_stores(case):
        tables = store_tables(store, case[5])
        with gpu_index(case, store) as g:
            check(g, store, case, grid_runs(np.random.default_rng(11), tables, case[2] + 1, Ls=(1, 10, 40), beams=(1,),
                                            selectivities=(1.0, 0.2)), tables=tables)


@pytest.mark.gpu
def test_device_form_snapshot_and_destroy():
    import torch
    case = gpu_case(F32, O.L2, d=32)
    qs = case[5]
    rng = np.random.default_rng(2)
    labels = labels_for(rng, case[2] + 1, 0.3)
    masks = np.where(np.arange(NQ) % 3 == 0, 0b11, 1).astype(np.uint64)
    for store in three_stores(case):
        kind = kind_of(store)
        radius = radii_of(store_tables(store, qs), 20)[2]
        g = gpu_index(case, store)
        g.upload_labels(labels)
        d_q = torch.from_numpy(qs).cuda()
        d_m = torch.from_numpy(masks.view(np.int64)).cuda()
        device = getattr(g, f"range_search_filtered_{kind}_device")
        for rr in (False, True):
            want = getattr(g, f"range_search_filtered_{kind}")(qs, masks, 20, radius, beam_width=2, max_returned=60, rerank=rr)
            with device(d_q.data_ptr(), d_m.data_ptr(), NQ, 20, radius, beam_width=2, max_returned=60, rerank=rr) as r:
                offsets, cmps, hops, second = r.offsets()
                n = r.total()
                d_ids = torch.empty(n, dtype=torch.int32, device="cuda")
                d_dists = torch.empty(n, dtype=torch.float32, device="cuda")
                r.results_device(d_ids.data_ptr(), d_dists.data_ptr())
                torch.cuda.synchronize()
                same((offsets, d_ids.cpu().numpy(), d_dists.cpu().numpy(), cmps, hops, second), want, (kind, rr, "device form"))
        # a result set is a snapshot: later writes to the index leave it as it was
        r = device(d_q.data_ptr(), d_m.data_ptr(), NQ, 20, radius, beam_width=2, max_returned=60, rerank=True)
        g.delete(np.arange(0, case[2], 3, dtype=np.uint32))
        g.upload_labels(np.zeros(case[2] + 1, np.uint64))
        g.upload_vectors(np.zeros_like(case[0]))
        g.upload_graph(np.zeros_like(case[1]))
        offsets, cmps, hops, second = r.offsets()
        same((offsets, *r.results(), cmps, hops, second), want, (kind, "snapshot"))
        r2 = device(d_q.data_ptr(), d_m.data_ptr(), NQ, 20, radius)
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
    labels = labels_for(np.random.default_rng(1), n + 1, 0.5)

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
        calls = [g.range_search_filtered_pq, g.range_search_filtered_sq, g.range_search_filtered_minmax]
        for fn in calls:
            assert "graph must be uploaded first" in fails(NOT_READY, fn, qs, 1, 10, 1.0)
        g.upload_graph(adj)
        bad = [  # (L, beam, radius, keyword arguments, message): the checks of dab_range_search_filtered in its order
            (10, 0, 1.0, {}, "BeamWidthZero"), (0, 1, 1.0, {}, "LZero"), (10, 1, 1.0, dict(max_returned=9), "MaxReturnedLessThanInitialL"),
            (10, 1, 1.0, dict(initial_slack=1.5), "StartingListSlack"), (10, 1, 1.0, dict(initial_slack=nan), "StartingListSlack"),
            (10, 1, 1.0, dict(range_slack=0.5), "RangeSearchSlack"), (10, 1, 1.0, dict(inner_radius=2.0), "InnerRadius"),
            (10, 65, 1.0, {}, "beam_width 65 > 64"), (0, 0, 1.0, dict(inner_radius=2.0, initial_slack=2.0, range_slack=0.0), "BeamWidthZero"),
        ]
        for fn in calls:
            for L, beam, radius, kw, what in bad:  # before the label table and the store
                assert what in fails(INVALID_ARGUMENT, fn, qs, 1, L, radius, beam_width=beam, **kw)
            # the label table before the store
            assert "no label table" in fails(INVALID_ARGUMENT, fn, qs, 1, 10, 1.0)
        g.upload_labels(labels)
        for fn in calls:
            # L + #start before the store
            assert "L + #start = 1025 > 1024" in fails(INVALID_ARGUMENT, fn, qs, 1, 1024, 1.0)
        # stores never uploaded, or set up without rows: the k-NN calls' messages
        assert "no PQ codes" in fails(NOT_READY, g.range_search_filtered_pq, qs, 1, 10, 1.0)
        assert "no scalar-quantized rows" in fails(NOT_READY, g.range_search_filtered_sq, qs, 1, 10, 1.0)
        assert "no MinMax rows" in fails(NOT_READY, g.range_search_filtered_minmax, qs, 1, 10, 1.0)
        for s in (pq, sq, mm):
            s.upload(g)
        for fn in calls:
            # rerank without the full-precision vectors, naming the call; without rerank the rows are not needed
            msg = fails(NOT_READY, fn, qs, 1, 10, 1.0, rerank=True)
            assert "rerank needs the full-precision vectors" in msg and "dab_" + fn.__name__ in msg, msg
            assert len(fn(qs, 1, 10, 1.0)[0]) == 17
        # the C entry points, host and device forms: nothing is returned
        masks = np.ones(16, np.uint64)
        for name in ("pq", "sq", "minmax"):
            for suffix in ("", "_device"):
                out = ctypes.c_void_p()
                f = getattr(L_, f"dab_range_search_filtered_{name}{suffix}")
                assert f(g._h, O.ptr(qs), 16, 10, 0, 1.0, 0, 0.0, 1.0, 1.0, 0, O.ptr(masks), 0, 1, ctypes.byref(out)) == INVALID_ARGUMENT
                assert b"BeamWidthZero" in L_.dab_last_error() and not out.value
        assert not g._ranges
        # a MinMax query holding a NaN fails the call, naming it
        badq = qs.copy()
        badq[3, 4] = np.nan
        msg = fails(INVALID_ARGUMENT, g.range_search_filtered_minmax, badq, 1, 10, 1.0, staged=True)
        assert "dab_range_search_filtered_minmax: query 3 contains NaN after the transform (InputContainsNaN)" in msg, msg
        g.upload_vectors(vecs)
        for s in (pq, sq, mm):  # the index is usable after every refusal
            tables = store_tables(s, qs)
            check(g, s, case, [(10, 1, radii_of(tables, 10)[2], labels, 1, False, {})], tables=tables)
    with dab.GpuIndex(dab.DType.f32, O.COSINE, 16, n, 1, adj.shape[1] - 1) as g:
        g.upload_graph(adj)
        g.upload_labels(labels)
        sq.upload(g)
        # SQStore::distance_computer: UnsupportedDistanceMetric
        assert "supports L2, InnerProduct and CosineNormalized" in fails(INVALID_ARGUMENT, g.range_search_filtered_sq, qs, 1, 10, 1.0)
    # the filtered kernel's shared memory with the store's query area: 16000 f32 (the full-precision and the PQ query) do
    # not fit four warps, their 8-bit SQ code row does; 60000 do not fit either way
    for d, sq_fits in ((16000, True), (60000, False)):
        with dab.GpuIndex(dab.DType.f32, O.L2, d, 10, 1, 8) as g:
            g.upload_vectors(np.zeros((11, d), F32))
            g.upload_graph(np.zeros((11, 9), np.uint32))
            g.upload_labels(np.ones(11, np.uint64))
            g.upload_sq(8, np.zeros(d, F32), 1.0, 0.0)
            g.sq_encode_all()
            z = np.zeros((2, d), F32)
            if sq_fits:  # (the graph has no edges: only the start point, which is never returned, is evaluated)
                assert g.range_search_filtered_sq(z, 1, 4, 1.0)[0].tolist() == [0, 0, 0]
            else:
                assert "shared memory" in fails(INVALID_ARGUMENT, g.range_search_filtered_sq, z, 1, 4, 1.0)
            assert "shared memory" in fails(INVALID_ARGUMENT, g.range_search_filtered, z, 1, 4, 1.0)


@pytest.mark.gpu
def test_results_beyond_the_arena_limit(monkeypatch):
    """a batch whose results, or whose rerank's sort, pass the test hook's limit fails with DAB_ERR_OUT_OF_MEMORY, leaves
    nothing behind and the index usable"""
    case = gpu_case(F32, O.L2, d=32)
    qs = case[5]
    oidx = O.Index(*case[:5])
    labels = labels_for(np.random.default_rng(4), case[2] + 1, 0.7)
    for store in three_stores(case):
        tables = store_tables(store, qs)
        big, small = radii_of(tables, 20)[3], radii_of(tables, 20)[1]
        want_big = FRT.range_search_table(oidx, tables, qs, 20, big, labels, 1)
        want_small = FRT.range_search_table(oidx, tables, qs, 20, small, labels, 1)
        need = int(want_big[0][-1])
        assert need > int(want_small[0][-1]) + 8
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(need - 1))
        monkeypatch.setenv("DAB_TEST_RANGE_ARENA", "4")
        fn = f"range_search_filtered_{kind_of(store)}"
        with gpu_index(case, store) as g:
            g.upload_labels(labels)
            for rr in (False, True):
                with pytest.raises(dab.DabError) as e:
                    getattr(g, fn)(qs, 1, 20, big, rerank=rr)
                assert e.value.code == OUT_OF_MEMORY, str(e.value)
            assert not g._ranges
            same(getattr(g, fn)(qs, 1, 20, small), want_small, "under the limit")
        # the rerank's sort keys take twice the entries it keeps: a limit that holds the results but not the keys
        want_rr = FRT.range_search_table(oidx, tables, qs, 20, big, labels, 1, rerank=True)
        kept = int(want_rr[0][-1])
        assert 2 * kept > need
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(2 * kept - 1))
        with gpu_index(case, store) as g:
            g.upload_labels(labels)
            same(getattr(g, fn)(qs, 1, 20, big), want_big, "at the limit")
            with pytest.raises(dab.DabError) as e:
                getattr(g, fn)(qs, 1, 20, big, rerank=True)
            assert e.value.code == OUT_OF_MEMORY, str(e.value)
            assert not g._ranges
            same(getattr(g, fn)(qs, 1, 20, small, rerank=True), FRT.range_search_table(oidx, tables, qs, 20, small, labels, 1, rerank=True),
                 "usable")
        monkeypatch.setenv("DAB_TEST_RANGE_LIMIT", str(2 * kept))
        with gpu_index(case, store) as g:
            g.upload_labels(labels)
            same(getattr(g, fn)(qs, 1, 20, big, rerank=True), want_rr, "the sort at the limit")
        monkeypatch.delenv("DAB_TEST_RANGE_LIMIT")
        monkeypatch.delenv("DAB_TEST_RANGE_ARENA")
