"""The filtered range search with distances read from a table, and the optional full-precision rerank, over the unchanged
search of oracle/filtered_range_search.cpp.  TEST INFRASTRUCTURE ONLY.

graph::ext::labeled::Filtered wraps any search strategy (labeled.rs:96-129), so FilteredRange::search runs over a
quantized store's distances too: both phases read the strategy's accessor.  orc_filtered_range_search reads its
distances from the index's rows; here each query gets a one-dimensional InnerProduct view of the same graph whose row i
is table[q][i] and whose query is -1.0, the view filtered_table_oracle.py uses.  Its distance to row i is -(-1 *
table[q][i]): negation and a product by -1 are exact, so both phases see the table's values (up to the sign of a zero,
which the search treats as equal; NaN stays NaN).  The returned distances are looked up in the table by id, so their
bits are the table's.

With rerank the search runs without an inner radius, so its output is matched.take(max_returned) without start points
and deleted ids.  The quantized strategies' Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-401,
full_precision.rs:356-399) then gives each id its full-precision Distance<T, T> to the query and sorts by it, stably
(ties in matched order, -0.0 equal to +0.0, NaN after every number), and FilteredRange::search drops the ids with d <=
inner_radius (filtered_range_search.rs:230-245).  Nothing drops the ids above the radius: unlike Range::search, it
checks only the inner radius."""
import numpy as np

import filtered_range_oracle as FR
import oracle_lib as O

_MINUS_ONE = np.array([[-1.0]], np.float32)


def rerank_sorted(query, vecs, metric, ids, inner_radius, flavour=O.AVX2):
    """ids by their full-precision distance to `query`: sorted stably (NaN last, -0.0 == +0.0), those with d <=
    inner_radius (when given) dropped: (ids, dists)"""
    ids = np.asarray(ids, np.uint32)
    d = O.distance_rows(query, vecs[ids.astype(np.int64)], metric, flavour) if len(ids) else np.empty(0, np.float32)
    order = np.argsort(np.where(d == 0, np.float32(0.0), d), kind="stable")  # numpy sorts NaN after every number
    ids, d = ids[order], d[order]
    if inner_radius is not None:
        with np.errstate(invalid="ignore"):
            keep = ~(d <= np.float32(inner_radius))
        ids, d = ids[keep], d[keep]
    return ids, d


def range_search_table(index, tables, queries, l_search, radius, labels, masks, match_all=False, beam=1, inner_radius=None,
                       initial_slack=1.0, range_slack=1.0, max_returned=None, deleted=None, rerank=False, flavour=O.AVX2):
    """FilteredRange::search over an O.Index with the distance of query q to id i tables[q][i] (f32, one row per query over
    every id); with `rerank` the results are reranked by full-precision distance to `queries` (index dtype).  Other
    arguments and the result as filtered_range_oracle.range_search: (offsets, ids, dists, cmps, hops, second_round)."""
    tables = np.ascontiguousarray(tables, np.float32)
    total = index.n_points + index.n_start
    nq = tables.shape[0]
    assert tables.shape == (nq, total)
    masks = np.broadcast_to(np.asarray(masks, np.uint64), (nq,))
    assert not rerank or (queries is not None and len(queries) == nq)
    cmps, hops, second = np.empty(nq, np.uint32), np.empty(nq, np.uint32), np.empty(nq, np.uint8)
    offsets, all_ids, all_dists = [0], [], []
    for q in range(nq):
        view = O.Index(tables[q][:, None], index.adj, index.n_points, index.n_start, O.INNER_PRODUCT)
        _, ids, _, c, h, s = FR.range_search(view, _MINUS_ONE, l_search, radius, labels, masks[q], match_all, beam=beam,
                                             inner_radius=None if rerank else inner_radius, initial_slack=initial_slack,
                                             range_slack=range_slack, max_returned=max_returned, deleted=deleted, flavour=flavour)
        cmps[q], hops[q], second[q] = c[0], h[0], s[0]
        d = tables[q][ids.astype(np.int64)]
        if rerank:
            query = np.ascontiguousarray(queries[q], index.vectors.dtype)
            ids, d = rerank_sorted(query, index.vectors, index.metric, ids, inner_radius, flavour)
        all_ids.append(ids)
        all_dists.append(d)
        offsets.append(offsets[-1] + len(ids))
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.empty(0, dt)
    return np.array(offsets, np.uint64), cat(all_ids, np.uint32), cat(all_dists, np.float32), cmps, hops, second
