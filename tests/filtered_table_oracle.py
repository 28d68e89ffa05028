"""The filtered search with traversal distances read from a table, and the optional full-precision rerank, over the
unchanged traversal of oracle/filtered_search.cpp.  TEST INFRASTRUCTURE ONLY.

graph::ext::labeled::Filtered wraps any search strategy (labeled.rs:96-129), so InlineFilterSearch runs over a
quantized store's distances too.  orc_search_batch_filtered reads its distances from the index's rows; here each query
gets a one-dimensional InnerProduct view of the same graph whose row i is table[q][i] and whose query is -1.0.  Its
distance to row i is then -(-1 * table[q][i]): negation and a product by -1 are exact, so the traversal sees the table's
values (up to the sign of a zero, which the traversal and the matched list treat as equal; NaN stays NaN).  The
returned distances are looked up in the table by id, so their bits are the table's.  With rerank the first L matches
(start points and deleted ids dropped, matched-list order) get their full-precision Distance<T, T> to the query and the
first k in stable order of it are kept: Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-400,
full_precision.rs:356-399)."""
import numpy as np

import filtered_oracle as F
import oracle_lib as O

EMPTY = 0xFFFFFFFF
_MINUS_ONE = np.array([[-1.0]], np.float32)


def search_batch_table(index, tables, queries, k, l_search, labels, masks, match_all=False, adaptive_l=None, beam=1, deleted=None,
                       rerank=False, flavour=O.AVX2):
    """InlineFilterSearch over an O.Index with the traversal distance of query q to id i tables[q][i] (f32, one row per
    query over every id); with `rerank` the first L matches are reranked by full-precision distance to `queries` (index
    dtype).  Other arguments and the result as filtered_oracle.search_batch: (ids, dists, counts, cmps, hops)."""
    tables = np.ascontiguousarray(tables, np.float32)
    total = index.n_points + index.n_start
    nq = tables.shape[0]
    assert tables.shape == (nq, total)
    masks = np.broadcast_to(np.asarray(masks, np.uint64), (nq,))
    assert not rerank or (queries is not None and len(queries) == nq)
    ids = np.full((nq, k), EMPTY, np.uint32)
    dists = np.full((nq, k), np.inf, np.float32)
    counts, cmps, hops = (np.zeros(nq, np.uint32) for _ in range(3))
    for q in range(nq):
        view = O.Index(tables[q][:, None], index.adj, index.n_points, index.n_start, O.INNER_PRODUCT)
        # the first L matches, start points and deleted ids dropped, in matched-list order
        m_ids, _, m_count, m_cmps, m_hops = F.search_batch(view, _MINUS_ONE, l_search, l_search, labels, masks[q], match_all, adaptive_l,
                                                           beam, deleted, flavour)
        cmps[q], hops[q] = m_cmps[0], m_hops[0]
        kept = m_ids[0, :m_count[0]]
        d = tables[q][kept.astype(np.int64)]
        if rerank:
            query = np.ascontiguousarray(queries[q], index.vectors.dtype)
            d = O.distance_rows(query, index.vectors[kept.astype(np.int64)], index.metric, flavour)
            order = np.argsort(d, kind="stable")
            kept, d = kept[order], d[order]
        c = min(k, len(kept))
        ids[q, :c], dists[q, :c], counts[q] = kept[:c], d[:c], c
    return ids, dists, counts, cmps, hops
