"""ctypes binding of oracle/diverse_table.cpp (liboracle_diverse_table.so, oracle/diverse_table.mk, built by build()):
the diverse search with traversal distances read from a table, and the optional full-precision rerank.
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import diverse_oracle
import oracle_lib as O

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        diverse_oracle.lib()  # liboracle_diverse_search.so, whose queue this library drives
        path = os.path.join(O.ORACLE_DIR, "liboracle_diverse_table.so")
        src = os.path.join(O.ORACLE_DIR, "diverse_table.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "diverse_table.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        fn = L.orc_search_batch_diverse_table
        fn.restype = None
        fn.argtypes = [C.POINTER(O.OrcIndex), vp, vp, u64, u32, u32, u32, u32, u32, vp, vp, vp, i, i, vp, vp, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def search_batch_table(index, tables, queries, k, l_search, diverse_k, values, present=None, beam=1, deleted=None, rerank=False,
                       flavour=O.AVX2):
    """orc_search_batch_diverse_table over an O.Index: the traversal distance of query q to id i is tables[q][i] (f32, one
    row per query over every id); with `rerank` the post-processed list is reranked by full-precision distance to
    `queries` (index dtype).  Returns as diverse_oracle.search_batch: (ids, dists, counts, cmps, hops, failed removals)."""
    tables = np.ascontiguousarray(tables, np.float32)
    total = index.n_points + index.n_start
    nq = tables.shape[0]
    assert tables.shape == (nq, total)
    values = np.ascontiguousarray(values, np.uint32)
    present = np.ones(total, np.uint8) if present is None else np.ascontiguousarray(present, np.uint8)
    assert values.shape == (total,) and present.shape == (total,)
    words = None
    if deleted is not None:
        bits = np.zeros(((total + 31) // 32) * 32, np.uint8)
        bits[:total] = np.asarray(deleted, bool)
        words = np.packbits(bits, bitorder="little").view(np.uint32).copy()
    q = None if queries is None else np.ascontiguousarray(queries)
    assert not rerank or (q is not None and q.shape[0] == nq)
    ids = np.empty((nq, k), np.uint32)
    dists = np.empty((nq, k), np.float32)
    counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
    failed = np.empty(nq, np.uint64)
    lib().orc_search_batch_diverse_table(C.byref(index.c), O.ptr(tables), None if q is None else O.ptr(q), 0 if q is None else q.strides[0],
                                         nq, k, l_search, beam, diverse_k, O.ptr(values), O.ptr(present),
                                         None if words is None else O.ptr(words), int(bool(rerank)), flavour, O.ptr(ids), O.ptr(dists),
                                         O.ptr(counts), O.ptr(cmps), O.ptr(hops), O.ptr(failed))
    return ids, dists, counts, cmps, hops, failed
