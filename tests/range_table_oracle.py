"""ctypes binding of oracle/range_table.cpp (liboracle_range_table.so, oracle/range_table.mk, built by build()): the range
search with every traversal distance read from a table, and the optional full-precision rerank.
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O
import range_oracle as R

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_range_table.so")
        src = os.path.join(O.ORACLE_DIR, "range_table.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "range_table.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i, f = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float
        L.orc_range_search_table.restype = u64
        L.orc_range_search_table.argtypes = [C.POINTER(O.OrcIndex), vp, vp, u32, u32, f, i, f, f, f, u64, vp, i, i, vp, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def range_search_table(index, tables, queries, l_search, radius, beam=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                       max_returned=None, deleted=None, rerank=False, flavour=O.AVX2):
    """orc_range_search_table over an O.Index, one query after another: the traversal distance of query q to id i is
    tables[q][i]; with `rerank` the results are reranked by full-precision distance to `queries` (index dtype, may be
    None without rerank).  Returns as range_oracle.range_search: (offsets, ids, dists, cmps, hops, second_round)."""
    assert R.check(l_search, radius, beam, inner_radius, initial_slack, range_slack, max_returned) is None
    tables = np.ascontiguousarray(tables, np.float32)
    total = index.n_points + index.n_start
    nq = tables.shape[0]
    assert tables.shape == (nq, total)
    q = None if queries is None else np.ascontiguousarray(queries)
    assert not rerank or (q is not None and q.shape[0] == nq)
    words = None if deleted is None else R.deleted_words(deleted, total)
    ids = np.empty(max(index.n_points, 1), np.uint32)
    dists = np.empty(max(index.n_points, 1), np.float32)
    cmps, hops = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
    second = np.empty(nq, np.uint8)
    offsets, all_ids, all_dists = [0], [], []
    c, h, s = C.c_uint32(), C.c_uint32(), C.c_uint8()
    for i in range(nq):
        n = lib().orc_range_search_table(C.byref(index.c), O.ptr(tables[i]), None if q is None else q[i].ctypes.data, l_search, beam, radius,
                                         inner_radius is not None, 0.0 if inner_radius is None else inner_radius, initial_slack,
                                         range_slack, max_returned or 0, None if words is None else O.ptr(words), int(bool(rerank)),
                                         flavour, O.ptr(ids), O.ptr(dists), C.byref(c), C.byref(h), C.byref(s))
        all_ids.append(ids[:n].copy())
        all_dists.append(dists[:n].copy())
        offsets.append(offsets[-1] + n)
        cmps[i], hops[i], second[i] = c.value, h.value, s.value
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.empty(0, dt)
    return np.array(offsets, np.uint64), cat(all_ids, np.uint32), cat(all_dists, np.float32), cmps, hops, second
