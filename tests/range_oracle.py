"""ctypes binding of oracle/range_search.cpp (liboracle_range_search.so, oracle/range_search.mk, built by build()).
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

_LIB = None

# Range::validate_and_create's errors, numbered as orc_range_check returns them
ERRORS = {1: "BeamWidthZero", 2: "LZero", 3: "MaxReturnedLessThanInitialL", 4: "StartingListSlackValueError",
          5: "RangeSearchSlackValueError", 6: "InnerRadiusValueError"}


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_range_search.so")
        src = os.path.join(O.ORACLE_DIR, "range_search.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "range_search.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i, f = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float
        L.orc_range_check.restype = i
        L.orc_range_check.argtypes = [u32, u32, u64, f, i, f, f, f]
        L.orc_range_search.restype = u64
        L.orc_range_search.argtypes = [C.POINTER(O.OrcIndex), vp, u32, u32, f, i, f, f, f, u64, vp, i, vp, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def check(l_search, radius, beam=1, inner_radius=None, initial_slack=1.0, range_slack=1.0, max_returned=None):
    """The name of the error Range::validate_and_create returns for these arguments, or None"""
    rc = lib().orc_range_check(l_search, beam, max_returned or 0, radius, inner_radius is not None,
                               0.0 if inner_radius is None else inner_radius, initial_slack, range_slack)
    return ERRORS.get(rc)


def deleted_words(deleted, total):
    bits = np.zeros(((total + 31) // 32) * 32, np.uint8)
    bits[:total] = np.asarray(deleted, bool)
    return np.packbits(bits, bitorder="little").view(np.uint32).copy()


def range_search(index, queries, l_search, radius, beam=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                 max_returned=None, deleted=None, flavour=O.AVX2):
    """orc_range_search over an O.Index, one query after another: (offsets [nq + 1] u64, ids, dists, cmps, hops,
    second_round) with the results of query q at offsets[q]:offsets[q + 1].  `deleted`: bool per id, or None."""
    assert check(l_search, radius, beam, inner_radius, initial_slack, range_slack, max_returned) is None
    queries = np.ascontiguousarray(queries)
    total = index.n_points + index.n_start
    words = None if deleted is None else deleted_words(deleted, total)
    nq = queries.shape[0]
    ids = np.empty(max(index.n_points, 1), np.uint32)
    dists = np.empty(max(index.n_points, 1), np.float32)
    cmps, hops = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
    second = np.empty(nq, np.uint8)
    offsets, all_ids, all_dists = [0], [], []
    c, h, s = C.c_uint32(), C.c_uint32(), C.c_uint8()
    for q in range(nq):
        n = lib().orc_range_search(C.byref(index.c), queries[q].ctypes.data, l_search, beam, radius, inner_radius is not None,
                                   0.0 if inner_radius is None else inner_radius, initial_slack, range_slack, max_returned or 0,
                                   None if words is None else O.ptr(words), flavour, O.ptr(ids), O.ptr(dists), C.byref(c),
                                   C.byref(h), C.byref(s))
        all_ids.append(ids[:n].copy())
        all_dists.append(dists[:n].copy())
        offsets.append(offsets[-1] + n)
        cmps[q], hops[q], second[q] = c.value, h.value, s.value
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.empty(0, dt)
    return np.array(offsets, np.uint64), cat(all_ids, np.uint32), cat(all_dists, np.float32), cmps, hops, second
