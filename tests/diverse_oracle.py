"""ctypes binding of oracle/diverse_search.cpp (liboracle_diverse_search.so, oracle/diverse_search.mk, built by build()).
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_diverse_search.so")
        src = os.path.join(O.ORACLE_DIR, "diverse_search.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "diverse_search.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i, f = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float
        pu, pf, pi = C.POINTER(u32), C.POINTER(f), C.POINTER(i)
        sig = {
            "orc_npq_new": (vp, [u32]), "orc_npq_free": (None, [vp]), "orc_npq_insert": (None, [vp, u32, f]),
            "orc_npq_remove": (i, [vp, u32, f]), "orc_npq_retain": (None, [vp, vp]), "orc_npq_truncate": (None, [vp, u32]),
            "orc_npq_size": (u32, [vp]), "orc_npq_cursor": (u32, [vp]), "orc_npq_has_notvisited": (i, [vp]),
            "orc_npq_closest_notvisited": (i, [vp, pu, pf]), "orc_npq_get": (None, [vp, u32, pu, pf, pi]),
            "orc_diverse_queue_new": (vp, [u32, u32, u32, vp, vp, u64]), "orc_diverse_queue_free": (None, [vp]),
            "orc_diverse_queue_insert": (None, [vp, u32, f]), "orc_diverse_queue_post_process": (None, [vp]),
            "orc_diverse_queue_clear": (None, [vp]), "orc_diverse_queue_size": (u32, [vp]), "orc_diverse_queue_capacity": (u32, [vp]),
            "orc_diverse_queue_search_l": (u32, [vp]), "orc_diverse_queue_diverse_l": (u32, [vp]),
            "orc_diverse_queue_get": (None, [vp, u32, pu, pf, pi]), "orc_diverse_queue_has_notvisited": (i, [vp]),
            "orc_diverse_queue_closest_notvisited": (i, [vp, pu, pf]), "orc_diverse_queue_n_local": (u32, [vp]),
            "orc_diverse_queue_local_size": (i, [vp, u32]), "orc_diverse_queue_local_get": (None, [vp, u32, u32, pu, pf]),
            "orc_diverse_queue_failed_removals": (u64, [vp]),
            "orc_search_batch_diverse": (None, [C.POINTER(O.OrcIndex), vp, u64, u32, u32, u32, u32, u32, vp, vp, vp, i, vp, vp, vp, vp, vp,
                                                vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _LIB = L
    return _LIB


class Npq:
    """NeighborPriorityQueue (fixed capacity) of the oracle."""

    def __init__(self, capacity):
        self.h = lib().orc_npq_new(capacity)

    def __del__(self):
        lib().orc_npq_free(self.h)

    def insert(self, id_, d):
        lib().orc_npq_insert(self.h, id_, d)

    def remove(self, id_, d):
        return bool(lib().orc_npq_remove(self.h, id_, d))

    def retain(self, pred):
        keep = np.array([bool(pred(i, d)) for i, d, _ in self.entries()], np.uint8)
        lib().orc_npq_retain(self.h, O.ptr(keep) if keep.size else None)

    def truncate(self, n):
        lib().orc_npq_truncate(self.h, n)

    def size(self):
        return lib().orc_npq_size(self.h)

    @property
    def cursor(self):
        return lib().orc_npq_cursor(self.h)

    def has_notvisited_node(self):
        return bool(lib().orc_npq_has_notvisited(self.h))

    def closest_notvisited(self):
        i, d = C.c_uint32(), C.c_float()
        return (i.value, d.value) if lib().orc_npq_closest_notvisited(self.h, C.byref(i), C.byref(d)) else None

    def get(self, n):
        assert n < self.size(), "index out of bounds"
        i, d, v = C.c_uint32(), C.c_float(), C.c_int()
        lib().orc_npq_get(self.h, n, C.byref(i), C.byref(d), C.byref(v))
        return i.value, d.value, bool(v.value)

    def entries(self):
        return [self.get(n) for n in range(self.size())]


class DiverseQueue:
    """DiverseNeighborQueue of the oracle over the attribute map `attrs` ({id: value}; other ids have none)."""

    def __init__(self, l_value, k_value, diverse_k, attrs):
        n = max(attrs) + 1 if attrs else 1
        self._values = np.zeros(n, np.uint32)
        self._present = np.zeros(n, np.uint8)
        for i, a in attrs.items():
            self._values[i], self._present[i] = a, 1
        self.h = lib().orc_diverse_queue_new(l_value, k_value, diverse_k, O.ptr(self._values), O.ptr(self._present), n)

    def __del__(self):
        lib().orc_diverse_queue_free(self.h)

    def insert(self, id_, d):
        lib().orc_diverse_queue_insert(self.h, id_, d)

    def post_process(self):
        lib().orc_diverse_queue_post_process(self.h)

    def clear(self):
        lib().orc_diverse_queue_clear(self.h)

    def size(self):
        return lib().orc_diverse_queue_size(self.h)

    def capacity(self):
        return lib().orc_diverse_queue_capacity(self.h)

    def search_l(self):
        return lib().orc_diverse_queue_search_l(self.h)

    def diverse_results_l(self):
        return lib().orc_diverse_queue_diverse_l(self.h)

    def get(self, n):
        assert n < self.size(), "index out of bounds"
        i, d, v = C.c_uint32(), C.c_float(), C.c_int()
        lib().orc_diverse_queue_get(self.h, n, C.byref(i), C.byref(d), C.byref(v))
        return i.value, d.value

    def iter(self):
        return [self.get(n) for n in range(min(self.size(), self.search_l()))]

    def has_notvisited_node(self):
        return bool(lib().orc_diverse_queue_has_notvisited(self.h))

    def closest_notvisited(self):
        i, d = C.c_uint32(), C.c_float()
        return (i.value, d.value) if lib().orc_diverse_queue_closest_notvisited(self.h, C.byref(i), C.byref(d)) else None

    def n_local(self):
        return lib().orc_diverse_queue_n_local(self.h)

    def local_size(self, a):
        n = lib().orc_diverse_queue_local_size(self.h, a)
        return None if n < 0 else n

    def local_get(self, a, n):
        i, d = C.c_uint32(), C.c_float()
        lib().orc_diverse_queue_local_get(self.h, a, n, C.byref(i), C.byref(d))
        return i.value, d.value

    def failed_removals(self):
        return lib().orc_diverse_queue_failed_removals(self.h)


def search_batch(index, queries, k, l_search, diverse_k, values, present=None, beam=1, deleted=None, flavour=O.AVX2):
    """orc_search_batch_diverse over an O.Index: (ids, dists, counts, cmps, hops, failed removals per query).  `values` /
    `present` cover every id of the index; `deleted`: bool per id, or None."""
    queries = np.ascontiguousarray(queries)
    total = index.n_points + index.n_start
    values = np.ascontiguousarray(values, np.uint32)
    present = np.ones(total, np.uint8) if present is None else np.ascontiguousarray(present, np.uint8)
    assert values.shape == (total,) and present.shape == (total,)
    words = None
    if deleted is not None:
        bits = np.zeros(((total + 31) // 32) * 32, np.uint8)
        bits[:total] = np.asarray(deleted, bool)
        words = np.packbits(bits, bitorder="little").view(np.uint32).copy()
    nq = queries.shape[0]
    ids = np.empty((nq, k), np.uint32)
    dists = np.empty((nq, k), np.float32)
    counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
    failed = np.empty(nq, np.uint64)
    lib().orc_search_batch_diverse(C.byref(index.c), O.ptr(queries), queries.strides[0], nq, k, l_search, beam, diverse_k, O.ptr(values),
                                   O.ptr(present), None if words is None else O.ptr(words), flavour, O.ptr(ids), O.ptr(dists),
                                   O.ptr(counts), O.ptr(cmps), O.ptr(hops), O.ptr(failed))
    return ids, dists, counts, cmps, hops, failed
