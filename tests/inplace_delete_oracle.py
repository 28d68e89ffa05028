"""ctypes binding of the in-place delete oracle (oracle/inplace_delete.cpp -> liboracle_inplace_delete.so, built by
oracle/inplace_delete.mk).  TEST INFRASTRUCTURE ONLY: tests/test_inplace_delete.py and tools/bench_inplace_delete.py
--parity load it."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

VISITED_AND_TOPK, TWO_HOP_AND_ONE_HOP, ONE_HOP = 0, 1, 2
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_inplace_delete.so")
        src = os.path.join(O.ORACLE_DIR, "inplace_delete.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "inplace_delete.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, f, i, u32, u64 = C.c_void_p, C.c_float, C.c_int, C.c_uint32, C.c_uint64
        L.orc_inplace_delete.restype = None
        L.orc_inplace_delete.argtypes = [i, i, u32, u64, u32, vp, u64, u32, vp, u32, vp, vp, u64, i, u32, u32, u32, u32, f, u32, i]
        L.orc_drop_deleted_neighbors.restype = u64
        L.orc_drop_deleted_neighbors.argtypes = [u64, u32, u32, vp, u32, vp, u32, i]
        _LIB = L
    return _LIB


def deleted_words(n_total, ids=()):
    """The deletion bitmap of `ids` over n_total ids."""
    words = np.zeros((n_total + 31) // 32, np.uint32)
    for i in np.asarray(ids, np.int64).ravel():
        words[i >> 5] |= np.uint32(1 << (int(i) & 31))
    return words


def deleted_ids(words, n_total):
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:n_total]
    return np.flatnonzero(bits).astype(np.uint32)


def inplace_delete(vectors, adj, deleted, ids, n_points, n_start, metric, method, num_to_replace, pruned_degree, alpha=1.2,
                   k_value=20, l_value=50, batch_size=1, single=False):
    """dab_inplace_delete on copies: adj [n_points + n_start, max_degree + 1] and the bitmap `deleted`; returns both.
    single=True: inplace_delete called id by id."""
    vectors = np.ascontiguousarray(vectors)
    adj = np.array(adj, np.uint32, copy=True)
    deleted = np.array(deleted, np.uint32, copy=True)
    ids = np.ascontiguousarray(ids, np.uint32).ravel()
    lib().orc_inplace_delete(O.dtype_code(vectors), metric, vectors.shape[1], n_points, n_start, O.ptr(vectors), vectors.strides[0],
                             adj.shape[1] - 1, O.ptr(adj), adj.shape[1], O.ptr(deleted), O.ptr(ids), ids.shape[0], method,
                             num_to_replace, k_value, l_value, pruned_degree, alpha, batch_size, 1 if single else 0)
    return adj, deleted


def drop_deleted_neighbors(adj, deleted, n_points, n_start, pruned_degree, only_orphans=False):
    """dab_drop_deleted_neighbors on a copy of adj; returns (adj, lists written)."""
    adj = np.array(adj, np.uint32, copy=True)
    deleted = np.ascontiguousarray(deleted, np.uint32)
    n = lib().orc_drop_deleted_neighbors(n_points, n_start, adj.shape[1] - 1, O.ptr(adj), adj.shape[1], O.ptr(deleted), pruned_degree,
                                         1 if only_orphans else 0)
    return adj, int(n)
