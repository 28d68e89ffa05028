"""ctypes binding of the insert oracle (oracle/insert.cpp -> liboracle_insert.so, built by oracle/insert.mk).  TEST
INFRASTRUCTURE ONLY: tests/test_insert.py and tools/bench_insert.py --parity load it."""
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
        path = os.path.join(O.ORACLE_DIR, "liboracle_insert.so")
        src = os.path.join(O.ORACLE_DIR, "insert.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "insert.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, f, i, u32, u64 = C.c_void_p, C.c_float, C.c_int, C.c_uint32, C.c_uint64
        L.orc_insert_batched.restype = None
        L.orc_insert_batched.argtypes = [i, i, u32, u64, u32, vp, u64, u32, u32, u32, f, vp, u64, u32, i, vp, u32,
                                         C.POINTER(u64), C.POINTER(u64)]
        _LIB = L
    return _LIB


def insert_batched(vectors, adj, ids, n_points, n_start, metric, pruned_degree, max_degree, l_build, alpha=1.2, batch_size=0,
                   tie_mode=0, counts=False):
    """dab_insert's linking: `ids` in consecutive chunks of batch_size (0: 65536), one multi_insert each (no bootstrap), on
    a copy of `adj` ([n_points + n_start, max_degree + 1]); `vectors` already hold the new rows.  tie_mode 1: exactly tied
    prune candidates ordered as oracle_lib.build_graph(tie_mode=1) orders them.  Returns the new adjacency, and with
    counts=True also (set_neighbors, append_neighbors) of the call."""
    vectors = np.ascontiguousarray(vectors)
    adj = np.array(adj, np.uint32, copy=True)
    assert adj.shape == (n_points + n_start, max_degree + 1)
    ids = np.ascontiguousarray(ids, np.uint32).ravel()
    sets, appends = C.c_uint64(), C.c_uint64()
    lib().orc_insert_batched(O.dtype_code(vectors), metric, vectors.shape[1], n_points, n_start, O.ptr(vectors), vectors.strides[0],
                             pruned_degree, max_degree, l_build, alpha, O.ptr(ids), ids.shape[0], batch_size, tie_mode, O.ptr(adj),
                             adj.shape[1], C.byref(sets), C.byref(appends))
    return (adj, (sets.value, appends.value)) if counts else adj
