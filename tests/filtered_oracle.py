"""ctypes binding of oracle/filtered_search.cpp (liboracle_filtered_search.so, oracle/filtered_search.mk, built by build()),
and an independent Python restatement of the reference's inline filtered search to pin it.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

import oracle_lib as O

_LIB = None
EMPTY = 0xFFFFFFFF


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_filtered_search.so")
        src = os.path.join(O.ORACLE_DIR, "filtered_search.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "filtered_search.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i, dbl = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_double
        L.orc_compute_adaptive_l.restype, L.orc_compute_adaptive_l.argtypes = u64, [u64, u64, u64, dbl]
        L.orc_search_batch_filtered.restype = None
        L.orc_search_batch_filtered.argtypes = [C.POINTER(O.OrcIndex), vp, u64, u32, u32, u32, u32, vp, vp, i, u32, dbl, vp, i, vp, vp, vp,
                                                vp, vp]
        _LIB = L
    return _LIB


def compute_adaptive_l(base_l, visited, matched, scale):
    return int(lib().orc_compute_adaptive_l(base_l, visited, matched, scale))


def deleted_words(deleted, total):
    bits = np.zeros(((total + 31) // 32) * 32, np.uint8)
    bits[:total] = np.asarray(deleted, bool)
    return np.packbits(bits, bitorder="little").view(np.uint32).copy()


def search_batch(index, queries, k, l_search, labels, masks, match_all=False, adaptive_l=None, beam=1, deleted=None, flavour=O.AVX2):
    """orc_search_batch_filtered over an O.Index: (ids, dists, counts, cmps, hops).  `labels`: u64 per id of the index;
    `masks`: u64 per query (or one); adaptive_l: None or (samples, scale); `deleted`: bool per id, or None."""
    queries = np.ascontiguousarray(queries)
    nq = queries.shape[0]
    total = index.n_points + index.n_start
    labels = np.ascontiguousarray(labels, np.uint64)
    assert labels.shape == (total,)
    masks = np.ascontiguousarray(np.broadcast_to(np.asarray(masks, np.uint64), (nq,)))
    samples, scale = adaptive_l if adaptive_l is not None else (0, 1.0)
    words = None if deleted is None else deleted_words(deleted, total)
    ids = np.empty((nq, k), np.uint32)
    dists = np.empty((nq, k), np.float32)
    counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
    lib().orc_search_batch_filtered(C.byref(index.c), O.ptr(queries), queries.strides[0], nq, k, l_search, beam, O.ptr(labels), O.ptr(masks),
                                    int(bool(match_all)), samples, scale, None if words is None else O.ptr(words), flavour, O.ptr(ids),
                                    O.ptr(dists), O.ptr(counts), O.ptr(cmps), O.ptr(hops))
    return ids, dists, counts, cmps, hops


# ---------------------------------------------------------------- the reference's search, restated in Python

def py_adaptive_l(base_l, visited, matched, scale):
    """compute_adaptive_l (inline_filter_search.rs:294-310)"""
    if matched == 0 or visited == 0:
        return int(base_l * scale)
    s = matched / visited
    m = 1.0 if s >= 0.5 else 2.0 if s >= 0.1 else 2.0 ** (-math.log10(s))
    return int(base_l * min(max(m, 1.0), scale))


def py_search(vecs, adj, n_points, n_start, metric, query, k, L, labels, mask, match_all=False, adaptive_l=None, beam=1, deleted=None):
    """inline_filter_search_internal with NeighborPriorityQueue::{insert, closest_notvisited, reconfigure}, then a stable
    sort of the matches (NaN last), take(L) and the post-processing that drops start points and deleted ids"""
    total = n_points + n_start
    q = np.ascontiguousarray(query.astype(np.float32) if vecs.dtype == np.float16 else query)
    dist = lambda ids: O.distance_rows(q, vecs[ids], metric, O.AVX2)
    accept = lambda i: (int(labels[i]) & mask) == mask if match_all else (int(labels[i]) & mask) != 0
    best = {"cap": L + n_start, "ids": [], "ds": [], "done": [], "cursor": 0}

    def insert(i, d):
        if np.isnan(d):
            return
        if len(best["ids"]) == best["cap"] and best["ds"][-1] < d:
            return
        at = next((j for j, x in enumerate(best["ds"]) if x >= d), len(best["ds"]))
        if len(best["ids"]) == best["cap"]:
            for key in ("ids", "ds", "done"):
                del best[key][-1]
        best["ids"].insert(at, i), best["ds"].insert(at, d), best["done"].insert(at, False)
        best["cursor"] = min(best["cursor"], at)

    def closest_notvisited():
        if best["cursor"] >= min(best["cap"], len(best["ids"])):
            return None
        c = best["cursor"]
        best["done"][c] = True
        best["cursor"] += 1
        while best["cursor"] < len(best["ids"]) and best["done"][best["cursor"]]:
            best["cursor"] += 1
        return best["ids"][c]

    matched = []
    visited = set(range(n_points, total))
    for i, d in zip(range(n_points, total), dist(np.arange(n_points, total))):
        insert(i, d)
        if accept(i):
            matched.append((i, d))
    cmps = hops = sv = sm = 0
    adjusted = False
    while True:
        nodes = []
        while len(nodes) < beam:
            u = closest_notvisited()
            if u is None:
                break
            nodes.append(u)
        if not nodes:
            break
        fresh = []
        for u in nodes:
            for v in adj[u, 1:1 + adj[u, 0]].tolist():
                if v in visited:
                    continue
                visited.add(v)
                if v < total:
                    fresh.append(v)
        for i, d in zip(fresh, dist(np.array(fresh, np.int64)) if fresh else []):
            if accept(i):
                matched.append((i, d))
                sm += 1
            insert(i, d)
            sv += 1
        cmps += len(fresh)
        hops += len(nodes)
        if adaptive_l is not None and not adjusted and sv >= adaptive_l[0]:
            adjusted = True
            new_l = py_adaptive_l(L, sv, sm, adaptive_l[1])
            if new_l > L:  # reconfigure
                if new_l < len(best["ids"]):
                    for key in ("ids", "ds", "done"):
                        del best[key][new_l:]
                    best["cursor"] = min(best["cursor"], new_l)
                best["cap"] = new_l
    matched.sort(key=lambda m: (bool(np.isnan(m[1])), 0.0 if np.isnan(m[1]) else float(m[1])))  # stable
    out = [(i, d) for i, d in matched[:L] if i < n_points and not (deleted is not None and deleted[i])][:k]
    ids = np.full(k, EMPTY, np.uint32)
    ds = np.full(k, np.inf, np.float32)
    ids[:len(out)] = [i for i, _ in out]
    ds[:len(out)] = [d for _, d in out]
    return ids, ds, len(out), cmps, hops


def py_batch(vecs, adj, n_points, n_start, metric, queries, k, L, labels, masks, match_all=False, adaptive_l=None, beam=1, deleted=None):
    masks = np.broadcast_to(np.asarray(masks, np.uint64), (queries.shape[0],))
    rows = [py_search(vecs, adj, n_points, n_start, metric, q, k, L, labels, int(m), match_all, adaptive_l, beam, deleted)
            for q, m in zip(queries, masks)]
    return tuple(np.array([r[j] for r in rows]).astype(dt) for j, dt in enumerate((np.uint32, np.float32, np.uint32, np.uint32, np.uint32)))
